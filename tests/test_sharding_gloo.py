"""world_size-2 `gloo` tests (CPU) of the multi-GPU plumbing: contiguous clip sharding, checkpoint broadcast
from rank 0, sharded generate (kernels emulated by tests/fake_ops.py) == single-process generate."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def test_shard_range_partitions():
    from pantomatrix_b200.sharding import shard_range
    for n in (0, 1, 5, 32, 33, 256):
        for world in (1, 2, 3, 8):
            parts = [shard_range(n, r, world) for r in range(world)]
            assert parts[0][0] == 0 and parts[-1][1] == n
            assert all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
            sizes = [e - s for s, e in parts]
            assert max(sizes) - min(sizes) <= 1
    with pytest.raises(ValueError):
        shard_range(4, 2, 2)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_path):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    import fake_ops
    import pantomatrix_b200.ops as real
    from pantomatrix_b200.emage_audio import modeling
    from pantomatrix_b200 import sharding
    from helpers import build_product
    from oracle.weights import synth_audio
    for name in dir(fake_ops):
        if not name.startswith("_") and callable(getattr(fake_ops, name)) and hasattr(real, name):
            setattr(real, name, getattr(fake_ops, name))
    modeling._require_cuda = lambda module, what: torch.device("cpu")
    from pantomatrix_b200.emage_audio import engine
    engine.set_precision("fp32")
    # each rank starts from a DIFFERENT checkpoint; after the broadcast both must hold rank 0's
    model, vqm = build_product(seed=rank, device="cpu")
    nbytes = sharding.broadcast_checkpoint(model, vqm, src=0)
    probe = model.state_dict()["face_out_proj.weight"].double().sum() + vqm.vq_model_lower.state_dict()["decoder.main.8.bias"].double().sum()
    sums = [torch.zeros((), dtype=torch.double) for _ in range(world)]
    dist.all_gather(sums, probe)
    assert all(torch.equal(s, sums[0]) for s in sums), "checkpoint broadcast did not equalise the ranks"
    audio = torch.from_numpy(synth_audio(3, 21600, 77))                # 3 clips x 40 frames: uneven 2 + 1 split
    start, end, lat, pred = sharding.generate_sharded(model, vqm, audio)
    aa = sharding.gather_clips(pred["motion_axis_angle"], 3)
    idx = sharding.gather_clips(lat["cls_upper"].argmax(-1), 3)
    if rank == 0:
        torch.save({"aa": aa, "idx": idx, "nbytes": nbytes, "range": (start, end)}, out_path)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_rank_sharded_generate_matches_single_process(tmp_path, monkeypatch, request):
    out_path = str(tmp_path / "rank0.pt")
    mp.spawn(_worker, args=(2, _free_port(), out_path), nprocs=2, join=True)
    got = torch.load(out_path)
    assert got["range"] == (0, 2) and got["nbytes"] > 5e8            # 139 M + 14 M fp32 parameters
    # single-process reference with the same (rank-0) checkpoint and all three clips
    import fake_ops
    import pantomatrix_b200.ops as real
    from pantomatrix_b200.emage_audio import modeling
    from pantomatrix_b200.pipeline import generate
    from helpers import build_product, use_precision
    from oracle.weights import synth_audio
    for name in dir(fake_ops):
        if not name.startswith("_") and callable(getattr(fake_ops, name)) and hasattr(real, name):
            monkeypatch.setattr(real, name, getattr(fake_ops, name))
    monkeypatch.setattr(modeling, "_require_cuda", lambda module, what: torch.device("cpu"))
    use_precision(request, "fp32")
    model, vqm = build_product(seed=0, device="cpu")
    lat, pred = generate(model, vqm, torch.from_numpy(synth_audio(3, 21600, 77)))
    assert got["aa"].shape == pred["motion_axis_angle"].shape
    assert torch.equal(got["idx"], lat["cls_upper"].argmax(-1))
    assert (got["aa"] - pred["motion_axis_angle"]).abs().max() < 1e-3
