"""H.264 Intra 4x4 on the H100 (pantomatrix_b200/video.py, intra4x4=True): the samples are byte for byte the CPU
restatement's (tests/h264_ref.py) on the CPU cases, random clips and the first frames of rendered EMAGE and CaMN
clips at qp 0, 20 and 51, through all three kernels (gop 1, gop > 1 with search 0, search > 0); each GOP encodes as it
does alone at the same parity; calls are deterministic and capture in a CUDA graph; a 300-frame gop 30 write_mp4 file
decodes to the restatement's reconstruction."""
import numpy as np
import pytest
import torch

import h264_ref as R
from test_video import decode
from test_video_gop_gpu import rendered_gop  # noqa: F401  (the module fixture)
from test_video_i4 import GOPS, gop_of, i4_cases
from pantomatrix_b200 import video

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _samples(frames, qp, gop, search, intra4x4=True):
    data, nbytes = video.encode(frames, qp=qp, gop=gop, search=search, intra4x4=intra4x4)
    data, nbytes = data.cpu().numpy(), nbytes.cpu().numpy()
    assert all(not data[i, k:].any() for i, k in enumerate(nbytes))
    return [data[i, :k].tobytes() for i, k in enumerate(nbytes)]


@pytest.mark.parametrize("g", GOPS, ids=[str(g) for g in GOPS])
@pytest.mark.parametrize("name,frames,qp,search", i4_cases(), ids=[c[0] for c in i4_cases()])
def test_i4_cases_are_byte_identical_to_the_restatement(name, frames, qp, search, g):
    gop = gop_of(g, len(frames))
    got = _samples(torch.as_tensor(np.stack(frames), device=DEV), qp, gop, search)
    assert got == [e[0] for e in R.encode_clip(frames, qp, gop, search, True)]


def test_random_clips_are_byte_identical_to_the_restatement():
    rng = np.random.default_rng(19)
    for h, w in ((16, 32), (48, 64), (96, 160)):
        base = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        base[:, : w // 2] = base[:, : w // 2] // 64 * 64           # flat steps beside noise
        clip = [base]
        for t in range(1, 4):
            f = np.roll(clip[-1], (int(rng.integers(-3, 4)), int(rng.integers(-5, 6))), (0, 1))
            y, x = rng.integers(0, h - 8), rng.integers(0, w - 8)
            f[y:y + 8, x:x + 8] = rng.integers(0, 256, (8, 8, 3))
            clip.append(f)
        for qp, gop, search in ((0, 1, 0), (12, 3, 0), (30, 4, 7), (45, 2, 16)):
            got = _samples(torch.as_tensor(np.stack(clip), device=DEV), qp, gop, search)
            want = R.encode_clip(clip, qp, gop, search, True)
            for i, (b, e) in enumerate(zip(got, want)):
                assert b == e[0], (h, w, qp, gop, search, i)
                assert len(b) <= video.max_bytes(h, w, gop)


@pytest.mark.parametrize("qp", [0, 20, 51])
def test_rendered_clips_are_byte_identical_to_the_restatement(rendered_gop, qp):
    emage, body = rendered_gop
    for clip, gop, search in ((emage[0, :1], 1, 0), (emage[0, :3], 3, 0), (emage[0, :3], 3, 16),
                              (body[1, :1], 1, 0), (body[1, :3], 3, 0), (body[1, :3], 3, 16)):
        got = _samples(clip, qp, gop, search)
        assert got == [e[0] for e in R.encode_clip(list(clip.cpu().numpy()), qp, gop, search, True)], (qp, gop, search)


@pytest.mark.parametrize("search", [0, 16])
def test_batch_encodes_each_gop_as_alone_at_the_same_parity(rendered_gop, search):
    _, body = rendered_gop
    clips = body[:, :9].contiguous()                     # (2, 9, ...): GOPs t = 0..3, 4..7, 8 at gop 4
    both = _samples(clips, 20, 4, search)
    for b in range(2):
        for t0 in (0, 4, 8):
            t1 = min(t0 + 4, 9)
            alone = _samples(clips[b, t0:t1], 20, 4, search)
            if (t0 // 4) % 2:                            # parity 1: the GOP after a GOP of the same frames
                alone = _samples(torch.cat([clips[b, t0:t1], clips[b, t0:t1]]), 20, t1 - t0, search)[t1 - t0:]
            assert alone == both[9 * b + t0:9 * b + t1], (b, t0)
    assert _samples(clips[0], 20, 4, search) == _samples(clips[:1], 20, 4, search) == both[:9]


@pytest.mark.parametrize("gop,search", [(1, 0), (3, 0), (3, 16)])
def test_deterministic_and_captured_replay_equals_eager(rendered_gop, gop, search):
    emage, _ = rendered_gop
    frames = emage[0, :6]
    a, na = video.encode(frames, gop=gop, search=search, intra4x4=True)
    b, nb = video.encode(frames, gop=gop, search=search, intra4x4=True)
    assert torch.equal(a, b) and torch.equal(na, nb)
    out = (torch.full_like(a, 0xAB), torch.zeros_like(na))
    video.encode(frames, out=out, gop=gop, search=search, intra4x4=True)
    torch.cuda.synchronize()
    out[0].fill_(0xCD)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        video.encode(frames, out=out, gop=gop, search=search, intra4x4=True)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], a) and torch.equal(out[1], na)


def test_write_mp4_gop_30_intra4x4_of_a_300_frame_render_decodes_to_the_reconstruction(rendered_gop, tmp_path):
    emage, _ = rendered_gop
    path = video.write_mp4(emage[0], str(tmp_path / "clip.mp4"), fps=30, gop=30, intra4x4=True)
    lumas, _, fps = decode(path)
    assert len(lumas) == 300 and fps == 30
    host = emage[0].cpu().numpy()
    for t0 in (0, 270):
        for i, e in enumerate(R.encode_clip(list(host[t0:t0 + 3]), 20, 30, 0, True)):
            assert np.array_equal(lumas[t0 + i].reshape(-1)[:720 * 960].reshape(720, 960), e[1][0]), t0 + i
