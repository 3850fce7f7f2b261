"""Host-logic tests (no GPU): the product's Python scheduling - window plan, audio hoisting, BatchNorm
folding and weight packing, tail-only seed decode, the reference-facing API - run with every kernel
wrapper replaced by tests/fake_ops.py, and compared with the oracle and the reference's golden outputs.
The kernels themselves are tested on the GPU (tests/test_kernels_gpu.py, tests/test_emage_gpu.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import emage_oracle as O
from oracle.weights import make_checkpoint, synth_audio
import fake_ops
from helpers import build_product, use_precision

PARTS = ("face", "upper", "hands", "lower")


@pytest.fixture()
def cpu_product(monkeypatch, request):
    import pantomatrix_b200.ops as real
    from pantomatrix_b200.emage_audio import modeling
    for name in dir(fake_ops):
        if not name.startswith("_") and callable(getattr(fake_ops, name)) and hasattr(real, name):
            monkeypatch.setattr(real, name, getattr(fake_ops, name))
    monkeypatch.setattr(modeling, "_require_cuda", lambda module, what: torch.device("cpu"))
    use_precision(request, "fp32")                       # exact fp32 engine unless a test selects a tensor-core mode
    return build_product(seed=0, device="cpu")


@pytest.mark.parametrize("case", ["tail11", "drop_tail", "short40", "seeded"])
def test_schedule_reproduces_reference(case, cpu_product, golden_dir):
    from pantomatrix_b200.pipeline import generate
    model, vqm = cpu_product
    g = np.load(os.path.join(golden_dir, f"case_{case}.npz"))
    bs, n = int(g["bs"]), int(g["n_samples"])
    audio = torch.from_numpy(synth_audio(bs, n, int(g["audio_seed"])))
    mm = torch.from_numpy(g["masked_motion"]) if "masked_motion" in g else None
    mk = torch.from_numpy(g["mask"]) if "mask" in g else None
    lat, pred = generate(model, vqm, audio, masked_motion=mm, mask=mk)
    for p in PARTS:
        assert np.array_equal(lat["cls_" + p].argmax(-1).numpy(), g["idx_cls_" + p]), p
        np.testing.assert_allclose(lat["rec_" + p].numpy()[:, ::7], g["rec_" + p], atol=5e-4, rtol=0)
    for k in ("expression", "motion_axis_angle", "trans", "all_motion4inference"):
        np.testing.assert_allclose(pred[k].numpy(), g[k], atol=1e-3, rtol=0, err_msg=k)   # the 1e-3 pose gate


def test_forward_and_decode_api(cpu_product):
    model, vqm = cpu_product
    sd, cfg, vq = make_checkpoint(seed=0)
    bs = 2
    g = torch.Generator().manual_seed(3)
    audio = torch.from_numpy(synth_audio(bs, 34112, 5))
    motion, mask = torch.randn(bs, 64, 337, generator=g) * 0.3, (torch.rand(bs, 64, 337, generator=g) > 0.3).float()
    spk = torch.zeros(bs, 1, dtype=torch.long)
    with torch.no_grad():
        want = O.emage_forward(sd, audio, spk, motion, mask)
    got = model.forward(audio, spk, motion, mask)
    assert set(got) == set(want)
    for k in want:
        assert (got[k] - want[k]).abs().max() < 5e-4, k
    idx = torch.randint(0, 256, (bs, 20), generator=g)
    out = vqm.decode(upper_index=idx, lower_index=idx, get_global_motion=True, ref_trans=torch.zeros(1, 3))
    with torch.no_grad():
        ref = O.vq_decode(vq, upper_index=idx, lower_index=idx, get_global_motion=True, ref_trans=torch.zeros(1, 3))
    assert set(out) == {"expression", "all_motion4inference", "motion_axis_angle", "trans"}
    for k in out:
        assert (out[k] - ref[k]).abs().max() < 2e-4, k
    with pytest.raises(UnboundLocalError):
        vqm.decode()
    with pytest.raises(ValueError):                     # fewer audio frames than motion frames (reference: cat fails)
        model.forward(audio[:, :20000], spk, motion, mask)


def test_wav_out_len_matches_reference_geometry():
    from pantomatrix_b200.emage_audio.engine import wav_out_len, window_plan
    assert wav_out_len(34112) == 64 and wav_out_len(31980) == 60 and wav_out_len(5863) == 12
    for L in (4, 40, 64, 68, 69, 124, 131, 300):
        assert window_plan(L, 64, 4) == O.window_plan(L, 64, 4)


@pytest.mark.parametrize("precision,atol", [("bf16x6", 5e-4), ("bf16x3", 5e-3), ("fp16x3", 5e-4)])
def test_tensor_core_schedule_host_logic(cpu_product, golden_dir, precision, atol):
    """The tensor-core engine's host side (weight packing into padded bf16 planes, strided convs as reshaped
    stride-1 problems, clips-per-tile views) reproduces the reference with the kernels emulated."""
    from pantomatrix_b200.emage_audio import engine
    from pantomatrix_b200.pipeline import generate
    model, vqm = cpu_product
    g = np.load(os.path.join(golden_dir, "case_tail11.npz"))
    audio = torch.from_numpy(synth_audio(int(g["bs"]), int(g["n_samples"]), int(g["audio_seed"])))
    engine.set_precision(precision)
    lat, pred = generate(model, vqm, audio)          # (the cpu_product fixture restores the precision mode)
    for p in PARTS:
        np.testing.assert_allclose(lat["rec_" + p].numpy()[:, ::7], g["rec_" + p], atol=atol, rtol=0)
        agree = (lat["cls_" + p].argmax(-1).numpy() == g["idx_cls_" + p]).mean()
        assert agree > (0.97 if precision == "bf16x3" else 0.999), (p, agree)


def test_precision_names_the_mode_that_runs(request):
    """get_precision() names the mode set_precision() selected; after ops.set_plane_format() changes the plane format
    under a mode it names the mode that now runs, or refuses when no mode runs that pair.  The fp32 engine builds no
    planes, so it stays fp32 whatever the plane format."""
    from pantomatrix_b200 import ops
    from pantomatrix_b200.emage_audio import engine
    use_precision(request, "fp32")
    assert sorted(engine.PRECISIONS) == ["bf16", "bf16x3", "bf16x6", "fp16x3", "fp32"]
    for name, (nsplit, fmt) in engine.PRECISIONS.items():
        engine.set_precision(name)
        assert engine.get_precision() == name and (engine._STATE["nsplit"], ops.plane_format()) == (nsplit, fmt)
    engine.set_precision("fp16x3")
    ops.set_plane_format("bf16")                     # two bf16 planes now run: bf16x3 arithmetic, fp32 attention kernel
    assert engine.get_precision() == "bf16x3" and not engine._attn_tc() and engine.overflow_flag("cpu") is None
    ops.set_plane_format("fp16")
    assert engine.get_precision() == "fp16x3" and engine._attn_tc()
    engine.set_precision("fp32")
    ops.set_plane_format("fp16")
    assert engine.get_precision() == "fp32" and not engine._attn_tc() and engine.overflow_flag("cpu") is None
    for name in ("bf16", "bf16x6"):
        engine.set_precision(name)
        ops.set_plane_format("fp16")
        with pytest.raises(RuntimeError, match="set_precision"):
            engine.get_precision()


@pytest.mark.parametrize("kind", ["camn", "disco"])
def test_lstm_models_host_logic(kind, cpu_product, golden_dir):
    """CaMN / DisCo host side (WavEncoder variant, LSTM weight packing, feature assembly, seed handling) with the
    kernels emulated, against the reference's golden outputs."""
    from helpers import build_lstm_product
    model = build_lstm_product(kind, device="cpu")
    g = np.load(os.path.join(golden_dir, f"case_{kind}.npz"))
    bs, n = int(g["bs"]), int(g["n_samples"])
    audio = torch.from_numpy(synth_audio(bs, n, int(g["audio_seed"])))
    spk = torch.zeros(bs, 1, dtype=torch.long)
    a = model(audio, spk, seed_frames=4, seed_motion=None)
    b = model(audio, spk, seed_frames=4, seed_motion=torch.from_numpy(g["seed_motion"]))
    t = g["motion"].shape[1]
    assert a["motion"].shape[:2] == (bs, t) and a["motion_axis_angle"].shape == (bs, t, 165)
    np.testing.assert_allclose(a["motion"].reshape(bs, t, -1).numpy(), g["motion"], atol=1e-4, rtol=0)
    np.testing.assert_allclose(b["motion"].reshape(bs, t, -1).numpy(), g["seeded_motion"], atol=1e-4, rtol=0)
    np.testing.assert_allclose(a["motion_axis_angle"].numpy(), g["motion_axis_angle"], atol=1e-3, rtol=0)
    assert model(audio, spk, return_axis_angle=False)["motion_axis_angle"] is None


def test_tokenisation_host_logic_vs_reference(cpu_product, golden_dir):
    """EmageVQModel.map2index / map2latent / spilt_inputs and EmageVQVAEConv.forward of the product (kernels emulated)
    against the real reference's outputs (tests/golden/case_tokenise.npz)."""
    _, vqm = cpu_product
    g = np.load(os.path.join(golden_dir, "case_tokenise.npz"))
    rot6d, expr = torch.from_numpy(g["rot6d"]), torch.from_numpy(g["expression"])
    contact, trans = torch.from_numpy(g["tar_contact"]), torch.from_numpy(g["tar_trans"])
    idx = vqm.map2index(rot6d, expr, tar_contact=contact, tar_trans=trans)
    idx0 = vqm.map2index(rot6d, expr)
    lat = vqm.map2latent(rot6d, expr, tar_contact=contact, tar_trans=trans)
    parts = vqm.spilt_inputs(rot6d, expr, tar_contact=contact, tar_trans=trans)
    models = dict(face=vqm.vq_model_face, upper=vqm.vq_model_upper, hands=vqm.vq_model_hands, lower=vqm.vq_model_lower)
    for p in PARTS:
        assert np.array_equal(parts[p].numpy(), g["input_" + p]), p
        assert np.array_equal(idx[p].numpy(), g["idx_" + p]) and np.array_equal(idx0[p].numpy(), g["idx_default_" + p]), p
        assert np.array_equal(lat[p].numpy(), g["latent_" + p]), p
        fw = models[p].forward(parts[p])
        assert set(fw) == {"poses_feat", "embedding_loss", "perplexity", "rec_pose"}
        np.testing.assert_allclose(fw["rec_pose"].numpy(), g["rec_pose_" + p], atol=5e-5, rtol=0)
        np.testing.assert_allclose(fw["poses_feat"].numpy(), g["poses_feat_" + p], atol=1e-6, rtol=0)
        np.testing.assert_allclose(float(fw["embedding_loss"]), float(g["embedding_loss_" + p]), rtol=1e-5)
        np.testing.assert_allclose(float(fw["perplexity"]), float(g["perplexity_" + p]), rtol=1e-5)

