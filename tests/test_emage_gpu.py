"""End-to-end parity of the CUDA path (GPU): the drop-in modules against (1) the committed golden outputs
of the unmodified reference and (2) the live CPU oracle on the same seeded weights and audio.

Gates (BASELINE.md section 6): emitted VQ code indices bit-exact; SMPL-X parameters within 1e-3 max-abs
(and geodesic error reported, because axis-angle is discontinuous at pi)."""
import os

import numpy as np
import pytest
import torch

from oracle import emage_oracle as O
from oracle.weights import make_checkpoint, synth_audio
from helpers import build_product, geodesic_deg

pytestmark = pytest.mark.gpu
PARTS = ("face", "upper", "hands", "lower")
GOLDEN = ["tail11", "clip10s", "drop_tail", "short40", "seeded"]


@pytest.fixture(scope="module")
def product():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return build_product(seed=0)


@pytest.fixture(autouse=True)
def _exact_engine_by_default():
    """Tests run on the exact-order fp32 engine unless they select a tensor-core mode themselves (the product
    default is fp16x3; it is exercised by the `precision` parametrisations below)."""
    from pantomatrix_b200.emage_audio import engine
    engine.set_precision("fp32")
    yield
    engine.set_precision(engine.DEFAULT_PRECISION)


@pytest.fixture(scope="module")
def ckpt():
    return make_checkpoint(seed=0)


def _pose_checks(pred, want_aa, want_expr, want_trans, tag, frames=None, raw=None):
    """1e-3 max-abs gate on the emitted SMPL-X parameters.  `frames` (bs,T) bool restricts the check to
    frames whose code indices all agree (see _face_ties).  `raw` (oracle decoder outputs) enables the
    conditioning-aware bound: the rot6d Gram-Schmidt of a random-weight decoder is occasionally ill
    conditioned (|a1| or |b2| << 1), where two fp32 evaluations of the 7-9 layer conv decoder (abs error
    ~3e-5) differ by ~1e-4 * kappa rad; the 1e-3 gate is enforced wherever kappa <= 10 (about 99 % of the
    joints) and the scaled bound elsewhere."""
    aa = pred["motion_axis_angle"].cpu()
    bs, T = aa.shape[:2]
    keep = torch.ones(bs, T, dtype=torch.bool) if frames is None else frames
    geo = torch.deg2rad(geodesic_deg(aa.reshape(bs, T, 55, 3), want_aa.reshape(bs, T, 55, 3)))
    allowed = torch.full_like(geo, 1e-3)
    if raw is not None:
        kappa = O.rot6d_condition(raw, bs, T)
        allowed = torch.maximum(allowed, 1e-4 * kappa)
        assert (kappa > 10).double().mean() < 0.03, (tag, "too many ill-conditioned joints to be a meaningful gate")
    bad = (geo > allowed) & keep[:, :, None]
    used = geo[keep[:, :, None].expand_as(geo)] / allowed[keep[:, :, None].expand_as(geo)]
    print(f"[{tag}] pose gate: max geodesic error {geo[keep[:, :, None].expand_as(geo)].max().item():.2e} rad, "
          f"largest fraction of the allowed bound used {used.max().item():.3f}"
          + (f", joints under the conditioning-aware bound (kappa > 10): {(allowed > 1e-3).double().mean().item():.4f}" if raw is not None else ""))
    assert not bad.any(), (tag, "geodesic rad", geo[bad].max().item(), int(bad.sum()))
    # component-wise check away from the axis-angle discontinuity at pi (|aa| error <= ~1.5 x geodesic there)
    far = ((want_aa.reshape(bs, T, 55, 3).norm(dim=-1) < 2.0) & (allowed <= 1e-3)).repeat_interleave(3, dim=-1) & keep[:, :, None]
    assert (aa - want_aa)[far].abs().max() < 1e-3, (tag, (aa - want_aa)[far].abs().max().item())
    assert (pred["expression"].cpu() - want_expr)[keep].abs().max() < 1e-3, tag
    if frames is None:
        assert (pred["trans"].cpu() - want_trans).abs().max() < 1e-3, tag


def _face_ties(vqm, vq, lat, want_lat, tag, max_ties=0):
    """Face codes come from an L2-argmin over fp32 distances |d| ~ 10^2..10^3 (M.py:64); when the two best
    codes are closer than the fp32 noise of the latents themselves (two fp32 evaluations of the 4-layer
    face decoder differ by ~1e-5 relative, which moves d by ~1e-3), the reference's own choice is decided
    by its GEMM summation order.  Every disagreement must be such a tie (judged in float64 on the ORACLE's latents), and their
    number is bounded.  Returns the (bs,T) mask of frames whose face codes agree."""
    got = vqm.vq_model_face._index_of(lat["rec_face"]).cpu()
    cb = vq["face"][0]["quantizer.embedding.weight"]
    want = O.l2_argmin(want_lat["rec_face"], cb)
    diff = got != want
    if diff.any():
        z = want_lat["rec_face"][diff].double()
        d = (z ** 2).sum(1, keepdim=True) + (cb.double() ** 2).sum(1) - 2 * z @ cb.double().t()
        gap = (d.gather(1, got[diff][:, None]) - d.gather(1, want[diff][:, None])).abs()[:, 0]
        rel = gap / d.min(1).values.abs()
        assert bool((rel < 2e-5).all()), (tag, "face index differs on a decidable row", rel.max().item())
    print(f"\n[{tag}] face codes differing from the oracle: {int(diff.sum())} of {diff.numel()} (allowed: {max_ties} proven fp64 ties)")
    assert int(diff.sum()) <= max_ties, (tag, f"{int(diff.sum())} undecidable face ties")
    # a code feeds a k=3 conv decoder with a +-9 frame receptive field: exclude the neighbourhood too
    near = torch.nn.functional.max_pool1d(diff.float().unsqueeze(1), 19, 1, 9)[:, 0] > 0
    return ~near


@pytest.mark.parametrize("precision", ["fp32", "bf16x6", "fp16x3"])
@pytest.mark.parametrize("case", GOLDEN)
def test_matches_reference_golden(case, precision, product, golden_dir):
    from pantomatrix_b200.emage_audio import engine
    from pantomatrix_b200.pipeline import generate
    model, vqm = product
    engine.set_precision(precision)
    g = np.load(os.path.join(golden_dir, f"case_{case}.npz"))
    bs, n = int(g["bs"]), int(g["n_samples"])
    audio = torch.from_numpy(synth_audio(bs, n, int(g["audio_seed"]))).cuda()
    mm = torch.from_numpy(g["masked_motion"]).cuda() if "masked_motion" in g else None
    mk = torch.from_numpy(g["mask"]).cuda() if "mask" in g else None
    lat, pred = generate(model, vqm, audio, masked_motion=mm, mask=mk)
    for p in PARTS:
        assert lat["cls_" + p].shape[1] == g["idx_cls_" + p].shape[1], "emitted length (tail-drop rule)"
        got = lat["cls_" + p].argmax(-1).cpu().numpy()
        assert np.array_equal(got, g["idx_cls_" + p]), (case, p, int((got != g["idx_cls_" + p]).sum()))
        np.testing.assert_allclose(lat["rec_" + p].cpu().numpy()[:, ::7], g["rec_" + p], atol=1e-3, rtol=0)
        np.testing.assert_allclose(lat["cls_" + p].cpu().numpy()[:, ::7], g["cls_" + p], atol=2e-3, rtol=0)
    face_idx = vqm.vq_model_face._index_of(lat["rec_face"]).cpu().numpy()
    assert np.array_equal(face_idx, g["idx_l2_face"])
    _pose_checks(pred, torch.from_numpy(g["motion_axis_angle"]), torch.from_numpy(g["expression"]),
                 torch.from_numpy(g["trans"]), case)
    assert (pred["all_motion4inference"].cpu() - torch.from_numpy(g["all_motion4inference"])).abs().max() < 1e-3


def test_single_window_forward_matches_oracle(product, ckpt):
    """EmageAudioModel.forward (M.py:265-341) on one 64-frame window with a random partial mask."""
    model, _ = product
    sd, cfg, vq = ckpt
    bs = 3
    g = torch.Generator().manual_seed(7)
    audio = torch.from_numpy(synth_audio(bs, 34112, 77))
    motion = torch.randn(bs, 64, 337, generator=g) * 0.3
    mask = (torch.rand(bs, 64, 337, generator=g) > 0.3).float()
    spk = torch.zeros(bs, 1, dtype=torch.long)
    with torch.no_grad():
        want = O.emage_forward(sd, audio, spk, motion, mask)
    got = model.forward(audio.cuda(), spk.cuda(), motion.cuda(), mask.cuda())
    for k, v in want.items():
        assert (got[k].cpu() - v).abs().max() < 1e-3, (k, (got[k].cpu() - v).abs().max().item())
        if k.startswith("cls_"):
            assert torch.equal(got[k].argmax(-1).cpu(), v.argmax(-1)), k


@pytest.mark.parametrize("precision", ["fp32", "fp16x3"])
@pytest.mark.parametrize("tag,flag", [("audio", True), ("noaudio", False)])
def test_forward_matches_reference_golden(product, golden_dir, tag, flag, precision):
    """forward() against the unmodified reference's outputs, with and without use_audio (M.py:310-311)."""
    import sys
    from pantomatrix_b200.emage_audio import engine
    sys.path.insert(0, golden_dir)
    from make_golden_forward import BS, inputs
    model, _ = product
    g = np.load(os.path.join(golden_dir, "case_forward.npz"))
    audio, motion, mask = inputs()
    engine.set_precision(precision)
    try:
        got = model.forward(audio.cuda(), torch.zeros(BS, 1, dtype=torch.long).cuda(), motion.cuda(), mask.cuda(), use_audio=flag)
    finally:
        engine.set_precision("fp32")
    for k, v in got.items():
        np.testing.assert_allclose(v.cpu().numpy()[:, ::3], g[f"{tag}_{k}"], atol=1e-3 if k.startswith("rec_") else 2e-3, rtol=0, err_msg=k)
        if k.startswith("cls_"):
            assert np.array_equal(v.argmax(-1).cpu().numpy(), g[f"{tag}_idx_{k}"]), k


def test_vq_decode_and_tokenise_match_oracle(product, ckpt):
    """EmageVQModel.decode (index and latent inputs, zero branches) and map2index (training-side
    tokenisation, all four L2-argmin lookups)."""
    _, vqm = product
    sd, cfg, vq = ckpt
    bs, t = 2, 37
    g = torch.Generator().manual_seed(11)
    idx = {p: torch.randint(0, 256, (bs, t), generator=g) for p in PARTS}
    lat = {p: torch.randn(bs, t, 256, generator=g) for p in PARTS}
    with torch.no_grad():
        want = O.vq_decode(vq, face_latent=lat["face"], upper_index=idx["upper"], hands_index=idx["hands"],
                           lower_index=idx["lower"], get_global_motion=True, ref_trans=torch.zeros(1, 3))
        want_partial = O.vq_decode(vq, upper_latent=lat["upper"])
    got = vqm.decode(face_latent=lat["face"].cuda(), upper_index=idx["upper"].cuda(), hands_index=idx["hands"].cuda(),
                     lower_index=idx["lower"].cuda(), get_global_motion=True, ref_trans=torch.zeros(1, 3).cuda())
    _pose_checks(got, want["motion_axis_angle"], want["expression"], want["trans"], "decode", raw=want["_raw"])
    got_partial = vqm.decode(upper_latent=lat["upper"].cuda())
    assert got_partial["trans"] is None and got_partial["expression"].abs().max() == 0
    assert geodesic_deg(got_partial["motion_axis_angle"].cpu().reshape(bs, t, 55, 3),
                        want_partial["motion_axis_angle"].reshape(bs, t, 55, 3)).max() < 0.0573
    # tokenisation: encoder conv stack + L2-argmin for each part
    rot6d = O.axis_angle_to_rot6d(torch.randn(bs, t, 55, 3, generator=g) * 0.4).reshape(bs, t, 330)
    expr = torch.randn(bs, t, 100, generator=g)
    tok = vqm.map2index(rot6d.cuda(), expr.cuda())
    r = rot6d.reshape(bs, t, 55, 6)
    inputs = dict(face=torch.cat([r[:, :, 22], expr], 2), upper=r[:, :, list(O.UPPER_JOINTS)].reshape(bs, t, 78),
                  hands=r[:, :, 25:55].reshape(bs, t, 180),
                  lower=torch.cat([r[:, :, list(O.LOWER_JOINTS)].reshape(bs, t, 54), torch.zeros(bs, t, 7)], 2))
    for p in PARTS:
        psd, pcfg = vq[p]
        with torch.no_grad():
            z = O.vq_encoder(psd, "encoder", inputs[p], pcfg["vae_layer"])
        assert torch.equal(tok[p].cpu(), O.l2_argmin(z, psd["quantizer.embedding.weight"])), p


def test_teacher_forced_windows_and_free_run_vs_oracle(product, ckpt):
    """bs=4 x 10 s: free-running generate() vs the oracle, plus per-window comparison on the oracle's own
    window inputs (so one flipped near-tie cannot hide or amplify later differences)."""
    from pantomatrix_b200.pipeline import generate
    model, vqm = product
    sd, cfg, vq = ckpt
    bs = 4
    audio = torch.from_numpy(synth_audio(bs, 160000, 4321))
    spk = torch.zeros(bs, 1, dtype=torch.long)
    trace = []
    with torch.no_grad():
        want_lat, want_pred = O.emage_generate(sd, cfg, vq, audio, spk, trace=trace)
    for i, w in enumerate(trace):                                     # teacher-forced single windows
        got = model.forward(w["audio"].cuda(), spk.cuda(), w["motion"].cuda(), w["mask"].cuda())
        for p in PARTS:
            a = got["cls_" + p].argmax(-1).cpu()
            assert torch.equal(a, w["idx"][p]), (i, p, int((a != w["idx"][p]).sum()))
            err = (got["rec_" + p].cpu() - w["out"]["rec_" + p]).abs().max().item()
            assert err < 1e-3, (i, p, err)
    lat, pred = generate(model, vqm, audio.cuda())
    for p in PARTS:
        a, b = lat["cls_" + p].argmax(-1).cpu(), want_lat["cls_" + p].argmax(-1)
        assert torch.equal(a, b), (p, int((a != b).sum()))
    ok = _face_ties(vqm, vq, lat, want_lat, "free-run", max_ties=2)
    _pose_checks(pred, want_pred["motion_axis_angle"], want_pred["expression"], want_pred["trans"], "free-run",
                 frames=None if ok.all() else ok, raw=want_pred["_raw"])


@pytest.mark.parametrize("precision", ["fp32", "bf16x6", "fp16x3"])
def test_baseline_config_batch32(product, ckpt, precision):
    """BASELINE configs[1]: 32 clips x 300 frames, free-running, for the exact fp32 engine and the default
    tensor-core mode.  Index agreement must be total on this seeded input; size-independent properties:
    emitted length, unit-norm orthogonal rot6d rows."""
    from pantomatrix_b200.emage_audio import engine
    from pantomatrix_b200.pipeline import generate
    model, vqm = product
    sd, cfg, vq = ckpt
    bs = 32
    audio = torch.from_numpy(synth_audio(bs, 160000, 1234))
    engine.set_precision(precision)
    try:
        lat, pred = generate(model, vqm, audio.cuda())
    finally:
        engine.set_precision("fp32")
    assert lat["rec_face"].shape == (bs, 300, 256) and pred["motion_axis_angle"].shape == (bs, 300, 165)
    m4 = pred["all_motion4inference"][:, :, :330].reshape(bs, 300, 55, 2, 3)
    assert (m4.norm(dim=-1) - 1).abs().max() < 1e-4 and (m4[..., 0, :] * m4[..., 1, :]).sum(-1).abs().max() < 1e-4
    with torch.no_grad():
        want_lat, want_pred = O.emage_generate(sd, cfg, vq, audio, torch.zeros(bs, 1, dtype=torch.long))
    total = mismatched = 0
    for p in PARTS:
        a, b = lat["cls_" + p].argmax(-1).cpu(), want_lat["cls_" + p].argmax(-1)
        total += a.numel()
        mismatched += int((a != b).sum())
    assert mismatched == 0, f"{mismatched}/{total} code indices differ from the oracle"
    ok = _face_ties(vqm, vq, lat, want_lat, "bs32", max_ties=4)
    _pose_checks(pred, want_pred["motion_axis_angle"], want_pred["expression"], want_pred["trans"], "bs32",
                 frames=None if ok.all() else ok, raw=want_pred["_raw"])


@pytest.mark.parametrize("precision,rec_tol,min_agree", [("bf16x6", 1e-3, 0.9995), ("bf16x3", 2e-2, 0.99), ("bf16", 1.0, 0.80),
                                                         ("fp16x3", 1e-3, 0.9995)])
def test_tensor_core_precision_modes(product, ckpt, precision, rec_tol, min_agree):
    """The tensor-core engine end to end (teacher-forced single windows, so a flipped code cannot cascade):
    bf16x6 must meet the fp32 gate; bf16x3 / bf16 report their agreement and must stay above a floor."""
    from pantomatrix_b200.emage_audio import engine
    model, _ = product
    sd, cfg, vq = ckpt
    bs = 4
    audio = torch.from_numpy(synth_audio(bs, 160000, 4321))
    spk = torch.zeros(bs, 1, dtype=torch.long)
    trace = []
    with torch.no_grad():
        O.emage_generate(sd, cfg, vq, audio, spk, trace=trace)
    engine.set_precision(precision)
    try:
        total = same = 0
        worst = 0.0
        for w in trace[:3] + trace[-1:]:
            got = model.forward(w["audio"].cuda(), spk.cuda(), w["motion"].cuda(), w["mask"].cuda())
            for p in PARTS:
                a = got["cls_" + p].argmax(-1).cpu()
                total += a.numel()
                same += int((a == w["idx"][p]).sum())
                worst = max(worst, (got["rec_" + p].cpu() - w["out"]["rec_" + p]).abs().max().item())
    finally:
        engine.set_precision("fp32")
    print(f"\\n[{precision}] index agreement {same}/{total}, max |rec| error {worst:.3e}")
    assert worst < rec_tol, (precision, worst)
    assert same / total >= min_agree, (precision, same, total)


def test_fp16_overflow_is_detected_and_recomputed_in_bf16x6(product):
    """The default fp16x3 engine needs GEMM inputs below 65504 / 64.  Audio 2e4 times louder than the model's range
    drives the first tensor-core conv far beyond that: inference() must notice (NaN reaches the logits, the argmax
    kernels raise the flag), warn, and return what the bf16x6 engine computes - never NaNs or out-of-range codes."""
    from pantomatrix_b200.emage_audio import engine
    model, vqm = product
    audio = (torch.from_numpy(synth_audio(2, 40000, 5)) * 2e4).cuda()
    spk = torch.zeros(2, 1, dtype=torch.long, device="cuda")
    engine.set_precision("bf16x6")
    want = model.inference(audio, spk, vqm)
    assert all(bool(torch.isfinite(v).all()) for v in want.values())
    engine.set_precision("fp16x3")
    try:
        with pytest.warns(UserWarning, match="bf16x6"):
            got = model.inference(audio, spk, vqm)
        assert engine.get_precision() == "fp16x3"                      # the retry does not change the selected mode
    finally:
        engine.set_precision("fp32")
    for k in want:
        assert torch.equal(got[k], want[k]), k


def test_fp16_overflow_raises_in_the_captured_pipeline(product):
    """A replay cannot recompute: audio 2e4 times louder than the model's range makes the fp16x3 graph raise PmError
    naming bf16x6.  Every replay clears the in-graph flag, so the next call on normal audio returns finite outputs."""
    from pantomatrix_b200 import _lib
    from pantomatrix_b200.emage_audio import engine
    from pantomatrix_b200.pipeline import CapturedPipeline
    model, vqm = product
    audio = torch.from_numpy(synth_audio(2, 40000, 5))
    engine.set_precision("fp16x3")
    try:
        cap = CapturedPipeline(model, vqm, 2, 40000)
    finally:
        engine.set_precision("fp32")
    with pytest.raises(_lib.PmError, match="bf16x6"):
        cap((audio * 2e4).cuda())
    lat, pred = cap(audio.cuda())
    for k, v in list(lat.items()) + list(pred.items()):
        assert bool(torch.isfinite(v).all()), k


def test_tokenisation_matches_reference_golden(product, golden_dir):
    """map2index / map2latent / EmageVQVAEConv.forward on the GPU against the real reference's outputs
    (tests/golden/case_tokenise.npz); the CPU twin is tests/test_host_logic.py."""
    _, vqm = product
    g = np.load(os.path.join(golden_dir, "case_tokenise.npz"))
    rot6d, expr = torch.from_numpy(g["rot6d"]).cuda(), torch.from_numpy(g["expression"]).cuda()
    contact, trans = torch.from_numpy(g["tar_contact"]).cuda(), torch.from_numpy(g["tar_trans"]).cuda()
    idx = vqm.map2index(rot6d, expr, tar_contact=contact, tar_trans=trans)
    lat = vqm.map2latent(rot6d, expr, tar_contact=contact, tar_trans=trans)
    parts = vqm.spilt_inputs(rot6d, expr, tar_contact=contact, tar_trans=trans)
    models = dict(face=vqm.vq_model_face, upper=vqm.vq_model_upper, hands=vqm.vq_model_hands, lower=vqm.vq_model_lower)
    for p in PARTS:
        assert np.array_equal(idx[p].cpu().numpy(), g["idx_" + p]), p
        assert np.array_equal(lat[p].cpu().numpy(), g["latent_" + p]), p
        fw = models[p].forward(parts[p])
        np.testing.assert_allclose(fw["rec_pose"].cpu().numpy(), g["rec_pose_" + p], atol=1e-4, rtol=0)
        np.testing.assert_allclose(float(fw["embedding_loss"]), float(g["embedding_loss_" + p]), rtol=1e-4)
        np.testing.assert_allclose(float(fw["perplexity"]), float(g["perplexity_" + p]), rtol=1e-4)
