"""CaMN / DisCo in one CUDA graph (GPU): the LSTM-input assembly kernel and the strided add against torch restatements
bit for bit, the rewritten eager forward() against the composition it replaced (torch.cat / zeros / contiguous around
the same library kernels) bit for bit, and CapturedLstmPipeline replays against eager forward() bit for bit."""
import os
import re

import pytest
import torch

from oracle.weights import LSTM_CFG, load_synthetic, synth_audio

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from pantomatrix_b200 import ops as o
    return o


@pytest.fixture(autouse=True)
def _restore_precision():
    yield
    from pantomatrix_b200.emage_audio import engine
    engine.set_precision(engine.DEFAULT_PRECISION)


def _model(kind, speaker_dims=1, seed=0):
    from pantomatrix_b200.lstm_audio import CamnAudioConfig, CamnAudioModel, DiscoAudioConfig, DiscoAudioModel
    cls, ccls = (CamnAudioModel, CamnAudioConfig) if kind == "camn" else (DiscoAudioModel, DiscoAudioConfig)
    return load_synthetic(cls(ccls(**{**LSTM_CFG, "speaker_dims": speaker_dims})), seed, kind).cuda().eval()


def _same(a, b):
    """Bit-identical (NaN patterns included)."""
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---- kernels --------------------------------------------------------------------------------------------------------


def _cond_reference(spk, ids, seed_motion, t, seed_frames, pose_dims):
    """The parent commit's seed block (torch.zeros + slice assignment + torch.cat) next to the gathered speaker rows."""
    bs = ids.shape[0]
    dims = pose_dims + 1
    if seed_motion is None:
        seed = torch.zeros(bs, t, dims, device="cuda")
        seed[:, :seed_frames, -1] = 1
    else:
        t_m = seed_motion.shape[1]
        seed = torch.zeros(bs, t_m, dims, device="cuda")
        seed[:, :seed_frames, :-1] = seed_motion[:, :seed_frames]
        seed[:, :seed_frames, -1] = 1
        if t_m > t:
            seed = seed[:, :t]
        elif t_m < t:
            seed = torch.cat((seed, seed[:, -(t - t_m):]), 1)
    rows = spk[ids.clamp(0, spk.shape[0] - 1)].unsqueeze(1).expand(bs, t, -1)
    return torch.cat((rows, seed), 2)


@pytest.mark.parametrize("batch", [1, 5, 70])
@pytest.mark.parametrize("t", [7, 10])
@pytest.mark.parametrize("sf", ["0", "4", "t"])
@pytest.mark.parametrize("tm", ["none", "t", "t+7", "t-5", "sf"])
def test_lstm_cond_matches_torch_composition(ops, batch, t, sf, tm):
    from pantomatrix_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(batch * 100 + t)
    pose_dims, spk_f, n_spk = 13, 16, 4
    seed_frames = {"0": 0, "4": 4, "t": t}[sf]
    t_m = None if tm == "none" else {"t": t, "t+7": t + 7, "t-5": t - 5, "sf": seed_frames}[tm]
    spk = torch.randn(n_spk, spk_f, device="cuda", generator=g)
    ids = torch.randint(-1, n_spk + 1, (batch,), device="cuda", generator=g)           # out-of-range ids are clamped
    seed = None if t_m is None else torch.randn(batch, t_m, pose_dims, device="cuda", generator=g)
    cols = spk_f + pose_dims + 1
    # destination: a column range of a wider buffer with odd clip and row strides; everything around it is a sentinel
    buf = torch.full((batch, t + 3, 301), float("nan"), device="cuda")
    out = buf[:, 1:t + 1, 7:7 + cols]
    before = buf.clone()
    seed_len = t if t_m is None else t_m
    if t_m is not None and t > 2 * t_m:
        with pytest.raises(_lib.PmError):                                                # the reference's cat fails too
            ops.lstm_cond(spk, ids, seed, seed_len, seed_frames, pose_dims, out)
        return
    ops.lstm_cond(spk, ids, seed, seed_len, seed_frames, pose_dims, out)
    want = _cond_reference(spk, ids, seed, t, seed_frames, pose_dims)
    assert _same(out, want)
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[:, 1:t + 1, 7:7 + cols] = False
    assert _same(buf[mask], before[mask]), "write outside the destination columns"


def test_lstm_cond_reads_only_the_first_seed_rows(ops):
    """The captured pipeline's form: a seed buffer of seed_frames rows standing for a t-row seed."""
    g = torch.Generator(device="cuda").manual_seed(5)
    t, sf, pd = 12, 4, 9
    spk = torch.randn(2, 16, device="cuda", generator=g)
    ids = torch.tensor([1, 0], device="cuda")
    full = torch.randn(3, t, pd, device="cuda", generator=g)
    out = torch.empty(3, t, 16 + pd + 1, device="cuda")
    ops.lstm_cond(spk, ids.repeat(2)[:3].contiguous(), full[:, :sf].contiguous(), t, sf, pd, out)
    assert _same(out, _cond_reference(spk, ids.repeat(2)[:3], full, t, sf, pd))


@pytest.mark.parametrize("shape,lo,hi", [((3, 17, 1024), 0, 512), ((2, 9, 403), 5, 402), ((70, 3, 36), 1, 35)])
def test_strided_add2_matches_torch(ops, shape, lo, hi):
    """Column ranges read in place (16-byte aligned rows take the vector path, odd offsets the scalar one)."""
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(*shape, device="cuda", generator=g)
    y = torch.randn(*shape, device="cuda", generator=g)
    w = hi - lo
    a, b = x[:, :, lo:lo + w // 2], y[:, :, hi - w // 2:hi]
    got = ops.add2(a, b)
    assert got.is_contiguous() and _same(got, a + b)
    assert _same(ops.add2(x[:, :, lo:lo + w // 2], x[:, :, hi - w // 2:hi]), x[:, :, lo:lo + w // 2] + x[:, :, hi - w // 2:hi])


def test_dense_add2_unchanged(ops):
    g = torch.Generator(device="cuda").manual_seed(8)
    for n in (1, 3, 4, 1021, 4096 * 3 + 2):
        a, b = torch.randn(n, device="cuda", generator=g), torch.randn(n, device="cuda", generator=g)
        assert _same(ops.add2(a, b), a + b)
    a, b = torch.randn(5, 7, 256, device="cuda", generator=g), torch.randn(5, 7, 256, device="cuda", generator=g)
    found = ops.plane_format()
    for fmt in ("bf16", "fp16"):
        ops.set_plane_format(fmt)
        try:
            r = ops.add2(a, b, nsplit=2)
            assert _same(r.f, a + b)
            want = ops.split_bf16(a + b, 2)
            assert torch.equal(r.p.t[..., :256].view(torch.int16), want.t[..., :256].view(torch.int16))
        finally:
            ops.set_plane_format(found)


# ---- eager forward: no behaviour change ---------------------------------------------------------------------------


def _parent_forward(model, audio, speaker_id, seed_frames, seed_motion):
    """The parent commit's forward(): the same library kernels, features joined with torch.cat, the seed block built
    with torch.zeros and slice assignment, the BiLSTM halves copied with .contiguous() before add2."""
    from pantomatrix_b200 import ops
    from pantomatrix_b200.emage_audio import engine as E
    eng = model._eng()

    def bilstm(stack, x):
        for proj, whh in stack.layers:
            x = ops.lstm_bidir(proj(x), whh, stack.barrier, stack.hidden)
        H = stack.hidden
        return ops.add2(x[:, :, :H].contiguous(), x[:, :, H:].contiguous())

    audio = audio.cuda().float().contiguous()
    a = E._f32(eng.wav(audio, 0, 0, 1, audio.shape[1]))
    bs, t, _ = a.shape
    ids = speaker_id.cuda().reshape(-1).contiguous()
    spk = ops.gather_rows(eng.spk, ids).unsqueeze(1).expand(bs, t, -1)
    seed = _cond_reference(eng.spk, ids, seed_motion, t, seed_frames, eng.pose_dims)[:, :, eng.spk.shape[1]:]
    if hasattr(eng, "hands"):
        in_fea = torch.cat((a, spk, seed), dim=2)
        body = eng.body_out(bilstm(eng.body, in_fea))
        hands = eng.hands_out(bilstm(eng.hands, torch.cat((in_fea, body), dim=2)))
        motion = torch.cat((body, hands), dim=2).reshape(bs, t, eng.n_sel, 6)
        return {"motion": motion, "motion_axis_angle": eng.axis_angle(motion.contiguous(), bs, t)}
    a = a.contiguous()
    fea_c = ops.softmax2_mix(eng.selector(a), eng.c1(a), eng.c2(a))
    fea_r = eng.r(a)
    motion = eng.body_out(bilstm(eng.body, torch.cat((fea_c, fea_r, spk, seed), dim=2)))
    return {"motion": motion, "motion_axis_angle": eng.axis_angle(motion, bs, t), "audio_fea_c": fea_c, "audio_fea_r": fea_r}


@pytest.mark.parametrize("precision", ["fp32", "bf16x6", "fp16x3"])
@pytest.mark.parametrize("kind", ["camn", "disco"])
def test_eager_forward_is_bit_identical_to_parent_composition(ops, kind, precision):
    from pantomatrix_b200.emage_audio import engine
    engine.set_precision(precision)
    model = _model(kind, speaker_dims=3)
    bs, n = 5, 48000
    audio = torch.from_numpy(synth_audio(bs, n, 11)).cuda()
    spk = torch.tensor([[2], [0], [1], [2], [1]], device="cuda")
    g = torch.Generator(device="cuda").manual_seed(2)
    from pantomatrix_b200.lstm_audio.modeling import wav_frames
    t = wav_frames(n)
    for seed in (None, 0.3 * torch.randn(bs, t, 258, device="cuda", generator=g),
                 0.3 * torch.randn(bs, t - 9, 258, device="cuda", generator=g)):
        got = model(audio, spk, seed_frames=4, seed_motion=seed)
        want = _parent_forward(model, audio, spk, 4, seed)
        assert set(got) == set(want) | {"motion_axis_angle"}
        for k, v in want.items():
            assert got[k].is_contiguous() and _same(got[k], v), (kind, precision, k)
        assert bool(torch.isfinite(got["motion"]).all())


# ---- captured pipeline --------------------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["camn", "disco"])
@pytest.mark.parametrize("batch", [5, 70])
def test_captured_replay_matches_eager(ops, kind, batch):
    from pantomatrix_b200.lstm_audio.modeling import wav_frames
    from pantomatrix_b200.pipeline import CapturedLstmPipeline
    model = _model(kind, speaker_dims=3)
    n = 32000
    t = wav_frames(n)
    pipe = CapturedLstmPipeline(model, batch, n, seed_frames=4)
    assert pipe.kernels_per_replay > 0
    g = torch.Generator(device="cuda").manual_seed(batch)
    for i in range(2):
        audio = torch.from_numpy(synth_audio(batch, n, 40 + i)).pin_memory()
        spk = torch.randint(0, 3, (batch, 1), device="cuda", generator=g)
        for seeded in (False, True):
            full = 0.3 * torch.randn(batch, t, 258, device="cuda", generator=g) if seeded else None
            got = pipe(audio, spk, None if full is None else full[:, :4].contiguous())
            got = {k: v.clone() for k, v in got.items()}
            want = model(audio.cuda(), spk, seed_frames=4, seed_motion=full)
            assert set(got) == set(want)
            for k in want:
                assert _same(got[k], want[k]), (kind, batch, i, seeded, k)


@pytest.mark.parametrize("kind", ["camn", "disco"])
def test_captured_48k_int16_stereo_matches_eager_on_resampled_audio(ops, kind):
    from pantomatrix_b200.audio_io import Resampler
    from pantomatrix_b200.pipeline import CapturedLstmPipeline
    model = _model(kind)
    batch, n48 = 3, 96000
    pipe = CapturedLstmPipeline(model, batch, n48, input_rate=48000, input_channels=2, input_dtype=torch.int16)
    g = torch.Generator().manual_seed(9)
    for _ in range(2):
        pcm = torch.randint(-20000, 20000, (batch, n48, 2), dtype=torch.int16, generator=g).pin_memory()
        got = {k: v.clone() for k, v in pipe(pcm).items()}
        want = model(Resampler(48000, 16000, device="cuda")(pcm.cuda()), torch.zeros(batch, 1, dtype=torch.long, device="cuda"))
        for k in want:
            assert _same(got[k], want[k]), (kind, k)


@pytest.mark.parametrize("kind", ["camn", "disco"])
def test_captured_graph_holds_library_kernels_only(ops, kind, tmp_path, monkeypatch):
    """Dump the captured graph (cuGraphDebugDotPrint, verbose) and check every kernel node is a library kernel."""
    import ctypes
    from pantomatrix_b200.pipeline import CapturedLstmPipeline

    import functools
    # keep_graph: the graph keeps its cudaGraph_t for inspection (and is instantiated on the first replay)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", functools.partial(torch.cuda.CUDAGraph, keep_graph=True))
    pipe = CapturedLstmPipeline(_model(kind), 70, 16000, input_rate=44100, input_channels=2, input_dtype=torch.int16)
    path = str(tmp_path / f"{kind}.dot")
    rc = ctypes.CDLL("libcuda.so.1").cuGraphDebugDotPrint(ctypes.c_void_p(pipe.graph.raw_cuda_graph()), path.encode(),
                                                          ctypes.c_uint(1))
    assert rc == 0, rc
    dot = open(path).read()
    names = set(re.findall(r"_Z[0-9A-Za-z_]+", dot))
    assert names, "no kernel nodes in the dump"
    foreign = sorted(n for n in names if "pm_" not in n)
    assert not foreign, foreign
    assert any("lstm_bidir_kernel" in n for n in names) and any("resample" in n for n in names)
    # the recurrent kernel's spin barrier needs all its CTAs co-resident: its nodes must keep the cooperative attribute
    lstm_nodes = [blk for blk in dot.split("KERNEL")[1:] if "lstm_bidir_kernel" in blk.split("}")[0]]
    assert len(lstm_nodes) == 2 * 2 * 4 if kind == "camn" else len(lstm_nodes) == 2 * 4      # 70 clips: 2 launches per layer
    assert all("{cooperative | 1}" in blk.split('"]')[0] for blk in lstm_nodes)
    pipe(torch.zeros(70, 16000, 2, dtype=torch.int16, device="cuda"))             # a kept graph still replays


def test_fp16x3_overflow_raises_in_the_captured_pipeline(ops):
    from pantomatrix_b200 import _lib
    from pantomatrix_b200.emage_audio import engine
    from pantomatrix_b200.pipeline import CapturedLstmPipeline
    engine.set_precision("fp16x3")
    model = _model("camn")
    sd = model.state_dict()
    sd["body_out.fc1.weight"] = sd["body_out.fc1.weight"] * 1e5        # hidden activations far past 1023
    model.load_state_dict(sd)
    pipe = CapturedLstmPipeline(model, 2, 16000)
    with pytest.raises(_lib.PmError, match="bf16x6"):
        pipe(torch.from_numpy(synth_audio(2, 16000, 3)).cuda())
