"""CaMN / DisCo captured pipeline, host side (no GPU): argument marshalling of pm_lstm_cond_f32 and pm_add2_f32,
CapturedLstmPipeline's input validation on buffers that live on the CPU (no graph is built), and the captured step's
schedule (kernel_cond) against the eager one (host_cond) with the kernels emulated by tests/fake_ops.py plus a
restatement of pm_lstm_cond_f32."""
import ctypes

import pytest
import torch


@pytest.fixture()
def recorder(monkeypatch):
    """The real ops wrappers on CPU tensors with the library call replaced by a type-checking recorder."""
    from pantomatrix_b200 import _lib, ops
    calls = []

    def record(name, *args):
        sig = _lib.SIGNATURES[name]
        assert len(args) == len(sig), (name, len(args), len(sig))
        for i, (a, t) in enumerate(zip(args, sig)):
            if t is ctypes.c_void_p:
                assert a is None or isinstance(a, int), (name, i, type(a))
            else:
                assert isinstance(a, int) and not isinstance(a, bool), (name, i, type(a))
                t(a)
        calls.append((name, args))

    monkeypatch.setattr(_lib, "call", record)
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=torch.float32: t)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    return ops, calls


def test_add2_marshals_row_strides_and_the_dense_geometry(recorder):
    ops, calls = recorder
    y = torch.zeros(3, 5, 1024)
    out = ops.add2(y[:, :, :512], y[:, :, 512:])
    name, args = calls[-1]
    assert name == "pm_add2_f32" and out.shape == (3, 5, 512) and out.is_contiguous()
    assert args[1] == 1024 and args[2] == y.data_ptr() + 512 * 4 and args[3] == 1024 and args[5] == 512
    assert args[6] == 15 and args[7] == 512 and args[8] is None
    # dense operands: one row of n elements (16-byte access whatever ch is), or n / ch rows of ch with planes
    ops.add2(torch.zeros(3, 5, 61), torch.zeros(3, 5, 61))
    name, args = calls[-1]
    assert name == "pm_add2_f32" and (args[1], args[3], args[5]) == (915,) * 3 and args[6:8] == (1, 915)
    assert args[8] is None
    ops.add2(torch.zeros(3, 5, 64), torch.zeros(3, 5, 64), nsplit=2)
    name, args = calls[-1]
    assert name == "pm_add2_f32" and (args[1], args[3], args[5]) == (64,) * 3 and args[6:8] == (15, 64)
    assert args[8] is not None and args[11] & 0xff == 2
    with pytest.raises(Exception):                        # clip rows not evenly spaced: no single row stride
        ops.add2(torch.zeros(3, 6, 8)[:, :5], torch.zeros(3, 6, 8)[:, :5])


def test_lstm_cond_marshals_views(recorder):
    ops, calls = recorder
    spk, ids = torch.zeros(3, 16), torch.zeros(4, 1, dtype=torch.int64)
    buf = torch.zeros(4, 9, 484)
    seed = torch.zeros(4, 2, 258)
    ops.lstm_cond(spk, ids, seed, 9, 2, 258, buf[:, :, 128:403])
    name, a = calls[-1]
    assert name == "pm_lstm_cond_f32"
    assert a[1:3] == (3, 16) and a[5:10] == (2 * 258, 258, 9, 2, 258)
    assert a[10] == buf.data_ptr() + 128 * 4 and a[11:16] == (9 * 484, 484, 4, 9, 0)
    ops.lstm_cond(spk, ids, torch.zeros(4, 0, 258), 9, 0, 258, buf[:, :, 128:403])
    assert calls[-1][1][4] is None                          # an empty seed is no seed
    with pytest.raises(AssertionError):
        ops.lstm_cond(spk, ids, seed, 9, 2, 258, buf[:, :, 128:400])


def test_wav_frames_matches_the_encoder_geometry():
    from pantomatrix_b200.lstm_audio.modeling import wav_frames
    assert wav_frames(160000) == 149 and wav_frames(16000) == 15


def _cpu_pipeline(recorded=False):
    """A CapturedLstmPipeline whose static buffers live on the CPU, for the host-side checks of __call__."""
    from pantomatrix_b200.pipeline import CapturedLstmPipeline
    p = CapturedLstmPipeline.__new__(CapturedLstmPipeline)
    p.batch, p.seed_frames, p.speaker_dims, p.pose_dims = 2, 4, 3, 258
    p.audio = torch.zeros(2, 16000)
    p.pcm = torch.zeros(2, 48000, 2, dtype=torch.int16) if recorded else None
    p.speaker_id = torch.zeros(2, 1, dtype=torch.long)
    p.seed = torch.zeros(2, 4, 258)
    return p


def test_pipeline_stages_valid_inputs():
    p = _cpu_pipeline()
    seed = torch.randn(2, 4, 258)
    p._stage_inputs(torch.ones(2, 16000), torch.tensor([[2], [1]]), seed)
    assert torch.equal(p.audio, torch.ones(2, 16000)) and p.speaker_id.flatten().tolist() == [2, 1]
    assert torch.equal(p.seed, seed)


@pytest.mark.parametrize("case", ["id_high", "id_negative", "id_shape", "id_dtype", "seed_shape", "seed_dtype", "seed_rows"])
def test_pipeline_rejects_bad_speaker_and_seed(case):
    p = _cpu_pipeline()
    ids, seed = torch.tensor([[0], [1]]), None
    if case == "id_high":
        ids = torch.tensor([[0], [3]])
    elif case == "id_negative":
        ids = torch.tensor([[-1], [0]])
    elif case == "id_shape":
        ids = torch.tensor([0, 1])
    elif case == "id_dtype":
        ids = torch.tensor([[0], [1]], dtype=torch.int32)
    elif case == "seed_shape":
        seed = torch.zeros(2, 4, 257)
    elif case == "seed_dtype":
        seed = torch.zeros(2, 4, 258, dtype=torch.float64)
    else:
        seed = torch.zeros(2, 5, 258)
    with pytest.raises(ValueError):
        p._stage_inputs(torch.zeros(2, 16000), ids, seed)


@pytest.mark.parametrize("pcm", [torch.zeros(2, 48000, 2, dtype=torch.float32), torch.zeros(2, 48000, 1, dtype=torch.int16),
                                 torch.zeros(2, 47999, 2, dtype=torch.int16), torch.zeros(2, 48000, 2, dtype=torch.int16),
                                 "not a tensor"])
def test_pipeline_rejects_recorded_audio_of_the_wrong_form(pcm):
    """Wrong dtype, channel count or length, pageable host memory (the last tensor), not a tensor."""
    p = _cpu_pipeline(recorded=True)
    with pytest.raises(ValueError):
        p._stage_inputs(pcm, torch.tensor([[0], [1]]), torch.zeros(2, 4, 258))


def _lstm_cond_restated(spk, speaker_id, seed, seed_len, seed_frames, pose_dims, out):
    """pm_lstm_cond_f32 (include/pm_emage.h) in torch, for the host-schedule test below."""
    t = out.shape[1]
    ids = speaker_id.reshape(-1).clamp(0, spk.shape[0] - 1)
    out[:, :, :spk.shape[1]] = spk[ids][:, None]
    c = out[:, :, spk.shape[1]:]
    c.zero_()
    for r in range(t):
        j = r if r < seed_len else r - (t - seed_len)
        if j < min(seed_frames, seed_len):
            c[:, r, -1] = 1
            if seed is not None and seed.numel():
                c[:, r, :-1] = seed[:, j]
    return out


@pytest.fixture()
def emulated(monkeypatch, request):
    """The product's host schedule on the CPU: every kernel wrapper replaced by tests/fake_ops.py, and lstm_cond by
    the restatement above; exact fp32 engine."""
    import fake_ops
    import pantomatrix_b200.ops as real
    from pantomatrix_b200.emage_audio import modeling
    from helpers import use_precision
    for name in dir(fake_ops):
        if not name.startswith("_") and callable(getattr(fake_ops, name)) and hasattr(real, name):
            monkeypatch.setattr(real, name, getattr(fake_ops, name))
    monkeypatch.setattr(real, "lstm_cond", _lstm_cond_restated)
    monkeypatch.setattr(modeling, "_require_cuda", lambda module, what: torch.device("cpu"))
    use_precision(request, "fp32")


@pytest.mark.parametrize("kind", ["camn", "disco"])
def test_captured_schedule_matches_eager_forward_on_emulated_kernels(emulated, kind):
    """What the captured step runs (engine.forward with kernel_cond over the pipeline's static buffers: speaker ids,
    the first seed_frames seed rows standing for a t-row seed) equals forward() with the full seed, or with none."""
    from helpers import build_lstm_product
    from oracle.weights import synth_audio
    from pantomatrix_b200.lstm_audio.modeling import wav_frames
    model = build_lstm_product(kind, device="cpu")
    eng = model._eng()
    bs, n = 2, 16000
    t = wav_frames(n)
    audio = torch.from_numpy(synth_audio(bs, n, 21))
    ids = torch.tensor([[0], [0]])
    full = 0.3 * torch.randn(bs, t, 258, generator=torch.Generator().manual_seed(3))
    for seed, static in ((full, full[:, :4].contiguous()), (None, torch.zeros(bs, 4, 258))):
        want = model(audio, ids, seed_frames=4, seed_motion=seed)
        got = eng.forward(audio, eng.kernel_cond(ids, static, t, 4), True)
        assert set(got) == set(want)
        for k in want:
            assert torch.equal(got[k], want[k]), (kind, seed is None, k)
