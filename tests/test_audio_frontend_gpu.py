"""The audio front-end kernel (pm_resample_poly_f32) and CapturedPipeline on the GPU.

Every resampled element is held to its own bound: |y - y64| <= (n_m + 1) * 2^-24 * sum_k |h_k| |x_k|, y64 the float64
sum over the same float32 taps and float32 mixed samples, n_m the taps output m visits (an fp32 FMA chain).  The scipy
fixture (tests/golden/resample.npz) is matched within twice that.  Conversion, mix-down, indexing and layout are exact."""
import os
import struct
import wave

import numpy as np
import pytest
import torch

from helpers import build_product
from resample_ref import mix_down, polyphase_sum
from pantomatrix_b200 import _lib, audio_io
from pantomatrix_b200.pipeline import CapturedPipeline, generate

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _pcm(rng, batch, n, ch, dtype):
    if dtype == torch.int16:
        return rng.integers(-32768, 32767, (batch, n, ch), endpoint=True).astype(np.int16)
    return (rng.standard_normal((batch, n, ch)) * np.exp(rng.uniform(-3, 1, (batch, n, ch)))).astype(np.float32)


def _check_bound(got, pcm, rs, factor=1.0, want=None):
    """Per-element bound against the float64 sum (or, with `want`, against a float32 result held to the same sum)."""
    bank = rs.bank.cpu().numpy()
    for b in range(pcm.shape[0]):
        y64, mag, taps = polyphase_sum(mix_down(pcm[b]), bank, rs.up, rs.down, rs.n_pre_remove)
        ref = y64 if want is None else want[b].astype(np.float64)
        err = np.abs(got[b].astype(np.float64) - ref)
        bound = factor * (taps + 1) * U * mag
        bad = np.nonzero(err > bound)[0]
        assert bad.size == 0, (b, bad[:5], err[bad[:5]], bound[bad[:5]])


@pytest.mark.parametrize("dtype", [torch.int16, torch.float32], ids=["i16", "f32"])
@pytest.mark.parametrize("ch", [1, 2])
@pytest.mark.parametrize("rate", [8000, 11025, 22050, 24000, 32000, 44056, 44100, 48000, 96000])
def test_resample_per_element_bound(rate, ch, dtype):
    rng = np.random.default_rng(rate * 10 + ch)
    rs = audio_io.Resampler(rate, 16000, device="cuda")
    n = 2 * (rate // 10) + 1 + 2 * ch                      # 0.2 s, odd
    pcm = _pcm(rng, 3, n, ch, dtype)
    got = rs(torch.from_numpy(pcm).cuda())
    torch.cuda.synchronize()
    assert got.shape == (3, rs.n_out(n)) and got.dtype == torch.float32
    _check_bound(got.cpu().numpy(), pcm, rs)


def test_resample_matches_scipy_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "resample.npz"))
    cases = sorted(k[:-4] for k in g.files if k.endswith("_pcm"))
    assert len(cases) == 4
    for c in cases:
        pcm = g[c + "_pcm"]
        rs = audio_io.Resampler(int(g[c + "_rate"]), 16000, device="cuda")
        got = rs(torch.from_numpy(pcm).cuda()).cpu().numpy()
        assert got.shape == g[c + "_out"].shape, c
        _check_bound(got, pcm, rs, factor=2.0, want=g[c + "_out"])


@pytest.mark.parametrize("rate", [8000, 22050, 44056, 44100, 48000, 96000])
@pytest.mark.parametrize("dtype", [torch.int16, torch.float32], ids=["i16", "f32"])
def test_resample_impulse_is_exact(rate, dtype):
    """0.5 at the first, an interior and the last sample: each output has at most one nonzero product, so it is exactly
    0.5 * h'[k] at the right place and 0 elsewhere."""
    rs = audio_io.Resampler(rate, 16000, device="cuda")
    bank = rs.bank.cpu().numpy()
    n = rate // 5 + 7
    for pos in (0, n // 2 + 3, n - 1):
        pcm = np.zeros((1, n, 1), np.int16 if dtype == torch.int16 else np.float32)
        pcm[0, pos, 0] = 16384 if dtype == torch.int16 else 0.5
        got = rs(torch.from_numpy(pcm).cuda()).cpu().numpy()[0]
        y64, _, _ = polyphase_sum(mix_down(pcm[0]), bank, rs.up, rs.down, rs.n_pre_remove)
        want = y64.astype(np.float32)
        assert np.array_equal(got, want), (pos, np.nonzero(got != want)[0][:5])
        assert np.count_nonzero(want) > 0


@pytest.mark.parametrize("ch", [1, 2, 3, 8])
@pytest.mark.parametrize("dtype", [torch.int16, torch.float32], ids=["i16", "f32"])
def test_convert_and_mix_down_equal_host_load_audio(tmp_path, ch, dtype):
    """16 kHz in and out: the kernel is the pure conversion and mix-down, bit for bit the host reader's."""
    rng = np.random.default_rng(ch)
    n = 4099
    pcm = _pcm(rng, 1, n, ch, dtype)[0]
    if dtype == torch.float32:
        pcm[::7] = -0.0                                    # all-negative-zero rows mix to +0, as on the host
        pcm[1::11] = rng.uniform(-1e-39, 1e-39, (pcm[1::11].shape)).astype(np.float32)
    path = str(tmp_path / "a.wav")
    if dtype == torch.int16:
        with wave.open(path, "wb") as w:
            w.setnchannels(ch), w.setsampwidth(2), w.setframerate(16000)
            w.writeframes(pcm.astype("<i2").tobytes())
    else:
        data = pcm.astype("<f4").tobytes()
        with open(path, "wb") as f:
            f.write(b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVEfmt "
                    + struct.pack("<IHHIIHH", 16, 3, ch, 16000, 16000 * ch * 4, ch * 4, 32)
                    + b"data" + struct.pack("<I", len(data)) + data)
    host = audio_io.load_audio(path, sr=16000)
    dev = audio_io.load_audio(path, sr=16000, device="cuda")
    assert dev.is_cuda and dev.dtype == torch.float32 and dev.shape == (n,)
    got = dev.cpu().numpy()
    assert np.array_equal(got.view(np.int32), host.view(np.int32)), np.nonzero(got.view(np.int32) != host.view(np.int32))[0][:5]


def test_resample_layout():
    rng = np.random.default_rng(5)
    rs = audio_io.Resampler(44100, 16000, device="cuda")
    n = 12347
    pcm = torch.from_numpy(_pcm(rng, 5, n, 2, torch.int16)).cuda()
    batch = rs(pcm)
    for b in range(5):                                     # a clip alone == the same clip inside the batch
        assert torch.equal(rs(pcm[b:b + 1].contiguous()), batch[b:b + 1]), b
    n_out = rs.n_out(n)
    wide = torch.full((5, n_out + 37), 7.25, device="cuda")
    view = wide[:, 11:11 + n_out]
    assert rs(pcm, out=view).data_ptr() == view.data_ptr()
    assert torch.equal(view, batch)
    assert bool((wide[:, :11] == 7.25).all()) and bool((wide[:, 11 + n_out:] == 7.25).all())
    pcm_wide = torch.from_numpy(_pcm(rng, 3, n + 100, 2, torch.int16)).cuda()      # clip stride > n_in * channels
    assert torch.equal(rs(pcm_wide[:, 50:50 + n])[1], rs(pcm_wide[1:2, 50:50 + n].contiguous())[0])
    big = torch.from_numpy(_pcm(rng, 64, 4801, 1, torch.float32)).cuda()
    rs48 = audio_io.Resampler(48000, 16000, device="cuda")
    y = rs48(big)
    assert y.shape == (64, 1601)
    assert torch.equal(y[63], rs48(big[63:64])[0]) and torch.equal(y[0], rs48(big[0:1])[0])
    empty = rs48(torch.zeros(2, 0, 1, device="cuda"))
    torch.cuda.synchronize()
    assert empty.shape == (2, 0)
    with pytest.raises(_lib.PmError):                      # more than 8 channels
        rs48(torch.zeros(1, 10, 9, device="cuda"))


def test_resample_unstaged_path_for_large_ratios():
    """A reduced ratio whose tile span cannot fit shared memory even for one row: the kernel reads and mixes the input
    straight from global memory, under the same per-element bound."""
    rng = np.random.default_rng(9)
    rs = audio_io.Resampler(96001, 16000, device="cuda")     # down = 96001: read from global memory, not staged
    assert rs.down > 16384
    pcm = _pcm(rng, 2, 3001, 2, torch.int16)
    got = rs(torch.from_numpy(pcm).cuda()).cpu().numpy()
    _check_bound(got, pcm, rs)


# ---- CapturedPipeline -----------------------------------------------------------------------------------------------

BATCH, N16 = 2, 70000                                      # 131 frames: 2 full windows + a short tail


@pytest.fixture(scope="module")
def product():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return build_product(seed=0)


@pytest.fixture(scope="module")
def default_pipeline(product):
    return CapturedPipeline(*product, BATCH, N16)


def _equal_dicts(a, b):
    assert set(a) == set(b)
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), k


def test_captured_pipeline_defaults_equal_generate(product, default_pipeline):
    model, vqm = product
    cap = default_pipeline
    assert cap.pcm is None and cap.audio.shape == (BATCH, N16) and cap.audio.dtype == torch.float32
    rng = np.random.default_rng(3)
    for _ in range(2):
        audio = torch.from_numpy(rng.uniform(-0.1, 0.1, (BATCH, N16)).astype(np.float32))
        lat, pred = cap(audio.pin_memory())
        torch.cuda.synchronize()
        lat, pred = {k: v.clone() for k, v in lat.items()}, {k: v.clone() if torch.is_tensor(v) else v for k, v in pred.items()}
        want_lat, want_pred = generate(model, vqm, audio.cuda())
        torch.cuda.synchronize()
        _equal_dicts(lat, want_lat)
        _equal_dicts(pred, want_pred)


def test_captured_pipeline_from_48k_int16_stereo(product, default_pipeline):
    model, vqm = product
    cap = CapturedPipeline(model, vqm, BATCH, 3 * N16, input_rate=48000, input_channels=2, input_dtype=torch.int16)
    assert cap.pcm.shape == (BATCH, 3 * N16, 2) and cap.pcm.dtype == torch.int16 and cap.audio.shape == (BATCH, N16)
    assert cap.kernels_per_replay == default_pipeline.kernels_per_replay + 1
    rng = np.random.default_rng(4)
    for _ in range(2):
        t = np.arange(3 * N16) / 48000.0
        pcm = torch.from_numpy(np.clip(np.rint(3000 * np.sin(2 * np.pi * 180 * t)[None, :, None]
                                               + rng.normal(0, 2000, (BATCH, 3 * N16, 2))), -32768, 32767).astype(np.int16))
        lat, pred = cap(pcm.pin_memory())
        torch.cuda.synchronize()
        audio16 = cap.audio.clone()
        lat, pred = {k: v.clone() for k, v in lat.items()}, {k: v.clone() if torch.is_tensor(v) else v for k, v in pred.items()}
        want16 = audio_io.Resampler(48000, device="cuda")(pcm.cuda())
        assert torch.equal(audio16, want16)
        want_lat, want_pred = generate(model, vqm, want16)
        torch.cuda.synchronize()
        _equal_dicts(lat, want_lat)
        _equal_dicts(pred, want_pred)
    for bad in (pcm.float().pin_memory(), pcm[:, :-1].contiguous().pin_memory(), pcm, pcm[:, :, :1].contiguous()):
        with pytest.raises(ValueError):                    # wrong dtype, wrong shape, pageable host memory, one channel
            cap(bad)


def test_load_audio_on_the_gpu_from_a_44k_stereo_wav(tmp_path):
    rng = np.random.default_rng(11)
    n = 44100 // 2 + 13
    t = np.arange(n) / 44100.0
    frames = np.clip(np.rint(np.stack([9000 * np.sin(2 * np.pi * 440 * t), 5000 * np.sin(2 * np.pi * 97 * t)], 1)
                             + rng.normal(0, 500, (n, 2))), -32768, 32767).astype("<i2")
    path = str(tmp_path / "s.wav")
    with wave.open(path, "wb") as w:
        w.setnchannels(2), w.setsampwidth(2), w.setframerate(44100)
        w.writeframes(frames.tobytes())
    got = audio_io.load_audio(path, sr=16000, device="cuda")
    rs = audio_io.Resampler(44100, 16000, device="cuda")
    assert got.is_cuda and got.shape == (rs.n_out(n),)
    host_mono = audio_io.load_audio(path, sr=44100)       # the host reader's mono signal at the file's rate
    y64, mag, taps = polyphase_sum(host_mono, rs.bank.cpu().numpy(), rs.up, rs.down, rs.n_pre_remove)
    err = np.abs(got.cpu().numpy().astype(np.float64) - y64)
    assert (err <= (taps + 1) * U * mag).all()
