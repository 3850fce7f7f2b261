"""Audio front-end on the host side: the resampler's filter design and packing against scipy, the WAV reader's raw
PCM path, and the marshalling of ops.resample_poly (no GPU needed)."""
import ctypes
import os
import struct
import wave

import numpy as np
import pytest
import torch

from pantomatrix_b200 import audio_io
from resample_ref import mix_down, polyphase_sum

RATES = (8000, 11025, 12000, 22050, 24000, 32000, 44056, 44100, 48000, 88200, 96000, 192000)


@pytest.mark.parametrize("rate", RATES)
def test_filter_design_is_bit_identical_to_scipy(rate):
    signal = pytest.importorskip("scipy.signal")
    up, down = audio_io.resample_ratio(rate, 16000)
    h, half_len = audio_io.design_filter(up, down)
    want = signal.firwin(2 * half_len + 1, 1.0 / max(up, down), window=("kaiser", 5.0)).astype(np.float32)
    want *= np.float32(up)
    assert h.dtype == np.float32 and np.array_equal(h.view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("rate", RATES + (16000, 16001))
def test_polyphase_sum_equals_resample_poly(rate):
    """The packed bank, n_pre_remove and n_out, read with the kernel's indexing, give resample_poly's output."""
    signal = pytest.importorskip("scipy.signal")
    up, down = audio_io.resample_ratio(rate, 16000)
    bank, n_pre_remove = audio_io.polyphase_bank(up, down, np.float64)
    assert bank.shape[0] == up and bank.flags.c_contiguous
    half_len = 10 * max(up, down)
    rng = np.random.default_rng(rate)
    for n_in in sorted({1, 2, 5, 17, 100, 1001, half_len // 7 + 1, half_len - 1, half_len + 3, 3 * half_len + 11}):
        x = rng.standard_normal(n_in)
        y, _, _ = polyphase_sum(x, bank, up, down, n_pre_remove)
        want = signal.resample_poly(x, up, down)
        assert y.shape == want.shape == (-(-n_in * up // down),), (n_in, y.shape, want.shape)
        assert np.abs(y - want).max() <= 1e-12, (n_in, np.abs(y - want).max())


def test_float32_bank_holds_the_float32_taps():
    up, down = audio_io.resample_ratio(44100, 16000)
    bank, _ = audio_io.polyphase_bank(up, down)
    h, half_len = audio_io.design_filter(up, down)
    pad = down - half_len % down
    flat = bank.T.reshape(-1)                               # phase-major -> tap order k = p + up*j
    assert bank.dtype == np.float32
    assert np.array_equal(flat[:pad], np.zeros(pad, np.float32)) and np.array_equal(flat[pad:pad + h.size], h)
    assert not flat[pad + h.size:].any()
    ident, n_pre_remove = audio_io.polyphase_bank(1, 1)
    assert ident.shape == (1, 1) and ident[0, 0] == 1.0 and n_pre_remove == 0


def test_golden_resample_fixture_is_within_the_fp32_bound(golden_dir):
    """scipy's float32 outputs in the fixture lie within (taps + 1) * 2^-24 * sum|h||x| of the float64 sum over the
    float32 taps: the GPU tests compare against them with twice that bound."""
    g = np.load(os.path.join(golden_dir, "resample.npz"))
    cases = sorted(k[:-4] for k in g.files if k.endswith("_pcm"))
    assert len(cases) == 4
    for c in cases:
        up, down = audio_io.resample_ratio(int(g[c + "_rate"]), 16000)
        bank, n_pre_remove = audio_io.polyphase_bank(up, down)
        for pcm, out in zip(g[c + "_pcm"], g[c + "_out"]):
            y, mag, taps = polyphase_sum(mix_down(pcm), bank, up, down, n_pre_remove)
            assert out.shape == y.shape
            assert (np.abs(out - y) <= (taps + 1) * 2.0 ** -24 * mag).all(), c


def _write_wav(path, rate, frames, fmt_tag, bits):
    data = frames.tobytes()
    ch = frames.shape[1]
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVEfmt "
                + struct.pack("<IHHIIHH", 16, fmt_tag, ch, rate, rate * ch * bits // 8, ch * bits // 8, bits)
                + b"data" + struct.pack("<I", len(data)) + data)


def _legacy_read(frames, bits, tag):
    """What the WAV reader has always returned for these frames (float32, [-1, 1])."""
    if tag == 3:
        return frames.astype(np.float32)
    if bits == 8:
        return (frames.astype(np.float32) - 128.0) / 128.0
    if bits == 16:
        return frames.astype(np.float32) / 32768.0
    if bits == 24:
        return frames.astype(np.float32) / float(1 << 23)
    return frames.astype(np.float32) / float(1 << 31)


@pytest.mark.parametrize("bits,tag", [(8, 1), (16, 1), (24, 1), (32, 1), (32, 3), (64, 3)])
def test_read_pcm_and_load_audio_unchanged(tmp_path, bits, tag):
    rng = np.random.default_rng(bits + tag)
    n, ch, rate = 997, 3, 22050
    if tag == 3:
        frames = rng.uniform(-1, 1, (n, ch)).astype("<f4" if bits == 32 else "<f8")
        raw = frames
    elif bits == 8:
        frames = rng.integers(0, 256, (n, ch)).astype(np.uint8)
        raw = frames
    elif bits == 24:
        frames = rng.integers(-(1 << 23), 1 << 23, (n, ch)).astype(np.int32)
        b = frames.astype("<i4").view(np.uint8).reshape(n, ch, 4)[:, :, :3]
        raw = np.ascontiguousarray(b)
    else:
        dt = "<i2" if bits == 16 else "<i4"
        frames = rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, (n, ch), endpoint=True).astype(dt)
        raw = frames
    path = str(tmp_path / "x.wav")
    _write_wav(path, rate, raw, tag, bits)
    want = _legacy_read(frames, bits, tag)
    pcm, r = audio_io.read_pcm(path)
    assert r == rate and pcm.shape == (n, ch)
    if bits == 16 and tag == 1:
        assert pcm.dtype == np.int16 and np.array_equal(pcm, frames)
    else:
        assert pcm.dtype == np.float32 and np.array_equal(pcm, want)
    x, r = audio_io._read_wav(path)
    assert r == rate and x.dtype == np.float32 and np.array_equal(x.view(np.int32), want.view(np.int32))
    mono = audio_io.load_audio(path, sr=rate)
    assert np.array_equal(mono.view(np.int32), want.mean(axis=1).astype(np.float32).view(np.int32))
    assert np.array_equal(mono.view(np.int32), mix_down(pcm).view(np.int32))
    signal = pytest.importorskip("scipy.signal")
    got = audio_io.load_audio(path)
    ref = signal.resample_poly(want.mean(axis=1).astype(np.float32), 320, 441).astype(np.float32)
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))


def test_read_pcm_keeps_16_bit_stereo_as_int16(tmp_path):
    frames = np.array([[0, -1], [32767, -32768], [123, -456]], dtype="<i2")
    path = str(tmp_path / "s.wav")
    with wave.open(path, "wb") as w:
        w.setnchannels(2), w.setsampwidth(2), w.setframerate(48000)
        w.writeframes(frames.tobytes())
    pcm, rate = audio_io.read_pcm(path)
    assert rate == 48000 and pcm.dtype == np.int16 and np.array_equal(pcm, frames)
    assert np.array_equal(audio_io.load_audio(path, sr=48000), (frames / 32768.0).astype(np.float32).mean(1))


def test_mix_down_of_negative_zeros_is_positive_zero():
    for ch in range(1, 9):
        y = mix_down(-np.zeros((4, ch), np.float32))
        assert not np.signbit(y).any(), ch


def test_resample_poly_marshals_valid_arguments(monkeypatch):
    """ops.resample_poly on CPU tensors with the library call replaced by a recorder: every argument converts to the
    ctypes type its binding declares, strides are in elements, an `out` view keeps its clip stride."""
    from pantomatrix_b200 import _lib, ops
    calls = []

    def record(name, *args):
        sig = _lib.SIGNATURES[name]
        assert len(args) == len(sig), (name, len(args), len(sig))
        for i, (a, t) in enumerate(zip(args, sig)):
            if t is ctypes.c_void_p:
                assert a is None or isinstance(a, int), (name, i, type(a))
            elif t is ctypes.c_float:
                assert isinstance(a, float), (name, i, type(a))
            else:
                assert isinstance(a, int) and not isinstance(a, bool), (name, i, type(a))
                t(a)
        calls.append((name, args))

    monkeypatch.setattr(_lib, "call", record)
    monkeypatch.setattr(ops, "_chk", lambda t, dtype=torch.float32: t)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    up, down = audio_io.resample_ratio(48000, 16000)
    bank, n_pre_remove = audio_io.polyphase_bank(up, down)
    bank = torch.from_numpy(bank)
    pcm = torch.zeros(3, 4801, 2, dtype=torch.int16)
    out = ops.resample_poly(pcm, bank, up, down, n_pre_remove)
    assert out.shape == (3, 1601) and out.dtype == torch.float32
    wide = torch.zeros(3, 2000)
    view = ops.resample_poly(pcm.float(), bank, up, down, n_pre_remove, out=wide[:, 7:1608])
    assert view.data_ptr() == wide[:, 7:].data_ptr()
    (n1, a1), (n2, a2) = calls
    assert n1 == n2 == "pm_resample_poly_f32"
    assert a1[1:6] == (1, 4801 * 2, 3, 4801, 2) and a2[1] == 0
    assert a1[7:11] == (up, down, bank.shape[1], n_pre_remove) and a1[12] == 1601 and a2[12] == 2000
    with pytest.raises(_lib.PmError):
        ops.resample_poly(pcm.to(torch.int32), bank, up, down, n_pre_remove)
    with pytest.raises(_lib.PmError):
        ops.resample_poly(pcm, bank, up, down, n_pre_remove, out=torch.zeros(3, 1600))
    with pytest.raises(_lib.PmError):
        ops.resample_poly(pcm[:, ::2], bank, up, down, n_pre_remove)
