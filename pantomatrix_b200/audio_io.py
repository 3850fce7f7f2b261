"""Audio front-end of the EMAGE path: the step right before the hot path (SURVEY.md section 8f-4).

The reference calls `librosa.load(path, sr=16000)` (test_emage_audio.py:17): decode, mix down to mono, resample
to 16 kHz float32 in [-1, 1].  librosa / soundfile / ffmpeg are not available offline, so this is a small
stand-alone reader for PCM / IEEE-float WAV files with a polyphase resampler (scipy).  It is not sample-identical
to librosa's default `soxr_hq` resampler; files already at 16 kHz are returned exactly as librosa would.

On the GPU, `Resampler` (kernel pm_resample_poly_f32) does the conversion, mix-down and resampling in one launch from
the samples as the file stores them (16-bit PCM stays int16: half the bytes of float32 cross PCIe).  It computes
scipy.signal.resample_poly's sum with the same float32 taps, in fp32 FMA; `load_audio(path, device="cuda")` uses it.
"""
from __future__ import annotations

import functools
import struct
from fractions import Fraction

import numpy as np


def read_pcm(path):
    """(samples (n, channels), rate) of a PCM / IEEE-float WAV file.  16-bit PCM stays np.int16 (the raw samples);
    every other format is converted to float32 in [-1, 1]."""
    with open(path, "rb") as f:
        head = f.read(12)
        if len(head) < 12 or head[:4] != b"RIFF" or head[8:12] != b"WAVE":
            raise ValueError(f"{path}: not a RIFF/WAVE file (compressed formats such as MP3 need an external decoder)")
        fmt = data = None
        while True:
            chunk = f.read(8)
            if len(chunk) < 8:
                break
            cid, size = chunk[:4], struct.unpack("<I", chunk[4:])[0]
            body = f.read(size + (size & 1))
            if cid == b"fmt ":
                fmt = body[:size]
            elif cid == b"data":
                data = body[:size]
        if fmt is None or data is None:
            raise ValueError(f"{path}: missing fmt or data chunk")
    tag, channels, rate, _, _, bits = struct.unpack("<HHIIHH", fmt[:16])
    if tag == 0xFFFE and len(fmt) >= 26:                     # WAVE_FORMAT_EXTENSIBLE: real tag in the sub-format GUID
        tag = struct.unpack("<H", fmt[24:26])[0]
    if tag == 1:                                             # integer PCM
        if bits == 8:
            x = (np.frombuffer(data, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
        elif bits == 16:
            x = np.frombuffer(data, dtype="<i2").astype(np.int16)
        elif bits == 24:
            b = np.frombuffer(data, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
            v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
            x = (np.where(v >= 1 << 23, v - (1 << 24), v)).astype(np.float32) / float(1 << 23)
        elif bits == 32:
            x = np.frombuffer(data, dtype="<i4").astype(np.float32) / float(1 << 31)
        else:
            raise ValueError(f"{path}: unsupported PCM width {bits}")
    elif tag == 3:                                           # IEEE float
        x = np.frombuffer(data, dtype="<f4" if bits == 32 else "<f8").astype(np.float32)
    else:
        raise ValueError(f"{path}: unsupported WAV format tag {tag}")
    return x.reshape(-1, channels), rate


def track_samples(x):
    """FLAC track samples (pantomatrix_b200/flac.py) of read_pcm's output: 16-bit PCM stays int16 (coded at 16 bits);
    every other format becomes int32 coded at 24 bits, clamp(round-half-even(x 2^23)) to -2^23 .. 2^23 - 1, which is
    exact for 8- and 24-bit sources."""
    if x.dtype == np.int16:
        return x
    v = np.rint(x.astype(np.float64) * float(1 << 23))
    return np.clip(v, -(1 << 23), (1 << 23) - 1).astype(np.int32)


def read_track(path, device):
    """(samples on device, rate) of a WAV file for video.write_mp4's audio track: read_pcm, then track_samples."""
    import torch
    pcm, rate = read_pcm(path)
    return torch.from_numpy(np.ascontiguousarray(track_samples(pcm))).to(device), rate


def _read_wav(path):
    """(float32 samples (n, channels) in [-1, 1], rate)."""
    x, rate = read_pcm(path)
    if x.dtype == np.int16:
        x = x.astype(np.float32) / 32768.0
    return x, rate


def load_audio(path, sr: int = 16000, device=None):
    """Mono float32 waveform at `sr` Hz: a NumPy array, or with a CUDA `device` a 1-D CUDA tensor made from the raw
    samples by the resampling kernel (same taps as the host path, fp32 FMA accumulation)."""
    if device is not None:
        import torch
        pcm, rate = read_pcm(path)
        x = torch.from_numpy(np.ascontiguousarray(pcm)).to(device)
        return Resampler(rate, sr, device=device)(x[None])[0]
    x, rate = _read_wav(path)
    mono = x.mean(axis=1).astype(np.float32)
    if rate != sr:
        from scipy.signal import resample_poly
        ratio = Fraction(sr, rate)
        mono = resample_poly(mono, ratio.numerator, ratio.denominator).astype(np.float32)
    return mono


def resample_ratio(rate_in: int, rate_out: int):
    """(up, down) in lowest terms."""
    r = Fraction(int(rate_out), int(rate_in))
    return r.numerator, r.denominator


@functools.lru_cache(maxsize=32)
def design_filter(up: int, down: int, dtype=np.float32):
    """The filter scipy.signal.resample_poly(x, up, down) applies to x of `dtype` (float32 or float64), and its half
    length: the default firwin(2*half_len + 1, 1/max(up, down), window=('kaiser', 5.0)) designed in float64 (windowed
    sinc, unit DC gain), cast to `dtype`, then multiplied by `up` in `dtype`.  NumPy only, no scipy at run time."""
    max_rate = max(up, down)
    half_len = 10 * max_rate
    n = 2 * half_len + 1
    fc = 1.0 / max_rate
    m = np.arange(0, n, dtype=np.float64) - 0.5 * (n - 1)
    h = fc * np.sinc(fc * m)
    alpha = (n - 1) / 2.0
    k = np.arange(0, n, dtype=np.float64)
    h = h * (np.i0(5.0 * np.sqrt(1 - ((k - alpha) / alpha) ** 2.0)) / np.i0(np.float64(5.0)))
    h = h / np.sum(h)
    h = h.astype(dtype)
    h *= dtype(up)
    h.setflags(write=False)
    return h, half_len


def polyphase_bank(up: int, down: int, dtype=np.float32):
    """(bank (up, taps), n_pre_remove) of resample_poly(x, up, down): resample_poly's filter front-padded with
    n_pre_pad = down - half_len % down zeros, split phase-major (bank[p, j] = h[p + up*j], zero past the end);
    n_pre_remove = (half_len + n_pre_pad) // down outputs of the full convolution are dropped.  up == down == 1 is the
    identity: bank [[1]], nothing removed."""
    if up == down == 1:
        return np.ones((1, 1), dtype), 0
    h, half_len = design_filter(up, down, dtype)
    n_pre_pad = down - half_len % down
    hp = np.concatenate([np.zeros(n_pre_pad, dtype), h])
    taps = -(-len(hp) // up)
    full = np.zeros(up * taps, dtype)
    full[:len(hp)] = hp
    return np.ascontiguousarray(full.reshape(taps, up).T), (half_len + n_pre_pad) // down


class Resampler:
    """Recorded audio -> mono float32 at `rate_out` on the GPU: int16 or float32 samples, 1-8 interleaved channels,
    any input rate; conversion, mix-down and polyphase resampling in one kernel launch.

    The filter is resample_poly's (designed once on the host, kept on the device phase-major), so the result is
    resample_poly's up to fp32 rounding of the sums; the mix-down is bit-identical to the host `load_audio`."""

    def __init__(self, rate_in: int, rate_out: int = 16000, device="cuda"):
        import torch
        self.rate_in, self.rate_out = int(rate_in), int(rate_out)
        if self.rate_in < 1 or self.rate_out < 1:
            raise ValueError(f"sample rates must be positive, got {rate_in} -> {rate_out}")
        self.up, self.down = resample_ratio(self.rate_in, self.rate_out)
        bank, self.n_pre_remove = polyphase_bank(self.up, self.down)
        self.bank = torch.from_numpy(bank).to(device)
        self.taps = bank.shape[1]

    def n_out(self, n_in: int) -> int:
        return -(-int(n_in) * self.up // self.down)

    def __call__(self, pcm, out=None):
        """pcm: (batch, n_in, channels) int16 / float32 CUDA tensor -> (batch, n_out(n_in)) float32 (into `out` if
        given: any clip stride)."""
        from . import ops
        return ops.resample_poly(pcm, self.bank, self.up, self.down, self.n_pre_remove, out=out)
