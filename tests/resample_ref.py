"""float64 NumPy restatement of the polyphase sum computed by pm_resample_poly_f32, shared by the CPU and GPU tests."""
import numpy as np


def mix_down(pcm):
    """(n, channels) int16 / float32 -> float32 mono, exactly as audio_io.load_audio does on the host."""
    x = pcm.astype(np.float32) / 32768.0 if pcm.dtype == np.int16 else pcm.astype(np.float32)
    return x.mean(axis=1).astype(np.float32)


def polyphase_sum(mono, bank, up, down, n_pre_remove):
    """(y, abs_sum, taps) in float64: y[m] = sum_j bank[p, j] * mono[q - j] with (m + n_pre_remove)*down = q*up + p,
    samples outside the clip read as zero; abs_sum[m] = sum_j |bank[p, j]| * |mono[q - j]|; taps = taps per output."""
    mono = np.asarray(mono, np.float64)
    bank = np.asarray(bank, np.float64)
    n_in = mono.shape[0]
    taps = bank.shape[1]
    n_out = -(-n_in * up // down)
    t = (np.arange(n_out, dtype=np.int64) + n_pre_remove) * down
    q, p = t // up, t % up
    idx = q[:, None] - np.arange(taps)[None, :]
    ok = (idx >= 0) & (idx < n_in)
    x = np.where(ok, mono[np.clip(idx, 0, max(n_in - 1, 0))] if n_in else 0.0, 0.0)
    h = bank[p]
    return (h * x).sum(axis=1), (np.abs(h) * np.abs(x)).sum(axis=1), taps
