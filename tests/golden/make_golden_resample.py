"""Generate tests/golden/resample.npz: scipy.signal.resample_poly outputs for the GPU resampler tests (which run where
scipy may be absent).

    python tests/golden/make_golden_resample.py

Each case is a seeded batch of recorded audio `<case>_pcm` (batch, n_in, channels) at `<case>_rate` Hz and the host
front-end's result for it, `<case>_out` (batch, n_out) float32: mix-down as in audio_io.load_audio, then
resample_poly(mono_float32, up, down) to 16 kHz (float32 taps, scipy's own accumulation).
"""
import os
from fractions import Fraction

import numpy as np
from scipy.signal import resample_poly

HERE = os.path.dirname(os.path.abspath(__file__))
# (case, input rate, channels, dtype, samples per clip)
CASES = [("s44100_i16x2", 44100, 2, np.int16, 9001), ("s48000_i16x2", 48000, 2, np.int16, 9003),
         ("s22050_f32x1", 22050, 1, np.float32, 6007), ("s44056_f32x1", 44056, 1, np.float32, 9011)]
BATCH = 2


def _mono(pcm):
    x = pcm.astype(np.float32) / 32768.0 if pcm.dtype == np.int16 else pcm
    return x.mean(axis=1).astype(np.float32)


def main():
    rng = np.random.default_rng(20261015)
    out = {}
    for name, rate, ch, dtype, n in CASES:
        if dtype == np.int16:
            t = np.arange(n) / rate
            tone = 12000 * np.sin(2 * np.pi * 440 * t)[:, None] + rng.normal(0, 3000, (BATCH, n, ch))
            pcm = np.clip(np.rint(tone), -32768, 32767).astype(np.int16)
        else:
            pcm = rng.uniform(-1, 1, (BATCH, n, ch)).astype(np.float32)
        r = Fraction(16000, rate)
        res = np.stack([resample_poly(_mono(c), r.numerator, r.denominator).astype(np.float32) for c in pcm])
        out[name + "_pcm"], out[name + "_rate"], out[name + "_out"] = pcm, np.int64(rate), res
    np.savez(os.path.join(HERE, "resample.npz"), **out)


if __name__ == "__main__":
    main()
