#!/usr/bin/env python
"""Audio front-end benchmark: the resampling kernel alone, the host resampler it replaces, and the EMAGE step end to
end from recorded audio.

    python tools/bench_audio_frontend.py OUT_DIR [--reps 200] [--steps 10] [--clips 32]

Writes OUT_DIR/audio_frontend.json (and prints it):
  kernel   per input format (44.1 / 48 kHz; int16 stereo / float32 mono), 32 clips x 10 s -> 16 kHz: CUDA events around
           each of `reps` launches after warm-up (median and mean), bytes moved = PCM read + fp32 output written
           (computed from shapes; filter and halo re-reads not counted), GB/s and the share of the H100 SXM data-sheet
           3.35 TB/s.  The kernel is bound by those bytes, not by its ~60 FMAs per output sample.
  host     scipy.signal.resample_poly on this machine's host for the same batch (int16 stereo -> float32 mono mix-down
           included, as audio_io.load_audio does it), median of 3.
  e2e      wall clock per step, median of `steps`: pinned host input -> H2D -> captured step -> D2H of the emitted
           SMPL-X parameters, for (a) CapturedPipeline(input_rate=48000, input_channels=2, input_dtype=int16) fed the
           int16 stereo PCM, (b) host resample_poly of that PCM, then the default 16 kHz CapturedPipeline, (c) the
           default pipeline fed 16 kHz float32 directly (no front-end).  The three alternate step by step.
  device   torch.cuda.get_device_name and nvidia-smi's name / power.limit, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_GBPS = 3350.0                  # H100 SXM data sheet (700 W); not measured here
SECONDS, FRAMES_PER_CLIP = 10, 300


def _pcm(clips, rate, channels, dtype, seed):
    """Seeded speech-level test signal: a few tones plus noise, int16 or float32 in [-1, 1]."""
    import numpy as np
    rng = np.random.default_rng(seed)
    n = rate * SECONDS
    t = np.arange(n, dtype=np.float64) / rate
    tone = 0.2 * np.sin(2 * np.pi * 220 * t) + 0.1 * np.sin(2 * np.pi * 1730 * t)
    x = tone[None, :, None] + rng.normal(0, 0.05, (clips, n, channels))
    if dtype == "int16":
        return np.clip(np.rint(x * 32767), -32768, 32767).astype(np.int16)
    return np.clip(x, -1, 1).astype(np.float32)


def _host_front_end(pcm, rate):
    """audio_io.load_audio's host path per clip: int16 -> float32, mean over channels, resample_poly to 16 kHz."""
    import numpy as np
    from scipy.signal import resample_poly
    from pantomatrix_b200 import audio_io
    up, down = audio_io.resample_ratio(rate, 16000)
    out = []
    for clip in pcm:
        x = clip.astype(np.float32) / 32768.0 if clip.dtype == np.int16 else clip
        out.append(resample_poly(x.mean(axis=1).astype(np.float32), up, down).astype(np.float32))
    return np.stack(out)


def kernel_times(clips, reps):
    import torch
    from pantomatrix_b200 import audio_io
    res = {}
    for rate in (44100, 48000):
        rs = audio_io.Resampler(rate, 16000, device="cuda")
        for fmt, ch, dtype in (("int16 stereo", 2, "int16"), ("float32 mono", 1, "float32")):
            pcm = torch.from_numpy(_pcm(clips, rate, ch, dtype, rate + ch)).cuda()
            n_in = pcm.shape[1]
            out = torch.empty(clips, rs.n_out(n_in), device="cuda")
            for _ in range(10):
                rs(pcm, out=out)
            torch.cuda.synchronize()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
            for s, e in ev:
                s.record()
                rs(pcm, out=out)
                e.record()
            torch.cuda.synchronize()
            ms = sorted(s.elapsed_time(e) for s, e in ev)
            med, mean = ms[len(ms) // 2], sum(ms) / len(ms)
            nbytes = pcm.numel() * pcm.element_size() + out.numel() * 4
            gbps = nbytes / (med * 1e-3) / 1e9
            res[f"{rate} Hz {fmt}"] = {
                "clips": clips, "n_in": n_in, "n_out": out.shape[1], "up": rs.up, "down": rs.down, "taps_per_phase": rs.taps,
                "launches": reps, "median_ms": med, "mean_ms": mean, "min_ms": ms[0],
                "bytes_moved": nbytes, "bytes_per_output_sample": nbytes / out.numel(), "GBps": gbps,
                "hbm_frac": gbps / HBM_GBPS, "bound": "bytes (HBM)",
                "fma_per_output_sample": rs.taps}
    return res


def host_times(clips):
    res = {}
    for rate in (44100, 48000):
        pcm = _pcm(clips, rate, 2, "int16", rate + 2)
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            _host_front_end(pcm, rate)
            ts.append(time.perf_counter() - t0)
        res[f"{rate} Hz int16 stereo"] = {"median_ms": 1e3 * sorted(ts)[1], "runs_ms": [1e3 * t for t in ts],
                                         "host_cores": os.cpu_count(), "what": "int16 -> float32, channel mean, "
                                         "scipy.signal.resample_poly to 16 kHz, clip by clip, one thread"}
    return res


def e2e(clips, steps):
    import torch
    from oracle.weights import synth_audio
    from pantomatrix_b200.pipeline import CapturedPipeline
    from synthetic_models import build_product
    model, vqm = build_product(seed=0, device="cuda")
    n16 = 16000 * SECONDS
    cap16 = CapturedPipeline(model, vqm, clips, n16)
    cap48 = CapturedPipeline(model, vqm, clips, 48000 * SECONDS, input_rate=48000, input_channels=2,
                             input_dtype=torch.int16)
    pcm48 = _pcm(clips, 48000, 2, "int16", 7)
    pcm48_pinned = torch.from_numpy(pcm48).pin_memory()
    audio16_pinned = torch.from_numpy(synth_audio(clips, n16, 1234)).pin_memory()
    staging = torch.empty(clips, n16).pin_memory()
    out_host = {k: torch.empty(clips, FRAMES_PER_CLIP, d).pin_memory() for k, d in
                (("motion_axis_angle", 165), ("expression", 100), ("trans", 3))}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")          # > the 50 MB L2

    def fetch(pred):
        for k, v in out_host.items():
            v.copy_(pred[k], non_blocking=True)

    def host_resample_then_16k():
        staging.copy_(torch.from_numpy(_host_front_end(pcm48, 48000)))
        fetch(cap16(staging)[1])

    arms = {
        "gpu_front_end_48k_int16_stereo": lambda: fetch(cap48(pcm48_pinned)[1]),
        "host_resample_poly_then_16k": host_resample_then_16k,
        "16k_float32_input": lambda: fetch(cap16(audio16_pinned)[1]),
    }
    for fn in arms.values():                                                # warm-up
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for i in range(steps):
        for k, fn in arms.items():
            flush.fill_(i & 0xFF)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    res = {}
    for k, ts in times.items():
        med = sorted(ts)[len(ts) // 2]
        res[k] = {"median_ms": 1e3 * med, "frames_per_s": clips * FRAMES_PER_CLIP / med,
                  "runs_ms": [round(1e3 * t, 3) for t in ts]}
    res["config"] = {"clips": clips, "seconds_per_clip": SECONDS, "steps": steps, "h2d_bytes": {
        "gpu_front_end_48k_int16_stereo": pcm48_pinned.numel() * 2, "host_resample_poly_then_16k": staging.numel() * 4,
        "16k_float32_input": audio16_pinned.numel() * 4}, "kernels_per_replay": {
        "48k int16 stereo": cap48.kernels_per_replay, "16k float32": cap16.kernels_per_replay},
        "timer": "wall clock, pinned host buffers, H2D + replay + D2H of motion_axis_angle / expression / trans, "
                 "256 MB L2 flush before each step (outside the timer), arms alternating"}
    g, h, d = (res[k]["frames_per_s"] for k in ("gpu_front_end_48k_int16_stereo", "host_resample_poly_then_16k",
                                                  "16k_float32_input"))
    res["ratios"] = {"gpu_front_end_vs_16k_input": g / d, "gpu_front_end_vs_host_resample": g / h}
    return res


def device_info():
    import torch
    info = {"torch_device_name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["nvidia_smi_name_power_limit"] = q.stdout.strip()
    except Exception as exc:
        info["nvidia_smi_name_power_limit"] = f"unavailable: {exc!r}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--clips", type=int, default=32)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_audio_frontend.py needs a CUDA device")
    os.makedirs(args.out_dir, exist_ok=True)
    res = {"device": device_info(), "kernel": kernel_times(args.clips, max(args.reps, 200)),
           "host": host_times(args.clips), "e2e": e2e(args.clips, max(args.steps, 10))}
    res["device_after"] = device_info()
    path = os.path.join(args.out_dir, "audio_frontend.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
