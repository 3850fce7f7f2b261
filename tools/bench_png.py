#!/usr/bin/env python
"""PNG encoding of rendered frames on one GPU (pantomatrix_b200/png.py), against Pillow on the host.

    python tools/bench_png.py OUT.json [--reps 5] [--pillow-frames 30]

Inputs: the frames tools/bench_render.py draws on the full-size synthetic surface model: render_sequence of EMAGE
generate() output (synthetic weights), 1 x 300 and 8 x 300 frames of 960 x 720, and render_body(upsample=2) of CaMN
forward() output, 1 and 8 clips of 270 frames of 480 x 720.
Reported per input, from CUDA events after a warm-up call (medians over --reps):
  the encode call (ms per call and per frame), each of its launches (memset, count, scan, emit, crc), bytes per frame,
  and the least bytes it must move (3 bytes read per pixel, the encoded bytes written) against the 3.35 TB/s HBM3
  figure;
  Pillow's default and compress_level=1 on --pillow-frames evenly spaced frames: host ms and bytes per frame, labelled
  with the host CPU model and thread count;
and, for one 300-frame EMAGE clip, the demos' output stage end to end on the host clock: render + encode + copy + file
writes (png.write_frames) against render + copy + Pillow's default, into a temporary directory removed afterwards.
The card's name, power limit and max SM clock are read in the same run.  Nothing is written except OUT."""
import argparse
import io
import json
import os
import platform
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.weights import synth_audio  # noqa: E402
from pantomatrix_b200 import _lib, ops, png  # noqa: E402
from pantomatrix_b200.body_model import SmplxBodyModel  # noqa: E402
from pantomatrix_b200.pipeline import generate  # noqa: E402
from pantomatrix_b200.render import MeshRenderer  # noqa: E402
from synthetic_models import build_lstm_product, build_product, smplx_surface_arrays  # noqa: E402

PEAK_BW = 3.35e12


def card():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
    out = subprocess.run(q + [f"--id=GPU-{torch.cuda.get_device_properties(0).uuid}"], capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "name_power_limit_max_sm_clock": out.stdout.strip() or None}


def host_cpu():
    model = None
    try:
        with open("/proc/cpuinfo") as f:
            model = next((ln.split(":", 1)[1].strip() for ln in f if ln.startswith("model name")), None)
    except OSError:
        pass
    return {"model": model or f"not reported in /proc/cpuinfo ({platform.machine()})", "threads": os.cpu_count(),
            "pillow_threads_used": 1}


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def stages(frames, data, nbytes, reps):
    """Median ms of each launch of one encode call, timed one by one in launch order."""
    n, h, w, _ = frames.shape
    rb = torch.empty(n, h, dtype=torch.int64, device="cuda")
    ra = torch.empty(n, h, dtype=torch.int64, device="cuda")
    st, cap, fs = ops._stream(), data.shape[1], 3 * h * w
    calls = {
        "memset": lambda: _lib.call("pm_memset_async", data.data_ptr(), 0, data.numel(), st),
        "count": lambda: _lib.call("pm_png_count", frames.data_ptr(), fs, n, h, w, rb.data_ptr(), ra.data_ptr(), st),
        "scan": lambda: _lib.call("pm_png_scan", n, h, w, rb.data_ptr(), ra.data_ptr(), data.data_ptr(), cap,
                                  nbytes.data_ptr(), st),
        "emit": lambda: _lib.call("pm_png_emit", frames.data_ptr(), fs, n, h, w, rb.data_ptr(), data.data_ptr(), cap,
                                  st),
        "crc": lambda: _lib.call("pm_png_crc", n, h, w, data.data_ptr(), cap, nbytes.data_ptr(), st),
    }
    times = {k: [] for k in calls}
    for _ in range(reps):
        for k, fn in calls.items():
            times[k].append(event_ms(fn))
    return {k: statistics.median(v) for k, v in times.items()}


def pillow(frames, count):
    idx = np.linspace(0, frames.shape[0] - 1, min(count, frames.shape[0])).astype(int)
    host = frames[torch.as_tensor(idx, device=frames.device)].cpu().numpy()
    res = {}
    for name, kw in (("default", {}), ("compress_level_1", {"compress_level": 1})):
        ms, size = [], []
        for img in host:
            buf = io.BytesIO()
            t0 = time.perf_counter()
            Image.fromarray(img).save(buf, format="PNG", **kw)
            ms.append((time.perf_counter() - t0) * 1e3)
            size.append(buf.tell())
        res[name] = {"frames": len(host), "ms_per_frame_median": statistics.median(ms),
                     "bytes_per_frame_mean": float(np.mean(size))}
    return res


def arm(frames, reps, pillow_frames):
    frames = frames.reshape(-1, *frames.shape[-3:])
    n, h, w, _ = frames.shape
    data = torch.empty(n, png.slot_bytes(h, w), dtype=torch.uint8, device="cuda")
    nbytes = torch.empty(n, dtype=torch.int64, device="cuda")
    png.encode(frames, out=(data, nbytes))                      # warm-up
    torch.cuda.synchronize()
    ms = [event_ms(lambda: png.encode(frames, out=(data, nbytes))) for _ in range(reps)]
    sizes = nbytes.cpu().numpy()
    med = statistics.median(ms)
    least = 3 * n * h * w + int(sizes.sum())
    return {"frames": n, "height": h, "width": w, "encode_ms_median": med, "encode_ms_all": ms,
            "encode_ms_per_frame": med / n, "frames_per_s": n / (med * 1e-3),
            "bytes_per_frame_mean": float(sizes.mean()), "bytes_per_frame_min": int(sizes.min()),
            "bytes_per_frame_max": int(sizes.max()), "slot_bytes": int(data.shape[1]),
            "least_bytes": least, "share_of_3.35TBps": least / (med * 1e-3) / PEAK_BW,
            "stage_ms_median": stages(frames, data, nbytes, reps),
            "pillow_host": pillow(frames, pillow_frames) if pillow_frames else "not measured"}


def output_stage(r, pred, reps):
    """One 300-frame EMAGE clip from poses to files: GPU encode vs Pillow, host clock around work that ends in files."""
    poses, expr, trans = (pred[k][:1] for k in ("motion_axis_angle", "expression", "trans"))
    res = {"gpu_png": [], "pillow_default": []}
    for _ in range(reps):
        for name in res:
            d = tempfile.mkdtemp()
            try:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                frames = r.render_sequence(poses, expr, trans)[0]
                if name == "gpu_png":
                    png.write_frames(frames, d)
                else:
                    for i, img in enumerate(frames.cpu().numpy()):
                        Image.fromarray(img).save(os.path.join(d, f"frame_{i:05d}.png"))
                res[name].append(time.perf_counter() - t0)
                assert len(os.listdir(d)) == frames.shape[0]
            finally:
                shutil.rmtree(d)
    out = {k: {"s_median": statistics.median(v), "s_all": v} for k, v in res.items()}
    out["speedup"] = out["pillow_default"]["s_median"] / out["gpu_png"]["s_median"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pillow-frames", type=int, default=30)
    ap.add_argument("--stage-reps", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the PNG benchmark measures the GPU: no CUDA device found"
    torch.cuda.set_device(0)
    model, vqm = build_product(seed=0, device="cuda")
    _, pred = generate(model, vqm, torch.from_numpy(synth_audio(8, 160000, 5)).cuda())
    r = MeshRenderer(SmplxBodyModel(smplx_surface_arrays(), "cuda"))
    res = {"card": card(), "host_cpu": host_cpu(),
           "parse_distances": "1, 2, 3, 4, 5, 6, 7, 8, 9, 12, s, s-3, s+3, s-6, s+6 (not retuned)"}
    for clips in (1, 8):
        frames = r.render_sequence(*(pred[k][:clips] for k in ("motion_axis_angle", "expression", "trans")))
        res[f"emage_sequence_{clips}x300"] = arm(frames, args.reps, args.pillow_frames if clips == 1 else 0)
        print("emage", clips, json.dumps(res[f"emage_sequence_{clips}x300"])[:600], flush=True)
        del frames
    camn = build_lstm_product("camn", device="cuda")
    poses = camn(torch.from_numpy(synth_audio(8, 160000, 5)).cuda(),
                 torch.zeros(8, 1, dtype=torch.long, device="cuda"))["motion_axis_angle"]
    poses = poses.reshape(8, poses.shape[1], 165)
    for clips in (1, 8):
        frames = r.render_body(poses[:clips], torch.zeros(clips, poses.shape[1], 3, device="cuda"), upsample=2)
        res[f"camn_body_{clips}x10s"] = arm(frames, args.reps, args.pillow_frames if clips == 1 else 0)
        print("camn", clips, json.dumps(res[f"camn_body_{clips}x10s"])[:600], flush=True)
        del frames
    res["output_stage_1x300"] = output_stage(r, pred, args.stage_reps)
    print("output stage", json.dumps(res["output_stage_1x300"]), flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
