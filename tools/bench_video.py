#!/usr/bin/env python
"""H.264 encoding of rendered frames on one GPU (pantomatrix_b200/video.py), beside PNG encoding of the same frames.

    python tools/bench_video.py OUT.json [--reps 5] [--stage-reps 3] [--psnr-frames 30]

Inputs: the frames tools/bench_png.py uses: render_sequence of EMAGE generate() output (synthetic weights, full-size
synthetic surface model), 1 x 300 and 8 x 300 frames of 960 x 720, and render_body(upsample=2) of CaMN forward()
output, 1 clip of 270 frames of 480 x 720.
Reported per input, from CUDA events after a warm-up call (medians over --reps):
  the video.encode call at qp 20 (ms per call and per frame), each of its launches (memset, encode, gather), bytes
  per frame (min, mean, max), and png.encode on the same frames in the same run;
  for the 1 x 300 EMAGE clip, bytes per frame and luma PSNR against the source Y (the colour rule's Y, in integers) at
  qp 16, 20, 26 and 32, the luma decoded by OpenCV's FFmpeg from a write_mp4 file of the first --psnr-frames frames;
and, for one 300-frame EMAGE clip, the demos' output stage on the host clock: render + encode + copy + write mp4
(video.write_mp4) against render + png.write_frames, alternating the two, into a temporary directory removed after.
The card's name, power limit and max SM clock are read in the same run.  Nothing is written except OUT."""
import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from measure import card, event_ms, launch_ms  # noqa: E402
from oracle.weights import synth_audio  # noqa: E402
from pantomatrix_b200 import _lib, ops, png, video  # noqa: E402
from pantomatrix_b200.body_model import SmplxBodyModel  # noqa: E402
from pantomatrix_b200.pipeline import generate  # noqa: E402
from pantomatrix_b200.render import MeshRenderer  # noqa: E402
from synthetic_models import build_lstm_product, build_product, smplx_surface_arrays  # noqa: E402

QP = 20


def stages(frames, clip_len, data, nbytes, reps):
    """Median ms of each launch of one encode call, timed one by one in launch order."""
    n, h, w, _ = frames.shape
    sc = video.slice_bytes(w)
    scratch = torch.empty(n, h // 16, sc, dtype=torch.uint8, device="cuda")
    sizes = torch.empty(n, h // 16, dtype=torch.int32, device="cuda")
    st, cap, fs = ops._stream(), data.shape[1], 3 * h * w
    calls = {
        "memset": lambda: _lib.call("pm_memset_async", data.data_ptr(), 0, data.numel(), st),
        "encode": lambda: _lib.call("pm_h264_encode", frames.data_ptr(), fs, n, clip_len, h, w, QP,
                                    scratch.data_ptr(), sc, sizes.data_ptr(), st),
        "gather": lambda: _lib.call("pm_h264_gather", n, h, w, scratch.data_ptr(), sc, sizes.data_ptr(),
                                    data.data_ptr(), cap, nbytes.data_ptr(), st),
    }
    return launch_ms(calls, reps)


def arm(frames, reps):
    clip_len = frames.shape[1] if frames.dim() == 5 else frames.shape[0]
    frames = frames.reshape(-1, *frames.shape[-3:])
    n, h, w, _ = frames.shape
    data = torch.empty(n, video.slot_bytes(h, w), dtype=torch.uint8, device="cuda")
    nbytes = torch.empty(n, dtype=torch.int64, device="cuda")
    video.encode(frames, qp=QP, out=(data, nbytes))             # warm-up
    torch.cuda.synchronize()
    ms = [event_ms(lambda: video.encode(frames, qp=QP, out=(data, nbytes))) for _ in range(reps)]
    sizes = nbytes.cpu().numpy()
    med = statistics.median(ms)
    split = stages(frames, clip_len, data, nbytes, reps)
    del data
    pdata = torch.empty(n, png.slot_bytes(h, w), dtype=torch.uint8, device="cuda")
    pn = torch.empty(n, dtype=torch.int64, device="cuda")
    png.encode(frames, out=(pdata, pn))
    torch.cuda.synchronize()
    pms = [event_ms(lambda: png.encode(frames, out=(pdata, pn))) for _ in range(reps)]
    psizes = pn.cpu().numpy()
    return {"frames": n, "height": h, "width": w, "qp": QP, "encode_ms_median": med, "encode_ms_all": ms,
            "encode_ms_per_frame": med / n, "frames_per_s": n / (med * 1e-3),
            "bytes_per_frame_mean": float(sizes.mean()), "bytes_per_frame_min": int(sizes.min()),
            "bytes_per_frame_max": int(sizes.max()), "slot_bytes": video.slot_bytes(h, w),
            "stage_ms_median": split,
            "png_encode_ms_median": statistics.median(pms), "png_bytes_per_frame_mean": float(psizes.mean())}


def source_y(frames):
    f = frames.to(torch.int32)
    return ((66 * f[..., 0] + 129 * f[..., 1] + 25 * f[..., 2] + 128) >> 8) + 16


def quality(frames, count, tmp):
    """Bytes per frame and luma PSNR (against the colour rule's Y) at several qp, decoded by OpenCV's FFmpeg."""
    import cv2
    clip = frames[:count]
    ys = source_y(clip).cpu().numpy().astype(np.float64)
    out = {}
    for qp in (16, 20, 26, 32):
        _, nbytes = video.encode(clip, qp=qp)
        sizes = nbytes.cpu().numpy()
        path = video.write_mp4(clip, os.path.join(tmp, f"q{qp}.mp4"), fps=30, qp=qp)
        cap = cv2.VideoCapture(path, cv2.CAP_FFMPEG)
        cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
        psnr = []
        h, w = clip.shape[1:3]
        for i in range(count):
            ok, fr = cap.read()
            assert ok, i
            y = np.asarray(fr).reshape(-1)[:h * w].reshape(h, w).astype(np.float64)
            mse = ((y - ys[i]) ** 2).mean()
            psnr.append(99.0 if mse == 0 else 10 * np.log10(255.0 ** 2 / mse))
        cap.release()
        out[f"qp{qp}"] = {"bytes_per_frame_min": int(sizes.min()), "bytes_per_frame_mean": float(sizes.mean()),
                          "bytes_per_frame_max": int(sizes.max()), "luma_psnr_db_mean": float(np.mean(psnr)),
                          "luma_psnr_db_min": float(np.min(psnr))}
    return out


def output_stage(r, pred, reps):
    """One 300-frame EMAGE clip from poses to files, alternating the two arms, host clock around work that ends in
    files: render + video.write_mp4 against render + png.write_frames."""
    poses, expr, trans = (pred[k][:1] for k in ("motion_axis_angle", "expression", "trans"))
    res, size = {"mp4": [], "png_files": []}, {}
    for _ in range(reps):
        for name in res:
            d = tempfile.mkdtemp()
            try:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                frames = r.render_sequence(poses, expr, trans)[0]
                if name == "mp4":
                    video.write_mp4(frames, os.path.join(d, "clip.mp4"), fps=30, qp=QP)
                else:
                    png.write_frames(frames, d)
                res[name].append(time.perf_counter() - t0)
                size[name] = sum(os.path.getsize(os.path.join(d, x)) for x in os.listdir(d))
            finally:
                shutil.rmtree(d)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    frames = r.render_sequence(poses, expr, trans)[0]
    torch.cuda.synchronize()
    render_s = time.perf_counter() - t0
    out = {k: {"s_median": statistics.median(v), "s_all": v} for k, v in res.items()}
    out["mp4_file_bytes"], out["png_files_bytes"] = size["mp4"], size["png_files"]
    out["render_only_s"] = render_s
    del frames
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stage-reps", type=int, default=3)
    ap.add_argument("--psnr-frames", type=int, default=30)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the video benchmark measures the GPU: no CUDA device found"
    torch.cuda.set_device(0)
    model, vqm = build_product(seed=0, device="cuda")
    _, pred = generate(model, vqm, torch.from_numpy(synth_audio(8, 160000, 5)).cuda())
    r = MeshRenderer(SmplxBodyModel(smplx_surface_arrays(), "cuda"))
    res = {"card": card()}
    for clips in (1, 8):
        frames = r.render_sequence(*(pred[k][:clips] for k in ("motion_axis_angle", "expression", "trans")))
        res[f"emage_sequence_{clips}x300"] = arm(frames, args.reps)
        print("emage", clips, json.dumps(res[f"emage_sequence_{clips}x300"])[:700], flush=True)
        if clips == 1:
            tmp = tempfile.mkdtemp()
            try:
                res["emage_quality"] = quality(frames[0], args.psnr_frames, tmp)
            finally:
                shutil.rmtree(tmp)
            print("quality", json.dumps(res["emage_quality"]), flush=True)
        del frames
    camn = build_lstm_product("camn", device="cuda")
    poses = camn(torch.from_numpy(synth_audio(1, 160000, 5)).cuda(),
                 torch.zeros(1, 1, dtype=torch.long, device="cuda"))["motion_axis_angle"]
    poses = poses.reshape(1, poses.shape[1], 165)
    frames = r.render_body(poses, torch.zeros(1, poses.shape[1], 3, device="cuda"), upsample=2)
    res["camn_body_1x10s"] = arm(frames, args.reps)
    print("camn", json.dumps(res["camn_body_1x10s"])[:700], flush=True)
    del frames
    res["output_stage_1x300"] = output_stage(r, pred, args.stage_reps)
    print("output stage", json.dumps(res["output_stage_1x300"]), flush=True)
    res["card_after"] = card()
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
