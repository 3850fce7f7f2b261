#!/usr/bin/env python
"""H.264 encoding of rendered frames on one GPU (pantomatrix_b200/video.py), beside PNG encoding of the same frames.

    python tools/bench_video.py OUT.json [--reps 5] [--stage-reps 3] [--psnr-frames 30] [--no-mb-types] [--gop-only]
                                         [--baseline-lib PARENT/pantomatrix_b200/libpm_emage.so]
                                         [--me-only [--me-mb-frames 4]] [--i4-only [--i4-mb-frames 2]]

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
GOP arms (keyframe interval gop 1, 30 and T, the clip length), per input: the video.encode call at qp 20 (median ms,
the three gops alternating), bytes per frame (min, mean, max), and luma PSNR of the first --psnr-frames frames decoded
by OpenCV's FFmpeg from a write_mp4 file; for the 1 x 300 EMAGE clip also the share of P_Skip / inter / intra / I_PCM
macroblocks over one whole GOP at gop 30 (frames 0..29: the IDR frame and 29 P frames), counted by the CPU
restatement (tests/h264_ref.py), whose bytes equal the GPU's; and the output stage (render + write_mp4) at gop 1
against gop 30, alternating.  --gop-only runs only the GOP arms and that output stage.
--baseline-lib: the libpm_emage.so of another build (for instance the parent commit's, built from a checkout of it):
pm_h264_encode of that library, pm_h264_encode of this tree and pm_h264_encode_gop(gop = 1) of this tree on the
EMAGE 1 x 300 and 8 x 300 frames, alternating, medians over 2 * --reps, and whether all three wrote the same slices.
Motion search arms (--me-only runs only these): gop 30 and T with search 0, 16 and 32, per input, the six arms
alternating in the timed loop: the video.encode call (median ms), bytes per frame (min, mean, max), luma PSNR of the
first --psnr-frames frames, and the time of one call's search and code kernels from torch.profiler; for the 1 x 300
EMAGE clip also the macroblock shares over the first --me-mb-frames frames of the first GOP at gop 30, with P split
into zero and non-zero vectors, counted by the CPU restatement (tests/h264_ref.py; the whole 30-frame GOP takes it
too long at 960 x 720); and the output stage (render + write_mp4) at gop 30 with search 0 against search 16.
Intra 4x4 arms (--i4-only runs only these): gop 1 and 30, search 0 and 16 (gop 30), qp 20 and 26, each with and
without intra4x4, per input (the EMAGE 1 x 300 and CaMN 1 x 270 clips), all alternating in the timed loop: the
video.encode call (median ms), bytes per frame (min, mean, max) and luma PSNR of the first --psnr-frames frames; for
the EMAGE clip also, from the CPU restatement (tests/h264_ref.py) over its first --i4-mb-frames frames at gop 30
and search 0, the macroblock shares, the histogram of the nine modes, and the bytes for several values of the rule's
constant c and without intra4x4.
The card's name, power limit and max SM clock are read in the same run.  Nothing is written except OUT."""
import ctypes
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

# the CPU restatement tests/h264_ref.py is imported only by the arms that count macroblocks with it
sys.path.insert(0, os.path.join(ROOT, "tests"))

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


def luma_psnr(frames, path, count):
    """Mean and min luma PSNR (dB) of the first count frames of an MP4 file against the colour rule's Y."""
    import cv2
    ys = source_y(frames[:count]).cpu().numpy().astype(np.float64)
    h, w = frames.shape[1:3]
    cap = cv2.VideoCapture(path, cv2.CAP_FFMPEG)
    cap.set(cv2.CAP_PROP_CONVERT_RGB, 0)
    psnr = []
    for i in range(count):
        ok, fr = cap.read()
        assert ok, i
        y = np.asarray(fr).reshape(-1)[:h * w].reshape(h, w).astype(np.float64)
        mse = ((y - ys[i]) ** 2).mean()
        psnr.append(99.0 if mse == 0 else 10 * np.log10(255.0 ** 2 / mse))
    cap.release()
    return float(np.mean(psnr)), float(np.min(psnr))


def baseline(frames, lib_path, reps):
    """pm_h264_encode of the library at lib_path against this tree's pm_h264_encode and pm_h264_encode_gop(gop = 1),
    alternating: median ms of each, and whether the three wrote the same slices and sizes."""
    clip_len = frames.shape[1]
    frames = frames.reshape(-1, *frames.shape[-3:])
    n, h, w, _ = frames.shape
    sc = video.slice_bytes(w)
    base = ctypes.CDLL(lib_path)
    base.pm_h264_encode.argtypes, base.pm_h264_encode.restype = _lib.SIGNATURES["pm_h264_encode"], ctypes.c_int
    bufs = {k: (torch.zeros(n, h // 16, sc, dtype=torch.uint8, device="cuda"),
                torch.zeros(n, h // 16, dtype=torch.int32, device="cuda"))
            for k in ("baseline", "encode", "encode_gop1")}
    args = lambda k: (frames.data_ptr(), 3 * h * w, n, clip_len, h, w, QP, bufs[k][0].data_ptr(), sc,
                      bufs[k][1].data_ptr())
    st = ops._stream()

    def run_base():
        assert base.pm_h264_encode(*args("baseline"), st) == 0

    calls = {"baseline": run_base,
             "encode": lambda: _lib.call("pm_h264_encode", *args("encode"), st),
             "encode_gop1": lambda: _lib.call("pm_h264_encode_gop", *args("encode_gop1"), 1, None, 0, st)}
    for fn in calls.values():
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in calls}
    for _ in range(2 * reps):
        for k, fn in calls.items():
            ms[k].append(event_ms(fn))
    same = all(torch.equal(bufs[k][i], bufs["baseline"][i]) for k in calls for i in (0, 1))
    return {"lib": lib_path, "identical": same,
            **{k: {"ms_median": statistics.median(v), "ms_all": v} for k, v in ms.items()}}


def gop_arms(frames, reps, psnr_frames, mb_types, tmp):
    """encode time, bytes per frame and luma PSNR at gop 1, 30 and T, the gops alternating in the timed loop; with
    mb_types, the macroblock shares over the first whole GOP at gop 30."""
    t = frames.shape[1] if frames.dim() == 5 else frames.shape[0]
    gops = (1, 30, t)
    ms = {g: [] for g in gops}
    for g in gops:
        video.encode(frames, qp=QP, gop=g)                    # warm-up
    torch.cuda.synchronize()
    for _ in range(reps):
        for g in gops:
            ms[g].append(event_ms(lambda: video.encode(frames, qp=QP, gop=g)))
    out = {}
    clip = frames[0] if frames.dim() == 5 else frames
    for g in gops:
        sizes = video.encode(frames, qp=QP, gop=g)[1].cpu().numpy()
        path = video.write_mp4(clip, os.path.join(tmp, f"g{g}.mp4"), fps=30, qp=QP, gop=g)
        psnr_mean, psnr_min = luma_psnr(clip, path, psnr_frames)
        out[f"gop{g}"] = {"encode_ms_median": statistics.median(ms[g]), "encode_ms_all": ms[g],
                          "bytes_per_frame_mean": float(sizes.mean()), "bytes_per_frame_min": int(sizes.min()),
                          "bytes_per_frame_max": int(sizes.max()), "file_bytes_clip0": os.path.getsize(path),
                          "luma_psnr_db_mean": psnr_mean, "luma_psnr_db_min": psnr_min}
        if mb_types and g == 30 < t:
            import h264_ref
            enc = h264_ref.encode_clip(list(clip[:g].cpu().numpy()), QP, g)
            types = np.concatenate([e[2].reshape(-1) for e in enc])
            out[f"gop{g}"]["mb_share_first_gop"] = {k: float((types == k).mean())
                                                    for k in ("SKIP", "P", "DC", "H", "PCM")}
    return out


def output_stage_gop(r, pred, reps):
    """Render + video.write_mp4 of one 300-frame EMAGE clip at gop 1 against gop 30, alternating, host clock."""
    poses, expr, trans = (pred[k][:1] for k in ("motion_axis_angle", "expression", "trans"))
    res, size = {1: [], 30: []}, {}
    for _ in range(reps):
        for g in res:
            d = tempfile.mkdtemp()
            try:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                frames = r.render_sequence(poses, expr, trans)[0]
                video.write_mp4(frames, os.path.join(d, "clip.mp4"), fps=30, qp=QP, gop=g)
                res[g].append(time.perf_counter() - t0)
                size[g] = os.path.getsize(os.path.join(d, "clip.mp4"))
            finally:
                shutil.rmtree(d)
    return {f"gop{g}": {"s_median": statistics.median(v), "s_all": v, "file_bytes": size[g]} for g, v in res.items()}


def kernel_split(frames, gop, search):
    """Summed CUDA time (ms) of each kernel kind in one video.encode call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    video.encode(frames, qp=QP, gop=gop, search=search)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        video.encode(frames, qp=QP, gop=gop, search=search)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        kind = next((k for k in ("search", "encode_kernel", "gather") if k in e.key), None)
        if kind:
            out[kind] = out.get(kind, 0.0) + e.device_time_total / 1e3
    return out


def me_arms(frames, reps, psnr_frames, mb_frames, tmp):
    """gop 30 and T with search 0, 16 and 32, alternating in the timed loop: encode ms, bytes per frame, luma PSNR,
    the search / code kernel split; with mb_frames, the macroblock shares of the first mb_frames frames at gop 30."""
    t = frames.shape[1] if frames.dim() == 5 else frames.shape[0]
    arms = [(g, s) for g in (30, t) for s in (0, 16, 32)]
    ms = {a: [] for a in arms}
    for g, s in arms:
        video.encode(frames, qp=QP, gop=g, search=s)          # warm-up
    torch.cuda.synchronize()
    for _ in range(reps):
        for g, s in arms:
            ms[(g, s)].append(event_ms(lambda: video.encode(frames, qp=QP, gop=g, search=s)))
    out = {}
    clip = frames[0] if frames.dim() == 5 else frames
    for g, s in arms:
        sizes = video.encode(frames, qp=QP, gop=g, search=s)[1].cpu().numpy()
        path = video.write_mp4(clip, os.path.join(tmp, f"g{g}s{s}.mp4"), fps=30, qp=QP, gop=g, search=s)
        psnr_mean, psnr_min = luma_psnr(clip, path, psnr_frames)
        a = out[f"gop{g}_search{s}"] = {
            "encode_ms_median": statistics.median(ms[(g, s)]), "encode_ms_all": ms[(g, s)],
            "bytes_per_frame_mean": float(sizes.mean()), "bytes_per_frame_min": int(sizes.min()),
            "bytes_per_frame_max": int(sizes.max()), "file_bytes_clip0": os.path.getsize(path),
            "luma_psnr_db_mean": psnr_mean, "luma_psnr_db_min": psnr_min,
            "kernel_ms": kernel_split(frames, g, s)}
        if mb_frames and g == 30:
            import h264_ref
            enc = h264_ref.encode_clip(list(clip[:mb_frames].cpu().numpy()), QP, g, s)
            types = np.concatenate([e[2].reshape(-1) for e in enc])
            moved = np.concatenate([(e.mv if e.mv is not None else np.zeros(e.types.shape + (2,), int)).any(-1)
                                    .reshape(-1) for e in enc])
            share = {k: float((types == k).mean()) for k in ("SKIP", "DC", "H", "PCM")}
            share["P_zero"] = float(((types == "P") & ~moved).mean())
            share["P_nonzero"] = float(((types == "P") & moved).mean())
            a["mb_share_first_frames"] = {"frames": mb_frames, **share}
            assert [e[0] for e in enc] == [bytes(x) for x in _first_samples(clip[:mb_frames], g, s)]
        print("  arm", g, s, json.dumps({k: v for k, v in a.items() if k != "encode_ms_all"}), flush=True)
    return out


def _first_samples(clip, gop, search, qp=QP, intra4x4=False):
    data, nbytes = video.encode(clip, qp=qp, gop=gop, search=search, intra4x4=intra4x4)
    return [data[i, :k].cpu().numpy().tobytes() for i, k in enumerate(nbytes.tolist())]


def output_stage_me(r, pred, reps):
    """Render + video.write_mp4 of one 300-frame EMAGE clip at gop 30, search 0 against search 16, alternating."""
    poses, expr, trans = (pred[k][:1] for k in ("motion_axis_angle", "expression", "trans"))
    res, size = {0: [], 16: []}, {}
    for _ in range(reps):
        for s in res:
            d = tempfile.mkdtemp()
            try:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                frames = r.render_sequence(poses, expr, trans)[0]
                video.write_mp4(frames, os.path.join(d, "clip.mp4"), fps=30, qp=QP, gop=30, search=s)
                res[s].append(time.perf_counter() - t0)
                size[s] = os.path.getsize(os.path.join(d, "clip.mp4"))
            finally:
                shutil.rmtree(d)
    return {f"search{s}": {"s_median": statistics.median(v), "s_all": v, "file_bytes": size[s]}
            for s, v in res.items()}


def run_me(args, r, pred, res, tmp):
    for clips in (1, 8):
        frames = r.render_sequence(*(pred[k][:clips] for k in ("motion_axis_angle", "expression", "trans")))
        print("me emage", clips, flush=True)
        res[f"me_emage_sequence_{clips}x300"] = me_arms(frames, args.reps, args.psnr_frames,
                                                        args.me_mb_frames if clips == 1 else 0, tmp)
        del frames
    camn = build_lstm_product("camn", device="cuda")
    poses = camn(torch.from_numpy(synth_audio(1, 160000, 5)).cuda(),
                 torch.zeros(1, 1, dtype=torch.long, device="cuda"))["motion_axis_angle"]
    poses = poses.reshape(1, poses.shape[1], 165)
    frames = r.render_body(poses, torch.zeros(1, poses.shape[1], 3, device="cuda"), upsample=2)
    print("me camn", flush=True)
    res["me_camn_body_1x10s"] = me_arms(frames, args.reps, args.psnr_frames, 0, tmp)
    del frames
    res["output_stage_me_1x300"] = output_stage_me(r, pred, args.stage_reps)
    print("output stage me", json.dumps(res["output_stage_me_1x300"]), flush=True)


def i4_arms(frames, reps, psnr_frames, mb_frames, tmp):
    """gop 1 / 30, search 0 / 16, qp 20 / 26, intra4x4 off / on, alternating in the timed loop: encode ms, bytes per
    frame, luma PSNR; with mb_frames, the restatement's macroblock shares, mode histogram and c sweep."""
    arms = [(g, s, q, i4) for g, s in ((1, 0), (30, 0), (30, 16)) for q in (20, 26) for i4 in (False, True)]
    ms = {a: [] for a in arms}
    for g, s, q, i4 in arms:
        video.encode(frames, qp=q, gop=g, search=s, intra4x4=i4)   # warm-up
    torch.cuda.synchronize()
    for _ in range(reps):
        for g, s, q, i4 in arms:
            ms[(g, s, q, i4)].append(event_ms(lambda: video.encode(frames, qp=q, gop=g, search=s, intra4x4=i4)))
    out = {}
    clip = frames[0] if frames.dim() == 5 else frames
    for g, s, q, i4 in arms:
        sizes = video.encode(frames, qp=q, gop=g, search=s, intra4x4=i4)[1].cpu().numpy()
        path = video.write_mp4(clip, os.path.join(tmp, f"g{g}s{s}q{q}i{int(i4)}.mp4"), fps=30, qp=q, gop=g, search=s,
                               intra4x4=i4)
        psnr_mean, psnr_min = luma_psnr(clip, path, psnr_frames)
        a = out[f"gop{g}_search{s}_qp{q}_i4{int(i4)}"] = {
            "encode_ms_median": statistics.median(ms[(g, s, q, i4)]), "encode_ms_all": ms[(g, s, q, i4)],
            "bytes_per_frame_mean": float(sizes.mean()), "bytes_per_frame_min": int(sizes.min()),
            "bytes_per_frame_max": int(sizes.max()), "luma_psnr_db_mean": psnr_mean, "luma_psnr_db_min": psnr_min}
        print("  arm", g, s, q, i4, json.dumps({k: v for k, v in a.items() if k != "encode_ms_all"}), flush=True)
    if mb_frames:
        import h264_ref
        host = list(clip[:mb_frames].cpu().numpy())
        for q in (20, 26):
            enc = h264_ref.encode_clip(host, q, 30, 0, True)
            assert [e[0] for e in enc] == [bytes(x) for x in _first_samples(clip[:mb_frames], 30, 0, q, True)]
            types = np.concatenate([e[2].reshape(-1) for e in enc])
            modes = np.concatenate([e.modes[e.types == "I4"].reshape(-1) for e in enc])
            sweep = {}
            for c in (0, 3, 6, 12, 24):
                sweep[c] = [len(e[0]) for e in h264_ref.encode_clip(host, q, 30, 0, True, c)]
            out[f"restatement_qp{q}"] = {
                "frames": mb_frames, "c": h264_ref.C_I4,
                "mb_share": {k: float((types == k).mean()) for k in ("SKIP", "P", "DC", "H", "I4", "PCM")},
                "mode_histogram": np.bincount(modes, minlength=9).tolist(),
                "bytes_by_c": sweep, "bytes_without_i4": [len(e[0]) for e in h264_ref.encode_clip(host, q, 30, 0)]}
            print("  restatement", q, json.dumps(out[f"restatement_qp{q}"]), flush=True)
    return out


def run_i4(args, r, pred, res, tmp):
    frames = r.render_sequence(*(pred[k][:1] for k in ("motion_axis_angle", "expression", "trans")))
    print("i4 emage", flush=True)
    res["i4_emage_sequence_1x300"] = i4_arms(frames, args.reps, args.psnr_frames, args.i4_mb_frames, tmp)
    del frames
    camn = build_lstm_product("camn", device="cuda")
    poses = camn(torch.from_numpy(synth_audio(1, 160000, 5)).cuda(),
                 torch.zeros(1, 1, dtype=torch.long, device="cuda"))["motion_axis_angle"]
    poses = poses.reshape(1, poses.shape[1], 165)
    frames = r.render_body(poses, torch.zeros(1, poses.shape[1], 3, device="cuda"), upsample=2)
    print("i4 camn", flush=True)
    res["i4_camn_body_1x10s"] = i4_arms(frames, args.reps, args.psnr_frames, 0, tmp)


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


def run(args, r, pred, res, tmp):
    """Every arm main() asks for, into res; tmp: a scratch directory for the MP4 files, removed by main()."""
    for clips in (1, 8):
        frames = r.render_sequence(*(pred[k][:clips] for k in ("motion_axis_angle", "expression", "trans")))
        res[f"gop_emage_sequence_{clips}x300"] = gop_arms(frames, args.reps, args.psnr_frames,
                                                          clips == 1 and not args.no_mb_types, tmp)
        print("gop emage", clips, json.dumps(res[f"gop_emage_sequence_{clips}x300"]), flush=True)
        if args.baseline_lib:
            res[f"baseline_emage_sequence_{clips}x300"] = baseline(frames, args.baseline_lib, args.reps)
            print("baseline", clips, json.dumps(res[f"baseline_emage_sequence_{clips}x300"])[:700], flush=True)
        if args.gop_only:
            del frames
            continue
        res[f"emage_sequence_{clips}x300"] = arm(frames, args.reps)
        print("emage", clips, json.dumps(res[f"emage_sequence_{clips}x300"])[:700], flush=True)
        if clips == 1:
            qtmp = os.path.join(tmp, "quality")
            os.makedirs(qtmp)
            res["emage_quality"] = quality(frames[0], args.psnr_frames, qtmp)
            print("quality", json.dumps(res["emage_quality"]), flush=True)
        del frames
    camn = build_lstm_product("camn", device="cuda")
    poses = camn(torch.from_numpy(synth_audio(1, 160000, 5)).cuda(),
                 torch.zeros(1, 1, dtype=torch.long, device="cuda"))["motion_axis_angle"]
    poses = poses.reshape(1, poses.shape[1], 165)
    frames = r.render_body(poses, torch.zeros(1, poses.shape[1], 3, device="cuda"), upsample=2)
    res["gop_camn_body_1x10s"] = gop_arms(frames, args.reps, args.psnr_frames, False, tmp)
    print("gop camn", json.dumps(res["gop_camn_body_1x10s"]), flush=True)
    if not args.gop_only:
        res["camn_body_1x10s"] = arm(frames, args.reps)
        print("camn", json.dumps(res["camn_body_1x10s"])[:700], flush=True)
    del frames
    res["output_stage_gop_1x300"] = output_stage_gop(r, pred, args.stage_reps)
    print("output stage gop", json.dumps(res["output_stage_gop_1x300"]), flush=True)
    if not args.gop_only:
        res["output_stage_1x300"] = output_stage(r, pred, args.stage_reps)
        print("output stage", json.dumps(res["output_stage_1x300"]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stage-reps", type=int, default=3)
    ap.add_argument("--psnr-frames", type=int, default=30)
    ap.add_argument("--no-mb-types", action="store_true", help="skip the macroblock shares (CPU restatement)")
    ap.add_argument("--baseline-lib", default=None,
                    help="libpm_emage.so of another build to time pm_h264_encode against")
    ap.add_argument("--gop-only", action="store_true", help="only the GOP arms and the gop output stage")
    ap.add_argument("--me-only", action="store_true", help="only the motion search arms and their output stage")
    ap.add_argument("--me-mb-frames", type=int, default=4, help="frames the restatement counts macroblocks over")
    ap.add_argument("--i4-only", action="store_true", help="only the Intra 4x4 arms")
    ap.add_argument("--i4-mb-frames", type=int, default=2, help="frames the Intra 4x4 restatement counts over")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the video benchmark measures the GPU: no CUDA device found"
    torch.cuda.set_device(0)
    model, vqm = build_product(seed=0, device="cuda")
    _, pred = generate(model, vqm, torch.from_numpy(synth_audio(8, 160000, 5)).cuda())
    r = MeshRenderer(SmplxBodyModel(smplx_surface_arrays(), "cuda"))
    res = {"card": card()}
    tmp = tempfile.mkdtemp()
    try:
        (run_i4 if args.i4_only else run_me if args.me_only else run)(args, r, pred, res, tmp)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    res["card_after"] = card()
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
