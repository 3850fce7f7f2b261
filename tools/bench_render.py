#!/usr/bin/env python
"""SMPL-X mesh render throughput on one GPU (pantomatrix_b200/render.py).

    python tools/bench_render.py OUT.json [--reps 5] [--arms surface,soup,camn_body,emage_pair]

Inputs: EMAGE generate() pose outputs (synthetic weights) for one 10 s clip (300 frames) and for 8 x 300 frames, on two
full-size (10 475-vertex) synthetic models:
  surface  synthetic_models.smplx_surface_arrays: closed capsules with body-like triangle sizes (the headline)
  soup     synthetic_models.smplx_arrays: 20 950 random vertex triples spanning the body (a worst case)
and, on the surface model, the other two layouts:
  camn_body  render_body(upsample=2) of CaMN forward() output (synthetic weights, 15 fps) for 1 x 10 s and 8 x 10 s:
             150 frames per clip upsampled to 300, one 480 x 720 view per frame
  emage_pair render_pair of the EMAGE clips, each beside the next clip as its ground truth, 1 and 8 clips
Reported, from CUDA events after a warm-up of every shape (medians over --reps):
  the layout's call end to end (frames/s), and the share of it taken by the body-model calls (render_sequence: body
  and jaw-only; render_pair: both sides; render_body: one) and, for render_body, by the upsampling kernel;
  per kernel, the median time per 8-frame chunk, and the least bytes it must move against the 3.35 TB/s HBM3 figure:
    vertex  read xyz (12 B), write snapped xy, depth and normal (24 B) per vertex and view
    raster  read each view's xy and depth (12 B per vertex) and the faces (12 B per triangle)
    shade   read the 8-byte visibility key, write 3 bytes of RGB per pixel and view
There is no reference arm: the reference renders with pyrender, which is not installed, so no comparison is made.
The card's name and power limit are read in the same run.  Nothing is written except OUT."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.weights import synth_audio  # noqa: E402
from pantomatrix_b200 import ops  # noqa: E402
from pantomatrix_b200.body_model import ALL_JOINTS, SmplxBodyModel  # noqa: E402
from pantomatrix_b200.pipeline import generate  # noqa: E402
from pantomatrix_b200.render import CHUNK, FACE_VIEW, BODY_VIEW, H, JAW_ONLY, VIEWS, W, MeshRenderer  # noqa: E402
from synthetic_models import (SMPLX_FULL_VERTS, build_lstm_product, build_product, smplx_arrays,  # noqa: E402
                              smplx_surface_arrays)

PEAK_BW = 3.35e12
SOUP_BUDGET_S = 5.0       # the soup's 8-clip run is skipped when one clip already takes longer than this


def card():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
    out = subprocess.run(q + [f"--id=GPU-{torch.cuda.get_device_properties(0).uuid}"], capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "name_power_limit_max_sm_clock": out.stdout.strip() or None}


def event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def kernels(r, verts, views, reps):
    """Median ms per chunk of each kernel over every chunk of the sequence (the memset is counted with raster); verts
    and views hold one entry per image view."""
    nv, n, nviews = r.n_verts, verts[0].shape[0], len(verts)
    xy = torch.empty(CHUNK, nviews, nv, 2, dtype=torch.int32, device="cuda")
    depth = torch.empty(CHUNK, nviews, nv, device="cuda")
    normal = torch.empty(CHUNK, nviews, nv, 3, device="cuda")
    vis = torch.empty(CHUNK, nviews, H, W, dtype=torch.int64, device="cuda")
    out = torch.empty(CHUNK, H, nviews * W, 3, dtype=torch.uint8, device="cuda")
    times = {"vertex": [], "raster": [], "shade": []}
    for _ in range(reps):
        for s in range(0, n - CHUNK + 1, CHUNK):
            v = [x[s:s + CHUNK] for x in verts]
            times["vertex"].append(event_ms(lambda: ops.mesh_vertex(v, views, r.faces, r.vf_csr, xy, depth, normal)))
            times["raster"].append(event_ms(lambda: ops.mesh_raster(xy, depth, r.faces, vis)))
            times["shade"].append(event_ms(lambda: ops.mesh_shade(vis, xy, normal, r.faces, out)))
    nf = r.n_faces
    least = {"vertex": CHUNK * nviews * nv * 36, "raster": CHUNK * nviews * (nv * 12 + nf * 12),
             "shade": CHUNK * nviews * H * W * 11}
    res = {}
    for k, t in times.items():
        med = statistics.median(t)
        res[k] = {"ms_per_chunk_median": med, "ms_per_chunk_max": max(t), "least_bytes_per_chunk": least[k],
                  "share_of_3.35TBps": least[k] / (med * 1e-3) / PEAK_BW}
    return res


def arm(name, arrays, pred, clips, reps):
    bm = SmplxBodyModel(arrays, "cuda")
    r = MeshRenderer(bm)
    poses, expr, trans = (pred[k][:clips] for k in ("motion_axis_angle", "expression", "trans"))
    n = poses.shape[1] // 30 * 30
    out = torch.empty(clips, n, H, VIEWS * W, 3, dtype=torch.uint8, device="cuda")
    t0 = time.time()
    r.render_sequence(poses, expr, trans, out=out)                  # warm-up (packs the body model's weights)
    torch.cuda.synchronize()
    first_s = time.time() - t0
    if name == "soup" and clips > 1 and first_s > SOUP_BUDGET_S * clips:
        return {"skipped": f"one warm-up call took {first_s:.1f} s"}
    reps = 1 if name == "soup" else reps
    p, e, tr = poses[:, :n], expr[:, :n], trans[:, :1].expand(clips, n, 3)
    e2e = [event_ms(lambda: r.render_sequence(poses, expr, trans, out=out)) for _ in range(reps)]
    bmt = [event_ms(lambda: (bm._vertices(p, None, e, tr, ALL_JOINTS), bm._vertices(p, None, e, tr, JAW_ONLY)))
           for _ in range(reps)]
    face = bm._vertices(p, None, e, tr, JAW_ONLY)[1].view(clips * n, -1, 3)
    body = bm._vertices(p, None, e, tr, ALL_JOINTS)[1].view(clips * n, -1, 3)
    med = statistics.median(e2e)
    return {"clips": clips, "frames_per_clip": n, "render_sequence_ms_median": med,
            "render_sequence_ms_all": e2e, "frames_per_s": clips * n / (med * 1e-3),
            "body_model_ms_median": statistics.median(bmt), "body_model_share": statistics.median(bmt) / med,
            "triangles": r.n_faces, "kernels": kernels(r, [face, body], (FACE_VIEW, BODY_VIEW), reps)}


def body_arm(bm, r, poses, clips, reps):
    """render_body(upsample=2) of 15 fps poses (clips, t, 165) with the pelvis at the origin."""
    poses = poses[:clips]
    t = poses.shape[1]
    n = 2 * t // 30 * 30
    trans = torch.zeros(clips, t, 3, device="cuda")
    out = torch.empty(clips, n, H, W, 3, dtype=torch.uint8, device="cuda")
    r.render_body(poses, trans, upsample=2, out=out)                # warm-up
    torch.cuda.synchronize()
    e2e = [event_ms(lambda: r.render_body(poses, trans, upsample=2, out=out)) for _ in range(reps)]
    up = [event_ms(lambda: ops.time_upsample(poses, 2)) for _ in range(reps)]
    p = ops.time_upsample(poses, 2)[:, :n]
    tr = trans[:, :1].expand(clips, n, 3)
    bmt = [event_ms(lambda: bm._vertices(p, None, None, tr, ALL_JOINTS)) for _ in range(reps)]
    body = bm._vertices(p, None, None, tr, ALL_JOINTS)[1].view(clips * n, -1, 3)
    med = statistics.median(e2e)
    return {"clips": clips, "frames_per_clip_15fps": t, "frames_per_clip": n, "render_body_ms_median": med,
            "render_body_ms_all": e2e, "frames_per_s": clips * n / (med * 1e-3),
            "time_upsample_ms_median": statistics.median(up), "time_upsample_share": statistics.median(up) / med,
            "body_model_ms_median": statistics.median(bmt), "body_model_share": statistics.median(bmt) / med,
            "triangles": r.n_faces, "kernels": kernels(r, [body], (BODY_VIEW,), reps)}


def pair_arm(bm, r, pred, clips, reps):
    """render_pair of EMAGE clips, clip i beside clip i+1 (mod 8) as its ground truth."""
    keys = ("motion_axis_angle", "trans", "expression")
    p, tr, e = (pred[k][:clips] for k in keys)
    gp, gtr, ge = (torch.roll(pred[k], -1, 0)[:clips].contiguous() for k in keys)
    n = p.shape[1] // 30 * 30
    out = torch.empty(clips, n, H, 2 * W, 3, dtype=torch.uint8, device="cuda")
    call = lambda: r.render_pair(p, tr, gp, gtr, e, None, ge, None, out=out)
    call()                                                          # warm-up
    torch.cuda.synchronize()
    e2e = [event_ms(call) for _ in range(reps)]
    sides = [(x[:, :n], y[:, :n], z[:, :1].expand(clips, n, 3)) for x, y, z in ((p, e, tr), (gp, ge, gtr))]
    bmt = [event_ms(lambda: [bm._vertices(a, None, b, c, ALL_JOINTS) for a, b, c in sides]) for _ in range(reps)]
    verts = [bm._vertices(a, None, b, c, ALL_JOINTS)[1].view(clips * n, -1, 3) for a, b, c in sides]
    med = statistics.median(e2e)
    return {"clips": clips, "frames_per_clip": n, "render_pair_ms_median": med, "render_pair_ms_all": e2e,
            "frames_per_s": clips * n / (med * 1e-3), "body_model_ms_median": statistics.median(bmt),
            "body_model_share": statistics.median(bmt) / med, "triangles": r.n_faces,
            "kernels": kernels(r, verts, (BODY_VIEW, BODY_VIEW), reps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--arms", default="surface,soup,camn_body,emage_pair", help="comma-separated subset to run")
    args = ap.parse_args()
    arms = args.arms.split(",")
    assert torch.cuda.is_available(), "the render benchmark measures the GPU: no CUDA device found"
    torch.cuda.set_device(0)
    model, vqm = build_product(seed=0, device="cuda")
    _, pred = generate(model, vqm, torch.from_numpy(synth_audio(8, 160000, 5)).cuda())
    res = {"card": card(), "reference_arm": "none: pyrender is not installed, so the reference is not measured",
           "frames_per_clip_generated": int(pred["motion_axis_angle"].shape[1])}
    for name, arrays in (("surface", smplx_surface_arrays()), ("soup", smplx_arrays(SMPLX_FULL_VERTS))):
        for clips in (1, 8) if name in arms else ():
            res[f"{name}_{clips}x300"] = arm(name, arrays, pred, clips, args.reps)
            print(name, clips, json.dumps(res[f"{name}_{clips}x300"])[:400], flush=True)
    camn = build_lstm_product("camn", device="cuda")
    audio = torch.from_numpy(synth_audio(8, 160000, 5)).cuda()
    camn_poses = camn(audio, torch.zeros(8, 1, dtype=torch.long, device="cuda"))["motion_axis_angle"]
    camn_poses = camn_poses.reshape(8, camn_poses.shape[1], 165)
    bm = SmplxBodyModel(smplx_surface_arrays(), "cuda")
    r = MeshRenderer(bm)
    for clips in (1, 8):
        if "camn_body" in arms:
            res[f"camn_body_{clips}x10s"] = body_arm(bm, r, camn_poses, clips, args.reps)
            print("camn_body", clips, json.dumps(res[f"camn_body_{clips}x10s"]), flush=True)
        if "emage_pair" in arms:
            res[f"emage_pair_{clips}x300"] = pair_arm(bm, r, pred, clips, args.reps)
            print("emage_pair", clips, json.dumps(res[f"emage_pair_{clips}x300"]), flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
