#!/usr/bin/env python
"""SMPL-X mesh render throughput on one GPU (pantomatrix_b200/render.py).

    python tools/bench_render.py OUT.json [--reps 5]

Inputs: EMAGE generate() pose outputs (synthetic weights) for one 10 s clip (300 frames) and for 8 x 300 frames, on two
full-size (10 475-vertex) synthetic models:
  surface  synthetic_models.smplx_surface_arrays: closed capsules with body-like triangle sizes (the headline)
  soup     synthetic_models.smplx_arrays: 20 950 random vertex triples spanning the body (a worst case)
Reported, from CUDA events after a warm-up of every shape (medians over --reps):
  render_sequence end to end (frames/s), and the share of it taken by the two body-model calls (body and jaw-only);
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
from synthetic_models import SMPLX_FULL_VERTS, build_product, smplx_arrays, smplx_surface_arrays  # noqa: E402

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


def kernels(r, face, body, reps):
    """Median ms per chunk of each kernel over every chunk of the sequence (the memset is counted with raster)."""
    nv, n = r.n_verts, face.shape[0]
    xy = torch.empty(CHUNK, VIEWS, nv, 2, dtype=torch.int32, device="cuda")
    depth = torch.empty(CHUNK, VIEWS, nv, device="cuda")
    normal = torch.empty(CHUNK, VIEWS, nv, 3, device="cuda")
    vis = torch.empty(CHUNK, VIEWS, H, W, dtype=torch.int64, device="cuda")
    out = torch.empty(CHUNK, H, VIEWS * W, 3, dtype=torch.uint8, device="cuda")
    times = {"vertex": [], "raster": [], "shade": []}
    for _ in range(reps):
        for s in range(0, n - CHUNK + 1, CHUNK):
            v = [face[s:s + CHUNK], body[s:s + CHUNK]]
            times["vertex"].append(event_ms(lambda: ops.mesh_vertex(v, (FACE_VIEW, BODY_VIEW), r.faces, r.vf_csr, xy,
                                                                    depth, normal)))
            times["raster"].append(event_ms(lambda: ops.mesh_raster(xy, depth, r.faces, vis)))
            times["shade"].append(event_ms(lambda: ops.mesh_shade(vis, xy, normal, r.faces, out)))
    nf = r.n_faces
    least = {"vertex": CHUNK * VIEWS * nv * 36, "raster": CHUNK * VIEWS * (nv * 12 + nf * 12),
             "shade": CHUNK * VIEWS * H * W * 11}
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
            "triangles": r.n_faces, "kernels": kernels(r, face, body, reps)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the render benchmark measures the GPU: no CUDA device found"
    torch.cuda.set_device(0)
    model, vqm = build_product(seed=0, device="cuda")
    _, pred = generate(model, vqm, torch.from_numpy(synth_audio(8, 160000, 5)).cuda())
    res = {"card": card(), "reference_arm": "none: pyrender is not installed, so the reference is not measured",
           "frames_per_clip_generated": int(pred["motion_axis_angle"].shape[1])}
    for name, arrays in (("surface", smplx_surface_arrays()), ("soup", smplx_arrays(SMPLX_FULL_VERTS))):
        for clips in (1, 8):
            res[f"{name}_{clips}x300"] = arm(name, arrays, pred, clips, args.reps)
            print(name, clips, json.dumps(res[f"{name}_{clips}x300"])[:400], flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
