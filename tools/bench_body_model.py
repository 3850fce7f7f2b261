#!/usr/bin/env python
"""SMPL-X body model throughput on one GPU: one EMAGE batch (32 clips x 300 frames) on the full-size synthetic model.

    python tools/bench_body_model.py OUT.json [--clips 32] [--frames 300] [--reps 5]

Arms, timed with CUDA events after a warm-up of every shape, alternated over --reps rounds (medians reported):
  joints      body_model.forward(vertices=False): the FK kernel alone
  fk          the FK kernel with vertices requested (also writes A and the GEMM operand planes)
  gemm_<p>    the vertex blend GEMM (rows x 886) @ (886 x 3V) in precision p; TFLOP/s from 2 rows 886 3V against the
              989 TFLOP/s dense fp16/bf16 data-sheet figure (fp16x3 issues 3 MMAs per product, bf16x6 6: the tensor cores
              execute that multiple of the useful FLOP) or the 67 TFLOP/s fp32 figure
  skin        pm_smplx_skin_f32; GB/s from 24 B per vertex-frame (read v_posed, write vertices) against 3.35 TB/s
  forward     forward(vertices=True) end to end, frames/s
  motion_rep  body_model.motion_rep
  torch_eager the float32 restatement (oracle/smplx_oracle.py: Python FK loop, dense matmuls; how an `smplx` user runs it)
The card's name and power limit are read in the same run.  The model is generated at run time (nothing is written
except OUT)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.smplx_oracle import SmplxRestatement, forward_poses  # noqa: E402
from pantomatrix_b200 import ops  # noqa: E402
from pantomatrix_b200.body_model import ALL_JOINTS, SmplxBodyModel  # noqa: E402
from pantomatrix_b200.emage_audio import engine  # noqa: E402
from synthetic_models import SMPLX_FULL_VERTS, smplx_arrays  # noqa: E402

PEAK_TC, PEAK_F32, PEAK_BW = 989e12, 67e12, 3.35e12
MMAS = {"fp16x3": 3, "bf16x6": 6, "fp32": 1}


def card():
    """Name, power limit and max SM clock of the device the run uses (selected by UUID: a host may hold cards set to
    different power limits)."""
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"]
    out = subprocess.run(q + [f"--id=GPU-{torch.cuda.get_device_properties(0).uuid}"], capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "name_power_limit_max_sm_clock": out.stdout.strip() or None}


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--clips", type=int, default=32)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the body model benchmark needs a GPU"
    B, T = args.clips, args.frames
    rows, nv = B * T, SMPLX_FULL_VERTS
    arrays = smplx_arrays(nv)
    bm = SmplxBodyModel(arrays, "cuda")
    eager = SmplxRestatement(arrays, torch.float32).cuda()
    rng = np.random.default_rng(0)
    f = lambda x: torch.from_numpy(np.asarray(x, np.float32)).cuda()
    poses = f(rng.normal(0, 0.5, (B, T, 165)))
    betas, expr, transl = f(rng.normal(0, 1, (B, 300))), f(rng.normal(0, 1, (B, T, 100))), f(rng.normal(0, 1, (B, T, 3)))
    flat = lambda x, c: x.reshape(-1, c)
    betas_rows = betas[:, None].expand(B, T, 300).reshape(-1, 300)

    arms = {
        "joints": (lambda: bm.forward(poses, betas, expr, transl), 50),
        "motion_rep": (lambda: bm.motion_rep(poses), 50),
        "forward": (lambda: bm.forward(poses, betas, expr, transl, vertices=True), 10),
        "torch_eager": (lambda: forward_poses(eager, flat(poses, 165), betas_rows, flat(expr, 100), flat(transl, 3)), 2),
    }
    state = {}

    def fk():
        state["fk"] = bm._fk(poses, betas, expr, transl, ALL_JOINTS, True)

    def gemm():
        state["v"] = bm._blend(state["fk"][2], rows)

    def skin():
        ops.smplx_skin(state["v"], nv, bm.skin_csr, state["fk"][1], transl, T)

    arms.update({"fk": (fk, 50), "gemm_fp16x3": (gemm, 10), "skin": (skin, 20)})
    for fn, _ in arms.values():            # warm-up: module load, weight packing, allocator
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.reps):
        for k, (fn, iters) in arms.items():
            times[k].append(timed(fn, iters))
    med = {k: statistics.median(v) for k, v in times.items()}
    spread = {k: (min(v), max(v)) for k, v in times.items()}
    # the GEMM in the other engine precisions (same operand format as each precision's FK output)
    for p in ("bf16x6", "fp32"):
        engine.set_precision(p)
        fk()
        gemm()
        torch.cuda.synchronize()
        med["gemm_" + p] = statistics.median(timed(gemm, 3 if p == "fp32" else 10) for _ in range(3))
    engine.set_precision("fp16x3")
    flop = 2.0 * rows * 886 * 3 * nv
    res = {
        "card": card(), "clips": B, "frames": T, "rows": rows, "n_verts": nv, "gemm_flop": flop,
        "seconds_median": med, "seconds_min_max": spread,
        "joints_frames_per_s": rows / med["joints"],
        "forward_vertices_frames_per_s": rows / med["forward"],
        "torch_eager_frames_per_s": rows / med["torch_eager"],
        "speedup_vs_torch_eager": med["torch_eager"] / med["forward"],
        "gemm_tflops": {p: flop / med["gemm_" + p] / 1e12 for p in MMAS},
        "gemm_share_of_peak": {p: flop / med["gemm_" + p] / (PEAK_F32 if p == "fp32" else PEAK_TC) for p in MMAS},
        "gemm_mmas_per_product": MMAS,
        "skin_gb_per_s": 24.0 * rows * nv / med["skin"] / 1e9,
        "skin_share_of_hbm": 24.0 * rows * nv / med["skin"] / PEAK_BW,
    }
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
