#!/usr/bin/env python
"""VQ-lookup microbenchmark (SURVEY.md section 8d: judged against HBM on >= 10^6 rows).

    python tools/bench_vq.py [--rows 2097152] [--reps 20] [--engine tc|simt|auto]

Algorithmic bytes per row: 1 024 B of fp32 latent read + 8 B of int64 index written (the 256 KB codebook is
amortised).  Inputs (rows x 1 KB) are far larger than the 50 MB L2, so every launch streams from HBM.
Prints one JSON object: rows/s, GB/s, fraction of MEASURED_PEAKS.json's HBM copy bandwidth (`frac` from the median
launch, `frac_best` from the fastest of the 20 - the peak itself is a best-of-10 copy)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BYTES_PER_ROW = 1032


def measure(rows, reps, engine="auto", max_ctas=0, scale=1.0, seed=0):
    import torch
    from pantomatrix_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(rows, 256, device="cuda", generator=g) * scale
    cb = torch.randn(256, 256, device="cuda", generator=g)
    e2 = ops.row_sqnorm(cb)
    for _ in range(3):
        idx = ops.l2_argmin(z, cb, e2, engine=engine, max_ctas=max_ctas)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for s, e in ev:
        s.record()
        ops.l2_argmin(z, cb, e2, engine=engine, max_ctas=max_ctas)
        e.record()
    torch.cuda.synchronize()
    ms = sorted(s.elapsed_time(e) for s, e in ev)
    med = ms[len(ms) // 2]
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
        src = "MEASURED_PEAKS.json hbm_gbs"
    except Exception:
        peak, src = 3350.0, "H100 SXM data sheet (not measured)"
    gbs = rows * BYTES_PER_ROW / (med * 1e-3) / 1e9
    return {"kernel": "l2_argmin_tc_kernel" if engine != "simt" else "l2_argmin_kernel", "engine": engine, "rows": rows,
            "ms": med, "ms_min": ms[0], "rows_per_s": rows / (med * 1e-3), "achieved": gbs, "peak": peak, "unit": "GB/s",
            "frac": gbs / peak, "frac_best": rows * BYTES_PER_ROW / (ms[0] * 1e-3) / 1e9 / peak, "bound": "hbm", "bytes_per_row": BYTES_PER_ROW, "peak_source": src, "reps": reps,
            "index_checksum": int(idx.sum())}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 21)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--engine", default="auto")
    ap.add_argument("--max-ctas", type=int, default=0)
    a = ap.parse_args()
    print(json.dumps(measure(a.rows, a.reps, a.engine, a.max_ctas)))
