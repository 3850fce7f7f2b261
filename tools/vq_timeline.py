#!/usr/bin/env python
"""Per-phase cycle counts of the tensor-core VQ lookup kernel (CTA 0) from an instrumented build:

    python -m pantomatrix_b200.build --variant vq_timing -DPM_VQ_TIMING     # on the build host
    PM_EMAGE_LIB=$PWD/pantomatrix_b200/csrc/_build/variants/libpm_emage_vq_timing.so python tools/vq_timeline.py
"""
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NAMES = ["loader: load + reduce (warp 8)", "loader: wait a_empty", "loader: convert + store", "-", "consumer: wait a_full (warp 0)",
         "-", "-", "consumer: MMAs + pass 1", "consumer: pass 2", "consumer: re-score + store", "kernel total (warp 0)", "tiles",
         "re-scored rows (warp 0)", "-"]


def main(rows=1 << 21):
    import torch
    from pantomatrix_b200 import _lib, ops
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(0)
    z = torch.randn(rows, 256, device="cuda", generator=g)
    cb = torch.randn(256, 256, device="cuda", generator=g)
    e2 = ops.row_sqnorm(cb)
    ops.l2_argmin(z, cb, e2, engine="tc")
    assert lib.pm_vq_timing_reset() == 0
    ops.l2_argmin(z, cb, e2, engine="tc")
    buf = (ctypes.c_ulonglong * 16)()
    assert lib.pm_vq_timing_read(buf) == 0
    vals = list(buf)
    tiles = max(vals[11], 1)
    out = {n: {"cycles": v, "per_tile": v / tiles} for n, v in zip(NAMES, vals) if n != "-"}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
