"""Where the time of one pm_tapgemm_tc launch goes: per-CTA clock64 stamps from the instrumented build.

    python -m pantomatrix_b200.build --variant timing -DPM_TC_TIMING
    PM_EMAGE_LIB=pantomatrix_b200/csrc/_build/variants/libpm_emage_timing.so python tools/gemm_timeline.py

Stamps, one set per CTA (= per output tile), written by the first consumer warp (cycles of the CTA's SM clock, relative
to kernel entry of that CTA): prologue done, first operand stage landed, all MMAs issued, accumulators complete, this
warp's epilogue issued, all consumer warps done.  The launch uses the automatically chosen N tile.  The launch-to-launch
period (CUDA events around a replayed graph of 20 launches) minus the in-kernel span is launch / drain / tail cost.
The first line printed is the card record."""
import ctypes
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from measure import card, graph_us  # noqa: E402
from pantomatrix_b200 import _lib, ops  # noqa: E402

SHAPES = [  # name, batch, rows, cin, cout, taps, pad, fp32 residual
    ("lin 2048x768x64", 1, 2048, 64, 768, 1, 0, False),
    ("lin 2048x768x768", 1, 2048, 768, 768, 1, 0, False),
    ("lin 2048x768x3072", 1, 2048, 3072, 768, 1, 0, False),
    ("lin 2048x2304x768", 1, 2048, 768, 2304, 1, 0, False),
    ("conv k3 32x64 256->256", 32, 64, 256, 256, 3, 1, False),
    ("conv k15 128x1241 64->64", 128, 1241, 64, 64, 15, 7, False),
    # with a residual, as the decoder layers' sa.out / ca.out / l2 and every WavEncoder conv2 run them
    ("lin 2048x768x768 +res", 1, 2048, 768, 768, 1, 0, True),
    ("lin 2048x768x1536 +res", 1, 2048, 1536, 768, 1, 0, True),
    ("lin 2048x2304x768 +res", 1, 2048, 768, 2304, 1, 0, True),
    ("conv k15 32x32638 64->64 +res", 32, 32638, 64, 64, 15, 7, True),   # WavEncoder block 0 conv2, 10 s clips
]
NAMES = ["prologue", "first stage", "mma issued", "acc ready", "epilogue w2", "all done"]


def main():
    lib = _lib.load()
    if not hasattr(lib, "pm_tc_timing_read"):
        sys.exit("not an instrumented build: set PM_EMAGE_LIB to the -DPM_TC_TIMING variant")
    lib.pm_tc_timing_read.argtypes = [ctypes.c_void_p]
    buf = np.zeros((4096, 8), dtype=np.uint64)
    print("card", json.dumps(card()))
    print(f"{'shape':28s} ns out  CTAs | cycles after entry (mean over CTAs): " + " | ".join(NAMES) +
          " || span max (cyc) | period us | span us @period clock")
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    fp16 = len(sys.argv) > 2 and sys.argv[2] == "fp16"          # the default engine: two fp16 planes
    if fp16:
        ops.set_plane_format("fp16")
    for name, b, rows, cin, cout, taps, pad, with_res in SHAPES:
        if only and only not in name:
            continue
        g = torch.Generator().manual_seed(0)
        x = torch.randn(b, rows, cin, generator=g).cuda()
        w = (torch.randn(taps, cout, cin, generator=g) / math.sqrt(cin * taps)).cuda()
        bias = torch.zeros(cout, device="cuda")
        rows_out = rows + 2 * pad - taps + 1
        res = torch.randn(b, rows_out, cout, generator=g).cuda() if with_res else None
        for ns in ((2,) if fp16 else (1, 3)):
            a, pw = ops.split_bf16(x, ns), ops.PackedW(w, ns)
            for out_mode in ("f32", "f+p", "p"):
                kw = dict(rows_out=rows_out, pad=pad, act=ops.ACT_RELU, residual=res,
                          out_nsplit=0 if out_mode == "f32" else ns)
                if out_mode == "p":
                    kw["want_f32"] = False
                else:
                    kw["out"] = torch.empty(b, rows_out, cout, device="cuda")
                period_us, graph = graph_us(lambda: ops.tapgemm_tc(a, pw, bias, **kw))
                assert lib.pm_tc_timing_reset() == 0
                graph.replay()                                  # stamps of the last (warm, back-to-back) launch survive
                assert lib.pm_tc_timing_read(buf.ctypes.data) == 0
                del graph                                       # free its memory pool before the next shape's capture
                st = buf[buf[:, 0] != 0].astype(np.int64)
                d = st[:, 1:7] - st[:, :1]
                span = d[:, 5]
                sm_mhz = _sm_clock_mhz()
                print(f"{name:28s} {ns:2d} {out_mode:>4s} {len(st):5d} | " + " | ".join(f"{v:8.0f}" for v in d.mean(0)) +
                      f" || {span.max():8d} | {period_us:7.2f} | {span.mean() / sm_mhz:6.2f} (SM {sm_mhz:.0f} MHz)")


def _sm_clock_mhz():
    try:
        import pynvml
        pynvml.nvmlInit()
        return float(pynvml.nvmlDeviceGetClockInfo(pynvml.nvmlDeviceGetHandleByIndex(0), pynvml.NVML_CLOCK_SM))
    except Exception:
        return 1920.0


if __name__ == "__main__":
    main()
