"""Microbenchmark of pm_tapgemm_tc on the EMAGE shapes (warm L2, CUDA events around CUDA-graph replays).
    python tools/bench_gemm.py [shape-substring] [fp16]      # fp16: two fp16 planes (the default engine) only
Each shape is timed with the N tile chosen automatically ("auto", the time the engine sees) and forced to 64 and to
128 columns (all three give bit-identical results)."""
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pantomatrix_b200 import ops  # noqa: E402

SHAPES = [  # name, batch, rows, cin, cout, taps, pad
    ("lin 2048x768x64", 1, 2048, 64, 768, 1, 0),
    ("lin 2048x768x256", 1, 2048, 256, 768, 1, 0),
    ("lin 2048x768x768", 1, 2048, 768, 768, 1, 0),
    ("lin 2048x768x1536", 1, 2048, 1536, 768, 1, 0),
    ("lin 2048x768x3072", 1, 2048, 3072, 768, 1, 0),
    ("lin 2048x2304x768", 1, 2048, 768, 2304, 1, 0),
    ("lin 2048x1536x768", 1, 2048, 768, 1536, 1, 0),
    ("lin 1920x768x768 (T=60 window)", 1, 1920, 768, 768, 1, 0),
    ("lin 1920x768x1536", 1, 1920, 1536, 768, 1, 0),
    ("lin 1920x2304x768", 1, 1920, 768, 2304, 1, 0),
    ("lin 1920x1536x768", 1, 1920, 768, 1536, 1, 0),
    ("lin 8192x1536x768 (kv hoist)", 1, 8192, 768, 1536, 1, 0),
    ("lin 10240x1536x768 (kv hoist)", 1, 10240, 768, 1536, 1, 0),
    ("conv k3 32x64 256->256", 32, 64, 256, 256, 3, 1),
    ("conv k3 32x16 256->256 (seed)", 32, 16, 256, 256, 3, 1),
    ("conv k3 32x300 256->256", 32, 300, 256, 256, 3, 1),
    ("conv k15 128x7460 64->64", 128, 7460, 64, 64, 15, 7),
    ("conv k15 128x1241 64->64", 128, 1241, 64, 64, 15, 7),
    ("conv k15 128x205 128->128", 128, 205, 128, 128, 15, 7),
]


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else ""
    fp16 = len(sys.argv) > 2 and sys.argv[2] == "fp16"
    if fp16:
        ops.set_plane_format("fp16")
    print(f"plane format {ops.plane_format()}")
    print(f"{'shape':34s} {'ns':>2s} {'out':>4s} {'us':>9s} {'TFLOP/s(alg)':>13s} {'bf16-equiv':>10s} "
          f"{'us BN=64':>9s} {'us BN=128':>9s}")
    for name, b, rows, cin, cout, taps, pad in SHAPES:
        if only and only not in name:
            continue
        g = torch.Generator().manual_seed(0)
        x = torch.randn(b, rows, cin, generator=g).cuda()
        w = (torch.randn(taps, cout, cin, generator=g) / math.sqrt(cin * taps)).cuda()
        bias = torch.zeros(cout, device="cuda")
        rows_out = rows + 2 * pad - taps + 1
        for ns in ((tuple(int(a) for a in sys.argv[3:]) or (2,)) if fp16 else (1, 2, 3)):
            a = ops.split_bf16(x, ns)
            pw = ops.PackedW(w, ns)
            for out_mode in ("f32", "f+p"):
                kw = dict(rows_out=rows_out, pad=pad, act=ops.ACT_RELU, out_nsplit=ns if out_mode == "f+p" else 0)
                out = torch.empty(b, rows_out, cout, device="cuda")
                kw["out"] = out
                us = {tile: _time(a, pw, bias, tile, kw) for tile in (0, 64, 128) if tile != 128 or pw.w_rows % 128 == 0}
                fl = 2.0 * b * rows_out * cout * cin * taps
                mult = {1: 1, 2: 3, 3: 6}[ns]          # tensor-core products per fp32 product
                print(f"{name:34s} {ns:2d} {out_mode:>4s} {us[0]:9.1f} {fl / us[0] / 1e6:13.1f} {fl * mult / us[0] / 1e6:10.1f} "
                      f"{us[64]:9.1f} {us.get(128, float('nan')):9.1f}")


def _time(a, pw, bias, tile, kw):
    for _ in range(3):
        ops.tapgemm_tc(a, pw, bias, tile=tile, **kw)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()          # 20 back-to-back launches replayed as a graph: GPU time,
    with torch.cuda.graph(graph):           # not Python / ctypes / descriptor-encode time
        for _ in range(20):
            ops.tapgemm_tc(a, pw, bias, tile=tile, **kw)
    graph.replay()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(3):
        graph.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / 60 * 1e3

if __name__ == "__main__":
    main()
