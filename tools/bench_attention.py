#!/usr/bin/env python
"""Microbenchmark of the attention kernels on the EMAGE shape (32 clips x 4 heads, T = 64, head_dim 192), warm L2:
CUDA events around 5 CUDA-graph replays of 20 back-to-back launches (GPU time, not launch / descriptor-encode time).
The first line printed is the card record.
    python tools/bench_attention.py"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from measure import card, graph_us  # noqa: E402
from pantomatrix_b200 import ops  # noqa: E402


def main():
    print("card", json.dumps(card()))
    bs, t, E, H, hd = 32, 64, 768, 4, 192
    g = torch.Generator().manual_seed(0)
    qkv = torch.randn(bs, t, 3 * E, generator=g).cuda()
    flop = 4.0 * bs * t * t * E
    us = graph_us(lambda: ops.attention(qkv.view(bs * t, 3 * E)[:, :E], qkv.view(bs * t, 3 * E)[:, E:2 * E], qkv.view(bs * t, 3 * E)[:, 2 * E:],
                                        bs, H, t, t, hd), replays=5)[0]
    print(f"attention_f32_kernel (fp32 SIMT)      {us:7.2f} us  {flop / us / 1e6:7.1f} TFLOP/s algorithmic")
    ops.set_plane_format("fp16")
    qp = ops.split_bf16(qkv, 2)
    for f32 in (False, True):
        us = graph_us(lambda: ops.attention_tc(qp, 0, qp, E, qp, 2 * E, bs, H, t, t, hd, nsplit=2, f32=f32), replays=5)[0]
        print(f"attention_tc_kernel planes{'+fp32' if f32 else '     '} out  {us:7.2f} us  {flop / us / 1e6:7.1f} TFLOP/s algorithmic "
              f"({3 * flop / us / 1e6:7.1f} of fp16 MMA work)")
    if "--timeline" in sys.argv:          # instrumented build: python -m pantomatrix_b200.build --variant attn_timing -DPM_ATTN_TIMING
        import ctypes
        from pantomatrix_b200 import _lib
        ops.attention_tc(qp, 0, qp, E, qp, 2 * E, bs, H, t, t, hd, nsplit=2)
        buf = (ctypes.c_ulonglong * 16)()
        assert _lib.load().pm_attn_timing_read(buf) == 0
        v = list(buf)
        names = ["entry", "prologue done", "S complete (warp 0)", "softmax done, P stored", "O complete", "outputs written", "-",
                 "all warps done", "Q|K block 0 landed", "block 1", "block 2"]
        for i, n in enumerate(names):
            print(f"  {n:28s} +{(v[i] - v[0]):7d} cycles")
    ops.set_plane_format("bf16")


if __name__ == "__main__":
    main()
