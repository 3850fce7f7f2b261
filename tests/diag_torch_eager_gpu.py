"""Diagnostic (not a test): the "library baseline" on the same GPU - the oracle port of the reference run on cuda:0
through stock torch eager kernels (cuDNN convolutions, cuBLAS GEMMs, ATen elementwise), i.e. what a user of the
reference gets by calling `.to("cuda")` (SURVEY §8d "reference-on-GPU" bar).  The unmodified reference cannot travel
to the GPU box, so this times oracle/emage_oracle.py, which restates it op for op with torch.nn.functional calls;
`sdpa=1` swaps its hand-written attention core for F.scaled_dot_product_attention (the fused path
nn.MultiheadAttention takes in eval mode).  Same workload and timed span as bench.py (configs[1]).

    python tests/diag_torch_eager_gpu.py [bs] [runs]   -> JSON lines on stdout."""
import json
import math
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import emage_oracle as O  # noqa: E402
from oracle.weights import make_checkpoint, synth_audio  # noqa: E402


def _mha_sdpa(sd, p, q_in, kv_in, nhead=4):
    E = q_in.shape[-1]
    w, b = sd[p + ".in_proj_weight"], sd[p + ".in_proj_bias"]
    q, k, v = F.linear(q_in, w[:E], b[:E]), F.linear(kv_in, w[E:2 * E], b[E:2 * E]), F.linear(kv_in, w[2 * E:], b[2 * E:])
    bs, tq, _ = q.shape
    split = lambda x: x.reshape(bs, x.shape[1], nhead, E // nhead).transpose(1, 2)
    o = F.scaled_dot_product_attention(split(q), split(k), split(v), scale=1.0 / math.sqrt(E // nhead))
    return O._lin(sd, p + ".out_proj", o.transpose(1, 2).reshape(bs, tq, E))


def to_cuda(x):
    if isinstance(x, torch.Tensor):
        return x.cuda()
    if isinstance(x, dict):
        return {k: to_cuda(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(to_cuda(v) for v in x)
    return x


def main():
    bs = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    runs = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    sd, cfg, vq = make_checkpoint(0)
    sd, vq = to_cuda(sd), to_cuda(vq)
    audio = torch.from_numpy(synth_audio(bs, 160000, 1234)).cuda()
    spk = torch.zeros(bs, 1, dtype=torch.long, device="cuda")
    torch.set_default_device("cuda")            # the oracle creates its scratch tensors with bare factory calls
    stock_mha = O._mha
    frames = bs * (160000 * 30 // 16000)
    for tf32_conv, tf32_mm, sdpa in ((True, False, 0), (True, False, 1), (False, False, 1), (True, True, 1)):
        torch.backends.cudnn.allow_tf32 = tf32_conv          # torch default: True
        torch.backends.cuda.matmul.allow_tf32 = tf32_mm      # torch default: False
        O._mha = _mha_sdpa if sdpa else stock_mha
        with torch.no_grad():
            O.emage_generate(sd, cfg, vq, audio, spk)        # warm-up (cuDNN autotune, allocator)
            torch.cuda.synchronize()
            times = []
            for _ in range(runs):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _, pred = O.emage_generate(sd, cfg, vq, audio, spk)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
        ms = sorted(times)[len(times) // 2]
        print(json.dumps({"impl": "torch-eager port on cuda:0", "bs": bs, "conv_tf32": tf32_conv, "matmul_tf32": tf32_mm,
                          "sdpa": bool(sdpa), "ms_per_step": ms, "frames_per_s": frames / ms * 1e3,
                          "out_frames": int(pred["motion_axis_angle"].shape[1])}), flush=True)
    O._mha = stock_mha


if __name__ == "__main__":
    main()
