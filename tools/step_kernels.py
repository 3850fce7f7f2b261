"""Where the time of one EMAGE step goes, per kernel: one warmed eager step (32 clips x 10 s, fp16x3 unless a precision
is given) under torch.profiler with CUDA activities.

    python tools/step_kernels.py OUT [precision]

Writes OUT/step_kernels.txt (kernel name, launches, total and mean device time, share of the summed kernel time) and
prints the card record, the step's wall time, the summed kernel time and the tap-GEMM's share of it.  Eager launches
on forked streams overlap, so the summed kernel time is busy time and can exceed the wall time; the share is of
the summed kernel time.  The profiler adds host overhead: take step times from bench.py, not from here."""
import os
import sys
import time
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from measure import card  # noqa: E402
from synthetic_models import build_product  # noqa: E402
from oracle.weights import synth_audio  # noqa: E402
from pantomatrix_b200.emage_audio import engine  # noqa: E402
from pantomatrix_b200.pipeline import generate  # noqa: E402


def main():
    if len(sys.argv) < 2:
        sys.exit(__doc__)
    out_dir = sys.argv[1]
    precision = sys.argv[2] if len(sys.argv) > 2 else "fp16x3"
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    os.makedirs(out_dir, exist_ok=True)
    engine.set_precision(precision)
    model, vqm = build_product(0)
    audio = torch.from_numpy(synth_audio(32, 160000, 1234)).cuda()
    for _ in range(2):                      # warm-up: weight packing, function attributes, allocator
        generate(model, vqm, audio)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        generate(model, vqm, audio)
        torch.cuda.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1e3
    per = defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time_total > 0:
            per[ev.name][0] += 1
            per[ev.name][1] += ev.device_time_total / 1e3            # ms
    total = sum(t for _, t in per.values())
    rows = sorted(per.items(), key=lambda kv: -kv[1][1])
    with open(os.path.join(out_dir, "step_kernels.txt"), "w") as f:
        f.write(f"# one eager EMAGE step, 32 x 10 s, {precision}; card {card()}\n")
        f.write(f"# wall {wall_ms:.2f} ms (profiled), summed kernel time {total:.2f} ms\n")
        f.write(f"{'ms':>9s} {'launches':>8s} {'us/launch':>9s} {'share':>6s}  kernel\n")
        for name, (n, t) in rows:
            f.write(f"{t:9.3f} {n:8d} {t / n * 1e3:9.2f} {t / total:6.1%}  {name}\n")
    tap = sum(t for name, (_, t) in per.items() if "tapgemm_tc_kernel" in name)
    print("card", card())
    print(f"{precision}: profiled eager step {wall_ms:.2f} ms, summed kernel time {total:.2f} ms, "
          f"tap-GEMM {tap:.2f} ms = {tap / total:.1%} of it ({sum(n for name, (n, _) in per.items() if 'tapgemm_tc_kernel' in name)} launches)")
    print(f"table: {os.path.join(out_dir, 'step_kernels.txt')}")


if __name__ == "__main__":
    main()
