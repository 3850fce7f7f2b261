"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel: count, total, share.
    python tools/summarize_launches.py launches.csv [skip_first_n] > launches.md"""
import csv
import re
import sys
from collections import defaultdict

path = sys.argv[1]
skip = int(sys.argv[2]) if len(sys.argv) > 2 else 0
rows = []
with open(path, newline="") as f:
    lines = [l for l in f if not l.startswith("==")]
for r in csv.DictReader(lines):
    if r.get("Metric Name") == "gpu__time_duration.sum":
        v = float(r["Metric Value"].replace(",", ""))
        unit = r.get("Metric Unit", "ns")
        ns = v * {"ns": 1, "us": 1e3, "usecond": 1e3, "msecond": 1e6, "ms": 1e6, "nsecond": 1}.get(unit, 1)
        rows.append((r["Kernel Name"], ns))
rows = rows[skip:]
agg = defaultdict(lambda: [0, 0.0])
for name, ns in rows:
    head = name.replace("void ", "").replace("<unnamed>::", "")
    m = re.match(r"([\w:]+)(<[\w, ]*>)?", head)
    short = (m.group(1) + (m.group(2) or "")) if m else head[:40]
    if short.startswith("at::"):
        f = re.search(r"at::(\w+(?:Functor|_kernel_cuda|Copy\w*)[\w]*)", name[len(short):])
        short = "torch:" + short.split("::")[-1].split("<")[0] + ("/" + f.group(1) if f else "")
    agg[short][0] += 1
    agg[short][1] += ns
total = sum(v[1] for v in agg.values())
print(f"| kernel | launches | total ms | share |\n|---|---:|---:|---:|")
for k, (n, ns) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print(f"| `{k}` | {n} | {ns / 1e6:.3f} | {100 * ns / total:.1f} % |")
print(f"| **all** | {len(rows)} | {total / 1e6:.3f} | 100 % |")
