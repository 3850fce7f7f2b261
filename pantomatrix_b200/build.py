"""In-tree nvcc build of libpm_emage.so (sm_90a: H100).

    python -m pantomatrix_b200.build [--force]
    python -m pantomatrix_b200.build --variant NAME -DMACRO[=V] ...   # instrumented / tuning build, see build_variant()
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "csrc", "_build")
LIB = os.path.join(HERE, "libpm_emage.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]
# per-file extra flags
EXTRA = {"pm_pose.cu": ["-fmad=false"], "pm_render.cu": ["-fmad=false"]}


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libpm_emage.so cannot be built")


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)) + ["../../include/pm_emage.h"]:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p) and (f.endswith((".cu", ".cuh", ".h"))):
            h.update(f.encode())
            h.update(open(p, "rb").read())
    h.update(" ".join(ARCH + COMMON + [k + str(v) for k, v in sorted(EXTRA.items())]).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "digest.txt")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(OBJ, src[:-3] + ".o")
        cmd = [nvcc, *ARCH, *COMMON, *EXTRA.get(src, []), "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            print(f"--- {src}\n{out}", file=sys.stderr)
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {src}")
    subprocess.check_call([nvcc, *ARCH, "-shared", "-o", LIB, *objs])
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


def build_variant(name: str, defines: list[str]) -> str:
    """Side build of the same sources with extra -D macros (e.g. PM_TC_TIMING: in-kernel clock stamps) into
    csrc/_build/variants/libpm_emage_<name>.so.  Never loaded by default: tools select it with PM_EMAGE_LIB=<path>."""
    vdir = os.path.join(OBJ, "variants", name)
    os.makedirs(vdir, exist_ok=True)
    nvcc = _nvcc()
    procs, objs = [], []
    for src in sources():
        obj = os.path.join(vdir, src[:-3] + ".o")
        cmd = [nvcc, *ARCH, *COMMON, *EXTRA.get(src, []), *defines, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode:
            print(f"--- {src}\n{out}", file=sys.stderr)
            raise RuntimeError(f"nvcc failed on {src}")
    lib = os.path.join(OBJ, "variants", f"libpm_emage_{name}.so")
    subprocess.check_call([nvcc, *ARCH, "-shared", "-o", lib, *objs])
    return lib


if __name__ == "__main__":
    if "--variant" in sys.argv:
        print(build_variant(sys.argv[sys.argv.index("--variant") + 1], [a for a in sys.argv if a.startswith("-D")]))
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
