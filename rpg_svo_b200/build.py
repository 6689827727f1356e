"""Builds libsvo_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

`python -m rpg_svo_b200.build` or `rpg_svo_b200.build.build()`.  nvcc cross-compiles without a GPU.
-fmad=false: every fused multiply-add in the kernels is explicit, so the f32 stages round exactly
like the oracle's restatement of the reference (see csrc/svo_math.cuh).
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libsvo_b200.so")
SOURCES = ["context.cu", "sparse_align.cu", "align.cu", "pose_opt.cu", "depth_filter.cu", "reproject.cu", "detect.cu", "klt.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-fmad=false",
              "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-O2", "-cudart", "static"]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def build(force: bool = False, verbose: bool = False) -> str:
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = srcs + [os.path.join(CSRC, h) for h in os.listdir(CSRC) if h.endswith((".h", ".cuh", ".inc"))]
    deps.append(os.path.join(HERE, "..", "include", "svo_b200.h"))
    if not force and os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    objdir = os.path.join(HERE, "..", "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for s in srcs:
        o = os.path.join(objdir, os.path.basename(s).replace(".cu", ".o"))
        objs.append(o)
        if force or not os.path.exists(o) or any(os.path.getmtime(d) > os.path.getmtime(o) for d in deps if not d.endswith(".cu") or d == s):
            extra = os.environ.get("SVO_B200_EXTRA_NVCC_FLAGS", "").split()  # e.g. -DSVO_SIA_DEBUG=1 for the clock64 section timers
            cmd = [_nvcc()] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            procs.append((cmd, subprocess.Popen(cmd)))
    for cmd, p in procs:
        if p.wait() != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    cmd = [_nvcc(), "-shared", "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a", "-o", OUT] + objs
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
