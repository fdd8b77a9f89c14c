"""Builds the CUDA library in-tree: stvo_pl_b200/lib/libplstvo_b200.so (sm_90a only).

nvcc cross-compiles without a GPU; the built .so is git-ignored.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libplstvo_b200.so")
SOURCES = ["match.cu", "match_tc.cu", "match_grid.cu", "lift.cu", "solve.cu", "gn_stream.cu", "orb.cu", "lbd.cu", "lsd.cu", "rectify.cu", "session.cu", "keyframe.cu", "capi.cu", "capi_stereo.cu",
           "capi_features.cu", "plot.cu"]
HEADERS = ["common.cuh", "records.h", "host.cuh", "match_finalize.cuh", "match_tc.cuh", "gn_stream.cuh", "orb_pattern.h", "remap.cuh", os.path.join("..", "..", "include", "plstvo.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-O2", "--use_fast_math=false"]


def nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not stale():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    flags = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [nvcc()] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-shared", "-o", LIB] + srcs + ["-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode:
        raise RuntimeError("nvcc failed: " + " ".join(cmd))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
