"""Builds and runs the packed min/max issue-rate probe (minmax_rates.cu); the probe prints one JSON line.

The binary goes to tools/probes/bin/ (git-ignored), compiled with the library's nvcc flags.  It is rebuilt only when the
source is newer, so a tree built beforehand runs without nvcc.

    python tools/probes/minmax_rates.py [--build-only] [--iters N]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from stvo_pl_b200 import build as B  # noqa: E402

SRC = os.path.join(HERE, "minmax_rates.cu")
BIN = os.path.join(HERE, "bin", "minmax_rates")


def build() -> str:
    if os.path.exists(BIN) and os.path.getmtime(BIN) >= os.path.getmtime(SRC):
        return BIN
    os.makedirs(os.path.dirname(BIN), exist_ok=True)
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    subprocess.run([B.nvcc()] + flags + ["-o", BIN, SRC], check=True)
    return BIN


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--iters", type=int, default=4096)
    a = ap.parse_args()
    exe = build()
    if not a.build_only:
        subprocess.run([exe, str(a.iters)], check=True)


if __name__ == "__main__":
    main()
