"""Builds oracle/_ref/libplstvo_ref_fld.so: the reference's FLD-branch KeyLine step (detectLineFeatures with
use_fld_lines, src/stereoFrame.cpp:260-299, and sort_flines_by_length, include/auxiliar.h:149-154) compiled from its OWN
text.

TEST INFRASTRUCTURE, the sibling of oracle/make_ref_lbd.py (same flags, same way of cutting).  This recipe

  1. cuts the UNMODIFIED lines listed in RANGES out of the reference by line range (each range is checked against the text
     expected on its first and last lines and for balanced braces) into oracle/_ref/extracted_fld_sort.inc and
     extracted_fld.inc (git-ignored: reference sources never enter the repository),
  2. compiles oracle/ref_shim/fld_driver.cpp, which includes them after the stand-in header oracle/ref_shim/fld_standin.h
     (ours: Vec4f, Point / Point2f, a Mat of a size, KeyLine, Config::lsdNFeatures and LineIterator's count),
  3. writes oracle/_ref/libplstvo_ref_fld.so with the C entry point fld_ref_key_lines (bound by tests/test_fld_keylines_host.py).

Every line from the filter to lines.push_back, and the sort functor, IS the reference's text; std::sort is libstdc++'s, as
in the reference's own build.

Runs only where the reference checkout exists.  Elsewhere a prebuilt library is used as it is.
`python oracle/make_ref_fld.py` builds; `--check` only verifies the ranges.
"""
from __future__ import annotations

import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PLSTVO_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libplstvo_ref_fld.so")
SHIM = os.path.join(HERE, "ref_shim")

# (output, file, first line, last line, regex the first line must match, text the last line must be)
RANGES = [
    ("extracted_fld_sort.inc", "include/auxiliar.h", 149, 154, r"^struct sort_flines_by_length$", "};"),
    ("extracted_fld.inc", "src/stereoFrame.cpp", 260, 300, r"^\s*// filter lines$", "}"),
]


def extract() -> dict:
    out = {}
    for name, path, a, b, sig, end in RANGES:
        with open(os.path.join(REF, path), encoding="utf-8", errors="replace") as f:
            src = f.read().split("\n")
        lines = src[a - 1:b]
        if not re.search(sig, lines[0].rstrip()):
            raise RuntimeError(f"{path}:{a} does not start with the expected text: {lines[0]!r}")
        if lines[-1].strip() != end:
            raise RuntimeError(f"{path}:{b} is not {end!r}: {lines[-1]!r}")
        text = "\n".join(lines)
        if text.count("{") != text.count("}"):
            raise RuntimeError(f"{path}:{a}-{b} has unbalanced braces")
        if name == "extracted_fld.inc" and "lines.push_back( kl );" not in text:
            raise RuntimeError(f"{path}:{a}-{b} does not hold the KeyLine loop")
        out[name] = f"// ---- {path}:{a}-{b} (verbatim) ----\n#line {a} \"{path}\"\n{text}\n"
    return out


def available() -> bool:
    return all(os.path.isfile(os.path.join(REF, r[1])) for r in RANGES)


def build(force: bool = False) -> str:
    srcs = [os.path.join(SHIM, n) for n in ("fld_driver.cpp", "fld_standin.h")] + [os.path.abspath(__file__)]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return LIB
    if not available():
        if os.path.exists(LIB):
            return LIB    # prebuilt library; the reference is not here to rebuild it
        raise RuntimeError(f"{REF} sources not found and no prebuilt {LIB}")
    os.makedirs(OUT, exist_ok=True)
    for name, text in extract().items():
        with open(os.path.join(OUT, name), "w") as f:
            f.write(text)
    # make_ref.build's flags: the reference's -O3 -march=native evaluated unfused (-ffp-contract=off) on a portable ISA
    cmd = ["g++", "-std=c++11", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fPIC", "-shared", "-w",
           "-I", SHIM, "-I", OUT, "-o", LIB, os.path.join(SHIM, "fld_driver.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("g++ failed: " + " ".join(cmd))
    return LIB


if __name__ == "__main__":
    if "--check" in sys.argv:
        print("ranges ok:", len(extract()))
    else:
        print(build(force="--force" in sys.argv))
