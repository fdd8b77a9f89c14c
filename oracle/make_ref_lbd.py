"""Builds oracle/_ref/libplstvo_ref_lbd.so: the reference's LBD line descriptor (BinaryDescriptor::compute with default
Params) compiled from its OWN text.

TEST INFRASTRUCTURE, the sibling of oracle/make_ref.py (same flags, same way of cutting).  This recipe

  1. cuts the UNMODIFIED definitions listed in RANGES out of
     3rdparty/line_descriptor/src/binary_descriptor_custom.cpp by line range (each range is checked against the text
     expected on its first line and for balanced braces) into oracle/_ref/extracted_lbd.inc (git-ignored: reference
     sources never enter the repository),
  2. compiles oracle/ref_shim/lbd_driver.cpp, which includes them inside namespace cv::line_descriptor after the stand-in
     header oracle/ref_shim/lbd_standin.h (ours: a minimal cv::Mat, the class declarations with the reference's member
     names, and GaussianBlur / Sobel held bit for bit to cv2),
  3. writes oracle/_ref/libplstvo_ref_lbd.so with C entry points (lbd_driver.cpp; bound by oracle/lbd.py).

Every line of NUM_OF_BANDS, combinations, Params(), the constructor (the coefficient tables), get2Pow, computeGaussianPyramid,
computeSobel, binaryConversion, computeImpl and computeLBD IS the reference's text.  The blur and the Sobel those lines
call are the stand-in's.

Runs only where the reference checkout exists.  Elsewhere a prebuilt library is used as it is.
`python oracle/make_ref_lbd.py` builds; `--check` only verifies the ranges.
"""
from __future__ import annotations

import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PLSTVO_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libplstvo_ref_lbd.so")
SHIM = os.path.join(HERE, "ref_shim")
SRC = "3rdparty/line_descriptor/src/binary_descriptor_custom.cpp"

# (first line, last line, regex the first line must match, text the last non-empty line must be)
RANGES = [
    (57, 57, r"^#define NUM_OF_BANDS 9$", "#define NUM_OF_BANDS 9"),
    (74, 107, r"^static const int combinations\[32\]\[2\] =$", "{ 7, 8 } };"),
    (110, 116, r"^BinaryDescriptor::Params::Params\(\)$", "}"),
    (217, 259, r"^BinaryDescriptor::BinaryDescriptor\( const BinaryDescriptor::Params &parameters \) :$", "}"),
    (338, 347, r"^static inline int get2Pow\( int i \)$", "}"),
    (350, 370, r"^void BinaryDescriptor::computeGaussianPyramid\( const Mat& image, const int numOctaves \)$", "}"),
    (373, 398, r"^void BinaryDescriptor::computeSobel\( const cv::Mat& image, const int numOctaves \)$", "}"),
    (401, 412, r"^unsigned char BinaryDescriptor::binaryConversion\( float\* f1, float\* f2 \)$", "}"),
    (539, 687, r"^void BinaryDescriptor::computeImpl\( const Mat& imageSrc, std::vector<KeyLine>& keylines, Mat& descriptors,", "}"),
    (1026, 1372, r"^int BinaryDescriptor::computeLBD\( ScaleLines &keyLines, bool useDetectionData \)$", "}"),
]


def extract() -> str:
    with open(os.path.join(REF, SRC), encoding="utf-8", errors="replace") as f:
        src = f.read().split("\n")
    parts = []
    for a, b, sig, end in RANGES:
        lines = src[a - 1:b]
        if not re.search(sig, lines[0].rstrip()):
            raise RuntimeError(f"{SRC}:{a} does not start with the expected definition: {lines[0]!r}")
        last = next(l for l in reversed(lines) if l.strip())
        if last.strip() != end:
            raise RuntimeError(f"{SRC}:{a}-{b} does not end with {end!r}: {last!r}")
        text = "\n".join(lines)
        if text.count("{") != text.count("}"):
            raise RuntimeError(f"{SRC}:{a}-{b} has unbalanced braces")
        parts.append(f"// ---- {SRC}:{a}-{b} (verbatim) ----\n#line {a} \"{SRC}\"\n{text}\n")
    return "\n".join(parts)


def available() -> bool:
    return os.path.isfile(os.path.join(REF, SRC))


def build(force: bool = False) -> str:
    srcs = [os.path.join(SHIM, n) for n in ("lbd_driver.cpp", "lbd_standin.h")] + [os.path.abspath(__file__)]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return LIB
    if not available():
        if os.path.exists(LIB):
            return LIB    # prebuilt library; the reference is not here to rebuild it
        raise RuntimeError(f"{os.path.join(REF, SRC)} not found and no prebuilt {LIB}")
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "extracted_lbd.inc"), "w") as f:
        f.write(extract())
    # make_ref.build's flags: the reference's -O3 -march=native evaluated unfused (-ffp-contract=off) on a portable ISA
    cmd = ["g++", "-std=c++11", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fPIC", "-shared", "-w",
           "-I", SHIM, "-I", OUT, "-o", LIB, os.path.join(SHIM, "lbd_driver.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("g++ failed: " + " ".join(cmd))
    return LIB


if __name__ == "__main__":
    if "--check" in sys.argv:
        extract()
        print("ranges ok:", len(RANGES))
    else:
        print(build(force="--force" in sys.argv))
