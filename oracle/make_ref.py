"""Builds oracle/_ref/libplstvo_ref.so: the pose half of rubengooj/stvo-pl compiled from the reference's OWN text.

TEST INFRASTRUCTURE.  The reference project cannot be built in this image (Eigen, OpenCV C++, Boost and yaml-cpp are
absent, and its CMake build is off limits).  Its pose path, however, only needs a small Eigen surface.  This recipe

  1. cuts the UNMODIFIED function definitions out of /root/reference by line range (each range is checked against the
     signature expected on its first line, so a drifted checkout fails loudly instead of compiling the wrong lines) into
     oracle/_ref/extracted_*.inc  (git-ignored: reference sources never enter the repository),
  2. compiles oracle/ref_shim/ref_driver.cpp, which includes them after the stand-in headers of oracle/ref_shim/
     (ours: a small Eigen look-alike and the class declarations with the reference's member names),
  3. writes oracle/_ref/libplstvo_ref.so, whose C entry points mirror the oracle's (oracle/plstvo_oracle.h).

What is and is not the reference's code in that library: every line of optimizeFunctions, optimizeFunctionsRobust,
gaussNewtonOptimization[Robust], removeOutliers, isGoodSolution, optimizePose, the key-frame test (needNewKF,
currFrameIsKF), lineSegmentOverlap, projection, the SE(3) helpers and the MAD statistics IS the reference's text.  The dense
6x6 decompositions those lines call (ColPivHouseholderQR::solve / logAbsDeterminant, Matrix::inverse, Matrix::determinant,
SelfAdjointEigenSolver::eigenvalues) are the stand-in's, not Eigen's.

Runs only where /root/reference exists (this container).  The GPU box uses the prebuilt .so that travels with the
snapshot.  `python oracle/make_ref.py` builds; `--check` only verifies the ranges.
"""
from __future__ import annotations

import hashlib
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PLSTVO_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libplstvo_ref.so")
STAMP = LIB + ".stamp"   # hash of the recipe the library was built from (see build())
SHIM = os.path.join(HERE, "ref_shim")

# (group, file, first line, last line, regex the first line must match)
RANGES = [
    ("aux", "src/auxiliar.cpp", 29, 44, r"^Matrix3d skew\(Vector3d v\)\{"),
    ("aux", "src/auxiliar.cpp", 58, 62, r"^Vector3d skewcoords\(Matrix3d M\)\{"),
    ("aux", "src/auxiliar.cpp", 113, 122, r"^Matrix4d inverse_se3\(Matrix4d T\)\{"),
    ("aux", "src/auxiliar.cpp", 124, 141, r"^Matrix4d expmap_se3\(Vector6d x\)\{"),
    ("aux", "src/auxiliar.cpp", 143, 173, r"^Vector6d logmap_se3\(Matrix4d T\)\{"),
    ("aux", "src/auxiliar.cpp", 175, 182, r"^Matrix6d adjoint_se3\(Matrix4d T\)\{"),
    ("aux", "src/auxiliar.cpp", 184, 190, r"^Matrix6d uncTinv_se3\(Matrix4d T, Matrix6d covT \)\{"),
    ("aux", "src/auxiliar.cpp", 192, 197, r"^Matrix6d unccomp_se3\(Matrix4d T1, Matrix6d covT1, Matrix6d covTinc \)\{"),
    ("aux", "src/auxiliar.cpp", 353, 355, r"^bool is_finite\(const MatrixXd x\)\{"),
    ("aux", "src/auxiliar.cpp", 387, 430, r"^void vector_mean_stdv_mad\( vector<double> residues, double &mean, double &stdv \)"),
    ("aux", "src/auxiliar.cpp", 444, 460, r"^double vector_stdv_mad\( vector<double> residues\)"),
    ("aux", "src/auxiliar.cpp", 556, 583, r"^double robustWeightCauchy\( double norm_res \)"),
    ("cam", "src/pinholeStereoCamera.cpp", 221, 229, r"^Vector3d PinholeStereoCamera::backProjection\("),
    ("cam", "src/pinholeStereoCamera.cpp", 231, 237, r"^Vector2d PinholeStereoCamera::projection\(const Vector3d &P \)"),
    ("frame", "src/stereoFrame.cpp", 510, 616, r"^double StereoFrame::lineSegmentOverlap\("),
    ("handler", "src/stereoFrameHandler.cpp", 292, 305, r"^bool StereoFrameHandler::isGoodSolution\("),
    ("handler", "src/stereoFrameHandler.cpp", 307, 392, r"^void StereoFrameHandler::optimizePose\(\)"),
    ("handler", "src/stereoFrameHandler.cpp", 394, 431, r"^void StereoFrameHandler::gaussNewtonOptimization\("),
    ("handler", "src/stereoFrameHandler.cpp", 433, 480, r"^void StereoFrameHandler::gaussNewtonOptimizationRobust\("),
    ("handler", "src/stereoFrameHandler.cpp", 549, 694, r"^void StereoFrameHandler::optimizeFunctions\("),
    ("handler", "src/stereoFrameHandler.cpp", 696, 962, r"^void StereoFrameHandler::optimizeFunctionsRobust\("),
    ("handler", "src/stereoFrameHandler.cpp", 988, 1067, r"^void StereoFrameHandler::removeOutliers\("),
    ("handler", "src/stereoFrameHandler.cpp", 1136, 1187, r"^bool StereoFrameHandler::needNewKF\(\)"),
    ("handler", "src/stereoFrameHandler.cpp", 1189, 1218, r"^void StereoFrameHandler::currFrameIsKF\(\)"),
]


def extract() -> dict:
    """Returns {group: text}; verifies each range begins with the expected signature and ends with a closing brace."""
    cache: dict = {}
    groups: dict = {}
    for group, rel, a, b, sig in RANGES:
        path = os.path.join(REF, rel)
        if path not in cache:
            with open(path, encoding="utf-8", errors="replace") as f:
                cache[path] = f.read().split("\n")
        lines = cache[path][a - 1:b]
        if not re.search(sig, lines[0]):
            raise RuntimeError(f"{rel}:{a} does not start with the expected definition: {lines[0]!r}")
        last = next(l for l in reversed(lines) if l.strip())
        if last.strip() != "}":
            raise RuntimeError(f"{rel}:{a}-{b} does not end with a closing brace: {last!r}")
        text = "\n".join(lines)
        if text.count("{") != text.count("}"):
            raise RuntimeError(f"{rel}:{a}-{b} has unbalanced braces")
        groups.setdefault(group, []).append(f"// ---- {rel}:{a}-{b} (verbatim) ----\n#line {a} \"{rel}\"\n{text}\n")
    return {g: "\n".join(parts) for g, parts in groups.items()}


def available() -> bool:
    return os.path.isdir(os.path.join(REF, "src"))


def recipe_hash() -> str:
    """sha256 of everything the library is built from in this repository: the driver, the stand-ins, the C-ABI header it
    marshals and this recipe (its RANGES).  A library is current only when its stamp holds this hash: file times say nothing
    once a tree has been checked out or copied."""
    h = hashlib.sha256()
    for p in [os.path.join(SHIM, n) for n in ("ref_driver.cpp", "eigen_standin.h", "stvo_standin.h")] + \
             [os.path.join(HERE, "..", "include", "plstvo.h"), os.path.abspath(__file__)]:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def current() -> bool:
    """The library exists and was built from this repository's recipe."""
    try:
        with open(STAMP) as f:
            return os.path.exists(LIB) and f.read().strip() == recipe_hash()
    except OSError:
        return False


def build(force: bool = False) -> str:
    if not force and current():
        return LIB
    if not available():
        if os.path.exists(LIB):
            return LIB    # prebuilt library travelled with the snapshot; the reference is not here to rebuild it
        raise RuntimeError(f"{REF} not found and no prebuilt {LIB}")
    os.makedirs(OUT, exist_ok=True)
    for group, text in extract().items():
        with open(os.path.join(OUT, f"extracted_{group}.inc"), "w") as f:
            f.write(text)
    # the reference's own flags are -std=c++11 -O3 -march=native (CMakeLists.txt:18); x86-64-v3 keeps the library portable
    # between this container and the GPU box, -ffp-contract=off matches the oracle's build
    cmd = ["g++", "-std=c++11", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fPIC", "-shared", "-w",
           "-I", SHIM, "-I", OUT, "-I", os.path.join(HERE, ".."), "-o", LIB, os.path.join(SHIM, "ref_driver.cpp")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("g++ failed: " + " ".join(cmd))
    with open(STAMP, "w") as f:
        f.write(recipe_hash() + "\n")
    return LIB


if __name__ == "__main__":
    if "--check" in sys.argv:
        extract()
        print("ranges ok:", len(RANGES))
    else:
        print(build(force="--force" in sys.argv))
