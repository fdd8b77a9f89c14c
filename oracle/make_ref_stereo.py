"""Builds oracle/_ref/libplstvo_ref_stereo.so: the reference's stereo step (matchGrid for points and lines, GridStructure,
LineIterator, matchStereoPoints / matchStereoLines and the helpers they call) compiled from its OWN text.

TEST INFRASTRUCTURE, the sibling of oracle/make_ref.py and oracle/make_ref_lbd.py (same flags, same way of cutting).  This
recipe

  1. cuts the UNMODIFIED definitions listed in RANGES out of the reference by line range (each range is checked against the
     text expected on its first line, for a closing brace on its last and for balanced braces) into
     oracle/_ref/extracted_stereo.inc and extracted_stereo_cam.inc (git-ignored: reference sources never enter the
     repository),
  2. compiles oracle/ref_shim/stereo_driver.cpp, which includes them after the stand-in header
     oracle/ref_shim/stereo_standin.h (ours: a minimal cv::Mat of 32-byte rows, KeyPoint / KeyLine, the Config accessors
     and the class declarations with the reference's member names, on oracle/ref_shim/eigen_standin.h),
  3. writes oracle/_ref/libplstvo_ref_stereo.so with C entry points (stereo_driver.cpp; bound by oracle/stereo_ref.py).

Every line of dot, normalize, distance, both matchGrid overloads, getLineCoords, GridStructure, LineIterator,
matchStereoPoints, matchStereoLines, filterLineSegmentDisparity, lineSegmentOverlapStereo, the PointFeature / LineFeature
constructors and backProjection IS the reference's text.  The containers they run on (std::unordered_set, std::list) are
libstdc++'s, as in the reference's own build.

Runs only where the reference checkout exists.  Elsewhere a prebuilt library is used as it is.
`python oracle/make_ref_stereo.py` builds; `--check` only verifies the ranges.
"""
from __future__ import annotations

import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PLSTVO_REFERENCE", "/root/reference")
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libplstvo_ref_stereo.so")
SHIM = os.path.join(HERE, "ref_shim")

# (group, file, first line, last line, regex the first line must match); cut in this order (declaration before use)
RANGES = [
    ("stereo", "include/matching.h", 39, 48, r"^inline double dot\(const std::pair<double, double> &a, const std::pair<double, double> &b\) \{$"),
    ("stereo", "src/lineIterator.cpp", 34, 77, r"^LineIterator::LineIterator\(const double x1_, const double y1_, const double x2_, const double y2_\)$"),
    ("stereo", "src/gridStructure.cpp", 33, 83, r"^void getLineCoords\(double x1, double y1, double x2, double y2, std::list<std::pair<int, int>> &line_coords\) \{$"),
    ("stereo", "src/matching.cpp", 93, 109, r"^int distance\(const cv::Mat &a, const cv::Mat &b\) \{$"),
    ("stereo", "src/matching.cpp", 111, 177, r"^int matchGrid\(const std::vector<point_2d> &points1, const cv::Mat &desc1, const GridStructure &grid,"),
    ("stereo", "src/matching.cpp", 179, 258, r"^int matchGrid\(const std::vector<line_2d> &lines1, const cv::Mat &desc1,$"),
    ("stereo", "src/stereoFeatures.cpp", 41, 47, r"^PointFeature::PointFeature\( Vector2d pl_, double disp_, Vector3d P_, int idx_, int level_ \) :$"),
    ("stereo", "src/stereoFeatures.cpp", 107, 115, r"^LineFeature::LineFeature\( Vector2d spl_, double sdisp_, Vector3d sP_,$"),
    ("stereo", "src/stereoFrame.cpp", 120, 173, r"^void StereoFrame::matchStereoPoints\( vector<KeyPoint> points_l, vector<KeyPoint> points_r, Mat &pdesc_l_, Mat pdesc_r, bool initial \)$"),
    ("stereo", "src/stereoFrame.cpp", 309, 398, r"^void StereoFrame::matchStereoLines\( vector<KeyLine> lines_l, vector<KeyLine> lines_r, Mat &ldesc_l_, Mat ldesc_r, bool initial \)$"),
    ("stereo", "src/stereoFrame.cpp", 405, 415, r"^void StereoFrame::filterLineSegmentDisparity\( Vector2d spl, Vector2d epl, Vector2d spr, Vector2d epr, double &disp_s, double &disp_e \)$"),
    ("stereo", "src/stereoFrame.cpp", 473, 508, r"^double StereoFrame::lineSegmentOverlapStereo\( double spl_obs, double epl_obs, double spl_proj, double epl_proj  \)$"),
    ("stereo_cam", "src/pinholeStereoCamera.cpp", 221, 229, r"^Vector3d PinholeStereoCamera::backProjection\( const double &u, const double &v, const double &disp \)$"),
]


def extract() -> dict:
    """Returns {group: text}; verifies each range begins with the expected definition and ends with a closing brace."""
    cache: dict = {}
    groups: dict = {}
    for group, rel, a, b, sig in RANGES:
        path = os.path.join(REF, rel)
        if path not in cache:
            with open(path, encoding="utf-8", errors="replace") as f:
                cache[path] = f.read().split("\n")
        lines = cache[path][a - 1:b]
        if not re.search(sig, lines[0].rstrip()):
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
    return all(os.path.isfile(os.path.join(REF, rel)) for rel in {r[1] for r in RANGES})


def build(force: bool = False) -> str:
    srcs = [os.path.join(SHIM, n) for n in ("stereo_driver.cpp", "stereo_standin.h", "eigen_standin.h")] + [os.path.abspath(__file__)]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return LIB
    if not available():
        if os.path.exists(LIB):
            return LIB    # prebuilt library; the reference is not here to rebuild it
        raise RuntimeError(f"{REF} not found and no prebuilt {LIB}")
    os.makedirs(OUT, exist_ok=True)
    for group, text in extract().items():
        with open(os.path.join(OUT, f"extracted_{group}.inc"), "w") as f:
            f.write(text)
    # make_ref.build's flags: the reference's -O3 -march=native evaluated unfused (-ffp-contract=off) on a portable ISA
    cmd = ["g++", "-std=c++11", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fPIC", "-shared", "-w",
           "-I", SHIM, "-I", OUT, "-I", os.path.join(HERE, ".."), "-o", LIB, os.path.join(SHIM, "stereo_driver.cpp")]
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
