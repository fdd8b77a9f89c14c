"""examples/orb_detect_cpp.cpp (plstvo::detectAndComputeORB + matchStereoPoints in C++) compiles and links everywhere; on the
GPU box it runs on the first KITTI-size golden stereo frame and must find the counts the Python binding finds."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from stvo_pl_b200 import types as T

LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")


def build_example(tmp_path):
    exe = str(tmp_path / "orb_detect_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "orb_detect_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_orb_detect_example_compiles_and_links(tmp_path):
    build_example(tmp_path)


@pytest.mark.gpu
def test_orb_detect_example_runs(tmp_path, engine):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_orb_golden as M
    imgs = M.kitti_views()[:2]
    path = tmp_path / "frame.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", imgs.shape[2], imgs.shape[1]))
        f.write(np.ascontiguousarray(imgs).tobytes())
    out = subprocess.run([build_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout.split()
    n, res = engine.orb_detect_and_compute_batch(T.default_orb_detect_config(), imgs)
    assert [int(out[1]), int(out[2])] == list(np.diff(res["off"]))
    assert int(out[4]) > 100
