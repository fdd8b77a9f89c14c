"""examples/orb_cpp.cpp (plstvo::computeORB + matchStereoPoints in C++) compiles and links everywhere; on the GPU box it runs on
the first KITTI-size golden stereo frame and must find what the Python binding finds."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from stvo_pl_b200 import types as T

LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")


def build_example(tmp_path):
    exe = str(tmp_path / "orb_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "orb_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_orb_example_compiles_and_links(tmp_path):
    build_example(tmp_path)


@pytest.mark.gpu
def test_orb_example_runs(tmp_path, engine):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_orb_golden as M
    z = np.load(os.path.join(GOLDEN, "orb_kitti.npz"))
    imgs, off = M.kitti_views()[:2], z["det_off"]
    path = tmp_path / "frame.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", imgs.shape[2], imgs.shape[1]))
        f.write(np.ascontiguousarray(imgs).tobytes())
        for s in range(2):
            for a, dt in ((z["det_xy"][off[s]:off[s + 1]], np.float32), (z["det_oct"][off[s]:off[s + 1]], np.int32)):
                a = np.ascontiguousarray(a, dt).ravel()
                f.write(struct.pack("<q", a.size))
                f.write(a.tobytes())
    out = subprocess.run([build_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout.split()
    n, res = engine.orb_compute_batch(T.default_orb_config(), imgs, off[:3], z["det_xy"][:off[2]], z["det_oct"][:off[2]], None)
    assert [int(out[1]), int(out[2])] == list(res["counts"])
    assert int(out[4]) > 100
