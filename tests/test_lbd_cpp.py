"""examples/lbd_cpp.cpp (plstvo::computeLBD + matchStereoLines in C++) compiles and links everywhere; on the GPU box it runs
on the first KITTI-size golden stereo frame and must give the reference's descriptors (their byte sums) and lift lines."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")


def build_example(tmp_path):
    exe = str(tmp_path / "lbd_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "lbd_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_lbd_example_compiles_and_links(tmp_path):
    build_example(tmp_path)


@pytest.mark.gpu
def test_lbd_example_runs(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_lbd_golden as M
    images, off, seg, ang, npix, desc = M.load_case(np.load(os.path.join(GOLDEN, "lbd.npz")), "kitti_stereo")
    path = tmp_path / "frame.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", images.shape[2], images.shape[1]))
        f.write(np.ascontiguousarray(images[:2]).tobytes())
        for s in range(2):
            for a, dt in ((seg[off[s]:off[s + 1]], np.float32), (ang[off[s]:off[s + 1]], np.float32),
                          (npix[off[s]:off[s + 1]], np.int32)):
                a = np.ascontiguousarray(a, dt).ravel()
                f.write(struct.pack("<q", a.size))
                f.write(a.tobytes())
    out = subprocess.run([build_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout.split()
    assert [int(out[1]), int(out[2])] == [off[1] - off[0], off[2] - off[1]]
    assert [int(out[4]), int(out[5])] == [int(desc[off[s]:off[s + 1]].astype(np.int64).sum()) for s in range(2)]
    assert int(out[7]) > 20
