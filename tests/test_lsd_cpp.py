"""examples/lsd_cpp.cpp (plstvo::detectLSD + computeLBD in C++) compiles and links everywhere; on the GPU box it runs on a
KITTI-size golden image and must give the golden key lines (their count and numOfPixels sum) and the same descriptors as the
Python binding."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")


def build_example(tmp_path):
    exe = str(tmp_path / "lsd_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "lsd_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_lsd_example_compiles_and_links(tmp_path):
    build_example(tmp_path)


def test_lsd_config_struct_matches_its_mirror(tmp_path):
    """sizeof(PlLsdConfig) in C equals the ctypes mirror's."""
    import ctypes
    from stvo_pl_b200 import types as T
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "plstvo.h"\nint main(void) { printf("%zu\\n", sizeof(PlLsdConfig)); return 0; }\n')
    exe = str(tmp_path / "sz")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe], check=True)
    assert int(subprocess.run([exe], capture_output=True, text=True, check=True).stdout) == ctypes.sizeof(T.PlLsdConfig)


@pytest.mark.gpu
def test_lsd_example_runs(tmp_path, engine):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_lsd_golden as M
    imgs, P, _, _, kl = M.load_case(np.load(os.path.join(GOLDEN, "lsd.npz")), "kitti_300")
    path = tmp_path / "img.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<ii", imgs.shape[2], imgs.shape[1]))
        f.write(np.ascontiguousarray(imgs[0]).tobytes())
    out = subprocess.run([build_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout.split()
    n = int(kl["off"][1])
    desc = engine.lbd_compute_batch(imgs[:1], kl["off"][:2], kl["seg"][:n], kl["angle"][:n], kl["npix"][:n])
    assert int(out[1]) == n
    assert int(out[3]) == int(kl["npix"][:n].astype(np.int64).sum())
    assert int(out[5]) == int(desc.astype(np.int64).sum())
