"""Host-side checks of rectification: the library's plstvo_init_undistort_rectify_map (host code, no GPU) equals
tests/golden/rectify.npz and oracle/rectify.py, rejects what it does not build, PlRectifyModel's ctypes mirror has the C size,
the new ctypes signatures have the header's parameter counts, and examples/raw_images_cpp.cpp compiles and links with
-Wall -Werror."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import rectify as R
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import PlstvoError, init_undistort_rectify_map, load_library

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_rectify_golden as M  # noqa: E402

LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")
G = np.load(os.path.join(GOLDEN, "rectify.npz"))


def build_raw_example(tmp_path):
    exe = str(tmp_path / "raw_images_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "raw_images_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


@pytest.mark.parametrize("case", list(G["map_cases"]))
def test_library_maps_equal_golden(case):
    w, h = (int(v) for v in G[f"{case}_size"])
    args = (int(G[f"{case}_model"]), G[f"{case}_K"], G[f"{case}_D"], G[f"{case}_R"], G[f"{case}_P"], w, h)
    m1, m2 = init_undistort_rectify_map(*args)
    assert (M.sha(m1, m2) == G[f"{case}_map_sha"]).all()
    o1, o2 = R.init_undistort_rectify_map(*args)
    np.testing.assert_array_equal(m1, o1)
    np.testing.assert_array_equal(m2, o2)


def test_library_maps_equal_restatement_on_a_sweep():
    rng = np.random.default_rng(3)
    for k in range(16):
        model = k % 2
        K = np.array([[300 + rng.uniform(0, 200), 0, 100 + rng.uniform(0, 50)], [0, 300 + rng.uniform(0, 200), 80], [0, 0, 1]])
        nd = 4 if model else (4, 5, 8)[k % 3]
        D = rng.normal(0, 0.2, nd) * np.array([1, 0.3, 0.01, 0.01, 0.1, 0.3, 0.1, 0.05])[:nd]
        c, s = np.cos(rng.normal(0, 0.03)), np.sin(rng.normal(0, 0.03))
        Rm = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
        P = np.hstack([K * rng.uniform(0.7, 1.2), np.zeros((3, 1))])
        P[2] = [0, 0, 1, 0]
        w, h = int(rng.integers(1, 260)), int(rng.integers(1, 90))
        m1, m2 = init_undistort_rectify_map(model, K, D, Rm, P, w, h)
        o1, o2 = R.init_undistort_rectify_map(model, K, D, Rm, P, w, h)
        np.testing.assert_array_equal(m1, o1)
        np.testing.assert_array_equal(m2, o2)


def _rc(model=0.0, n_dist=4.0, P=None, w=8, h=8, null=False):
    lib = load_library()
    m = T.rectify_model(0, np.eye(3), [0.1, 0, 0, 0], np.eye(3), np.eye(3) if P is None else P)
    m.model, m.n_dist = model, n_dist
    m1 = np.zeros((max(h, 1), max(w, 1), 2), np.int16)
    m2 = np.zeros((max(h, 1), max(w, 1)), np.uint16)
    return lib.plstvo_init_undistort_rectify_map(None if null else C.byref(m), w, h, m1.ctypes.data_as(C.POINTER(C.c_int16)),
                                                 m2.ctypes.data_as(C.POINTER(C.c_uint16)))


@pytest.mark.parametrize("bad", [dict(n_dist=12.0), dict(n_dist=14.0), dict(n_dist=3.0), dict(n_dist=4.5), dict(model=2.0),
                                 dict(model=1.0, n_dist=5.0), dict(P=np.zeros((3, 3))),
                                 dict(P=np.array([[1.0, 2, 3], [2, 4, 6], [0, 0, 1]])), dict(w=0), dict(h=32768),
                                 dict(w=-1), dict(null=True)])
def test_invalid_models_are_rejected(bad):
    assert _rc(**bad) == -1


def test_valid_model_passes_and_binding_raises():
    assert _rc() == 0 and _rc(model=1.0) == 0 and _rc(n_dist=8.0) == 0 and _rc(w=32767, h=1) == 0
    with pytest.raises(PlstvoError):
        init_undistort_rectify_map(0, np.eye(3), [0.1] * 12, np.eye(3), np.eye(3), 8, 8)


def test_rectify_model_struct_size(tmp_path):
    c = tmp_path / "s.c"
    c.write_text('#include <stdio.h>\n#include "plstvo.h"\n'
                 'int main(void) { printf("%zu\\n", sizeof(PlRectifyModel)); return 0; }\n')
    exe = str(tmp_path / "s")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", exe], check=True)
    assert int(subprocess.run([exe], capture_output=True, text=True, check=True).stdout) == C.sizeof(T.PlRectifyModel) == 320


def test_rectify_entry_point_signatures():
    header = open(os.path.join(ROOT, "include", "plstvo.h")).read()
    lib = load_library()
    for name in ("plstvo_init_undistort_rectify_map", "plstvo_rectifier_create", "plstvo_rectifier_destroy",
                 "plstvo_rectify_batch", "plstvo_rectify_kernel_times", "plstvo_track_stereo_raw_images_batch",
                 "plstvo_track_stereo_raw_images_sequence"):
        decl = re.search(r"\b(?:int|void|PlRectifier\*)\s+" + name + r"\s*\(([^;]*)\)\s*;", header).group(1)
        params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")]
        assert len(getattr(lib, name).argtypes) == len(params), (name, params)
    for name in ("plstvo_track_stereo_raw_images_batch", "plstvo_track_stereo_raw_images_sequence"):
        decl = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\)\s*;", header).group(1)
        params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")]
        assert params[6].startswith("const PlLsdConfig*") and params[7].startswith("const PlRectifier*"), params


def test_raw_images_example_compiles_and_links(tmp_path):
    build_raw_example(tmp_path)
