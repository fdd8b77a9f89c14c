"""Per-stream cameras without a GPU: plstvo_track_batch_cams and plstvo_stereo_session_create_cams are declared, exported and
bound with the header's signatures, and examples/cams_cpp.cpp (plstvo::StereoStreamsHandler with a camera per stream)
compiles and links."""
import ctypes as C
import os
import subprocess

from conftest import ROOT
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import EXPORTED_SYMBOLS, LIB_PATH, load_library
from test_stereo_session_host import declaration

LIBDIR = os.path.dirname(LIB_PATH)
CALLS = ("plstvo_track_batch_cams", "plstvo_stereo_session_create_cams")


def build_cams_example(tmp_path):
    exe = str(tmp_path / "cams_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "cams_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_cams_calls_are_declared_exported_and_bound():
    lib = C.CDLL(LIB_PATH)
    bound = load_library()
    for n in CALLS:
        assert hasattr(lib, n), n
        assert n in EXPORTED_SYMBOLS, n
        ret, params = declaration(n)
        fn = getattr(bound, n)
        assert len(fn.argtypes) == len(params), (n, params)
        for p, a in zip(params, fn.argtypes):
            if p.startswith("const PlCamera*"):
                assert a == C.POINTER(T.PlCamera), (n, p, a)
            elif "PlRectifier* const*" in p:
                assert a == C.POINTER(C.c_void_p), (n, p, a)
            elif "PlContext" in p or "PlPrior" in p or "PlPoseResult" in p:
                assert a is C.c_void_p, (n, p, a)
            elif p.startswith("int ") or p == "int":
                assert a is C.c_int, (n, p, a)
        assert fn.restype is (C.c_void_p if ret.startswith("PlStereoSession") else C.c_int), (n, ret)
    # the track call takes plstvo_track_batch's arguments with the camera made an array
    assert bound.plstvo_track_batch_cams.argtypes == bound.plstvo_track_batch.argtypes
    _, a = declaration("plstvo_track_batch_cams")
    _, b = declaration("plstvo_track_batch")
    assert a[2:] == b[2:]
    # the session call takes plstvo_stereo_session_create's, with cams and rects arrays
    _, a = declaration("plstvo_stereo_session_create_cams")
    _, b = declaration("plstvo_stereo_session_create")
    assert a[2:7] == b[2:7] and a[8:] == b[8:]
    assert C.sizeof(T.PlCamera) == 48   # the per-pair table's entry


def test_cams_example_compiles(tmp_path):
    exe = build_cams_example(tmp_path)
    assert os.path.exists(exe)
