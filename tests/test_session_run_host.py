"""plstvo_stereo_session_run without a GPU: the run and the handler-config calls are declared, exported and bound with the
header's signatures, PlHandlerConfig has the header's layout, the default and KITTI handler configs hold the values of
src/config.cpp and config_kitti.yaml, and examples/run_cpp.cpp compiles and links."""
import ctypes as C
import os
import subprocess

from conftest import ROOT
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import EXPORTED_SYMBOLS, LIB_PATH, load_library
from stvo_pl_b200.handler import HandlerConfig
from test_stereo_session_host import declaration

LIBDIR = os.path.dirname(LIB_PATH)
CALLS = ("plstvo_stereo_session_run", "plstvo_default_handler_config", "plstvo_kitti_handler_config")


def build_run_example(tmp_path):
    exe = str(tmp_path / "run_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "run_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_run_calls_are_declared_exported_and_bound():
    lib = C.CDLL(LIB_PATH)
    bound = load_library()
    for n in CALLS:
        assert hasattr(lib, n), n
        assert n in EXPORTED_SYMBOLS, n
        ret, params = declaration(n)
        fn = getattr(bound, n)
        assert len(fn.argtypes) == len(params), (n, params)
        for p, a in zip(params, fn.argtypes):
            if "PlStereoSession" in p or "PlContext" in p or "PlPrior" in p or "PlPoseResult" in p:
                assert a is C.c_void_p, (n, p, a)
            elif "PlHandlerConfig" in p:
                assert a == C.POINTER(T.PlHandlerConfig), (n, p, a)
            elif "PlStereoImages" in p:
                assert a == C.POINTER(T.PlStereoImages), (n, p, a)
            elif "int32_t*" in p:
                assert a == T.c_int32_p, (n, p, a)
            elif p.startswith("int ") or p == "int":
                assert a is C.c_int, (n, p, a)
            else:
                raise AssertionError((n, p))
        assert fn.restype is (None if ret == "void" else C.c_int), (n, ret)
    # the run takes insert's leading arguments, with the handler config after the session and T after ids
    _, run = declaration("plstvo_stereo_session_run")
    _, ins = declaration("plstvo_stereo_session_insert")
    assert run[:2] == ins[:2] and run[3:5] == ins[2:4] and run[6] == ins[4]


def test_handler_config_layout_and_values():
    assert C.sizeof(T.PlHandlerConfig) == 24
    assert [f for f, _ in T.PlHandlerConfig._fields_] == ["adaptative_fast", "fast_min_th", "fast_max_th", "fast_inc_th",
                                                         "fast_feat_th", "fast_err_th"]
    lib = load_library()
    h = T.PlHandlerConfig()
    lib.plstvo_default_handler_config(C.byref(h))   # src/config.cpp:52, :72-76
    assert (h.adaptative_fast, h.fast_min_th, h.fast_max_th, h.fast_inc_th, h.fast_feat_th, h.fast_err_th) == (1, 5, 50, 5, 50, 0.5)
    py = T.handler_config(HandlerConfig())   # the Python handler's defaults are the same values
    assert bytes(py) == bytes(h)
    lib.plstvo_kitti_handler_config(C.byref(h))     # config_kitti.yaml:10, :31-35
    assert (h.adaptative_fast, h.fast_min_th, h.fast_max_th, h.fast_inc_th, h.fast_feat_th, h.fast_err_th) == (1, 7, 30, 5, 50, 0.5)
    lib.plstvo_default_handler_config(None)          # a null pointer is ignored
    lib.plstvo_kitti_handler_config(None)


def test_run_example_compiles(tmp_path):
    assert os.path.exists(build_run_example(tmp_path))
