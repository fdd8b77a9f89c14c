"""Stereo sessions without a GPU: the new entry points are declared, exported and bound with the header's signatures, the
session handle is opaque to the bindings, and examples/streams_cpp.cpp (plstvo::StereoStreamsHandler) compiles and links."""
import ctypes as C
import os
import re
import subprocess

from conftest import ROOT
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import EXPORTED_SYMBOLS, LIB_PATH, load_library

LIBDIR = os.path.dirname(LIB_PATH)
HEADER = os.path.join(ROOT, "include", "plstvo.h")
SESSION_CALLS = ("plstvo_stereo_session_create", "plstvo_stereo_session_destroy", "plstvo_stereo_session_device_bytes",
                 "plstvo_stereo_session_initialize", "plstvo_stereo_session_insert")


def build_streams_example(tmp_path):
    exe = str(tmp_path / "streams_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "streams_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def declaration(name):
    txt = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"\b([A-Za-z_0-9]+\s*\*?)\s*" + name + r"\s*\(([^;]*)\)\s*;", txt)
    assert m, name
    return m.group(1).strip(), [p.strip() for p in m.group(2).split(",")]


def test_session_calls_are_declared_exported_and_bound():
    lib = C.CDLL(LIB_PATH)
    for n in SESSION_CALLS:
        assert hasattr(lib, n), n
        assert n in EXPORTED_SYMBOLS, n
    bound = load_library()
    for n in SESSION_CALLS:
        ret, params = declaration(n)
        fn = getattr(bound, n)
        assert len(fn.argtypes) == len(params), (n, params)
        # the session is an opaque handle: a void pointer in the bindings, PlStereoSession* in the header
        for p, a in zip(params, fn.argtypes):
            if "PlStereoSession" in p or "PlContext" in p or "PlRectifier" in p or "PlPrior" in p or "PlPoseResult" in p:
                assert a is C.c_void_p, (n, p, a)
            elif p.startswith("int ") or p == "int":
                assert a is C.c_int, (n, p, a)
            elif "int32_t*" in p:
                assert a == T.c_int32_p, (n, p, a)
            elif "PlStereoImages" in p:
                assert a == C.POINTER(T.PlStereoImages), (n, p, a)
        if ret.startswith("PlStereoSession"):
            assert fn.restype is C.c_void_p
        elif ret == "int64_t":
            assert fn.restype is C.c_int64
        elif ret == "void":
            assert fn.restype is None
        else:
            assert ret == "int" and fn.restype is C.c_int, (n, ret)


def test_session_create_parameter_order():
    _, params = declaration("plstvo_stereo_session_create")
    kinds = [re.match(r"(?:const\s+)?(\w+)", p).group(1) for p in params]
    assert kinds == ["PlContext", "PlCamera", "PlConfig", "PlStereoMatchConfig", "PlStereoConfig", "PlOrbDetectConfig",
                     "PlLsdConfig", "PlRectifier", "int"], kinds
    args = load_library().plstvo_stereo_session_create.argtypes
    assert args[1:7] == [C.POINTER(T.PlCamera), C.POINTER(T.PlConfig), C.POINTER(T.PlStereoMatchConfig),
                         C.POINTER(T.PlStereoConfig), C.POINTER(T.PlOrbDetectConfig), C.POINTER(T.PlLsdConfig)]


def test_header_record_sizes_match_the_record_table(tmp_path):
    """The header states bytes per kept point and line, per retained point and line, and per retained tracker row; they are
    the sizes the record table (csrc/records.h) gives the previous-frame role, the lifted records and the m12 / inlier rows."""
    txt = re.sub(r"\s*\n\s*\*?\s*", " ", open(HEADER).read())
    assert "per kept stereo point 64 bytes" in txt and "per kept stereo line 124 bytes" in txt
    assert "(96 bytes per stereo point, 176 per stereo line)" in txt and "(5 bytes per kept row)" in txt
    src = tmp_path / "sizes.cpp"
    src.write_text('''#include <cstdio>
#include "records.h"
using namespace plstvo;
int main() {
    std::printf("%d %d %d %d %d %d\\n", prev_row_bytes(true), prev_row_bytes(false), rec_row_bytes(PT_PL, LS_SPL),
                rec_row_bytes(LS_SPL, N_LIFT), rec_row_bytes(M12_PT, M12_LS), rec_row_bytes(M12_LS, N_REC));
}
''')
    exe = str(tmp_path / "sizes")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "stvo_pl_b200", "csrc"), str(src),
                    "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    assert out == ["64", "124", "96", "176", "5", "5"], out


def test_streams_example_compiles_and_links(tmp_path):
    build_streams_example(tmp_path)


def test_handler_examples_still_compile(tmp_path):
    for ex in ("images_lsd_cpp", "raw_images_cpp"):
        subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "examples", ex + ".cpp"), "-L", LIBDIR, "-lplstvo_b200",
                        f"-Wl,-rpath,{LIBDIR}", "-o", str(tmp_path / ex)], check=True)
