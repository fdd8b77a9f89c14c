"""Reading a session call's frames back, without a GPU: the ctypes PlStereoFrameOut has the header's layout (offsets printed
by a compiled C program), the new calls are bound with the header's signatures, and plstvo.hpp with examples/frames_out_cpp.cpp
(StereoImageHandler::keepFeatures feeding a features-in StereoFrameHandler) compiles and links."""
import ctypes as C
import os
import subprocess

from conftest import ROOT
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import EXPORTED_SYMBOLS, LIB_PATH, load_library

LIBDIR = os.path.dirname(LIB_PATH)
INCLUDE = os.path.join(ROOT, "include")


def build_frames_example(tmp_path):
    exe = str(tmp_path / "frames_out_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", INCLUDE, os.path.join(ROOT, "examples", "frames_out_cpp.cpp"),
                    "-L", LIBDIR, "-lplstvo_b200", f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_frame_out_layout_matches_the_header(tmp_path):
    names = [f for f, _ in T.PlStereoFrameOut._fields_]
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"plstvo.h\"\nint main(void) {\n"
    src += '  printf("%zu\\n", sizeof(PlStereoFrameOut));\n'
    for n in names:
        src += f'  printf("{n} %zu\\n", offsetof(PlStereoFrameOut, {n}));\n'
    src += "  return 0; }\n"
    c = tmp_path / "layout.c"
    c.write_text(src)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", INCLUDE, str(c), "-o", exe], check=True)
    lines = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n")
    assert int(lines[0]) == C.sizeof(T.PlStereoFrameOut) == 23 * 8
    got = dict((a, int(b)) for a, b in (ln.split() for ln in lines[1:] if ln))
    assert got == {n: getattr(T.PlStereoFrameOut, n).offset for n in names}


def test_record_keys_cover_the_struct_and_the_match_stereo_outputs():
    pt, ls = T.FRAME_OUT_POINT_KEYS, T.FRAME_OUT_LINE_KEYS
    fields = [f for f, _ in T.PlStereoFrameOut._fields_]
    assert list(pt) + list(ls) + ["m12_pt", "inlier_pt", "m12_ls", "inlier_ls"] == fields
    assert set(pt.values()) == {"pl", "disp", "P", "sigma2", "level", "desc", "src_idx"}
    assert set(ls.values()) == {"spl", "epl", "sdisp", "edisp", "sP", "eP", "le", "angle", "sigma2", "level", "desc", "src_idx"}


def test_retain_and_read_are_exported_and_bound():
    lib = C.CDLL(LIB_PATH)
    bound = load_library()
    for n in ("plstvo_stereo_session_retain", "plstvo_stereo_session_read"):
        assert hasattr(lib, n) and n in EXPORTED_SYMBOLS, n
    assert bound.plstvo_stereo_session_retain.argtypes == [C.c_void_p, C.c_void_p, C.c_int]
    assert bound.plstvo_stereo_session_read.argtypes[2]._type_ is T.PlStereoFrameOut
    assert bound.plstvo_stereo_session_read.restype is C.c_int


def test_null_context_is_rejected_without_a_device():
    lib = load_library()
    o = T.PlStereoFrameOut()
    assert lib.plstvo_stereo_session_retain(None, None, 1) == -1
    assert lib.plstvo_stereo_session_read(None, None, C.byref(o)) == -1


def test_frames_example_compiles_and_links(tmp_path):
    assert os.path.exists(build_frames_example(tmp_path))


def test_header_compiles_with_keep_features(tmp_path):
    src = tmp_path / "keep.cpp"
    src.write_text('#include "plstvo.hpp"\n'
                   "void f(plstvo::StereoImageHandler& a, plstvo::StereoStreamsHandler& b, plstvo::StereoSession& s) {\n"
                   "  a.keepFeatures(true); b.keepFeatures(false); s.retain(true);\n"
                   "  plstvo::StereoSession::Frames fr; const int32_t ns[4] = {0, 0, 0, 0}; s.read(1, ns, true, fr);\n"
                   "  plstvo::StereoFrameHandler* h = nullptr; if (h) h->insertStereoPair(a.curr_frame);\n"
                   "  (void)b.stream(0).matches_pt.size(); }\n")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", INCLUDE, "-c", str(src), "-o",
                    str(tmp_path / "keep.o")], check=True)
