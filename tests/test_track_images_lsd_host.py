"""Host-side checks of the images-only entry points: the ctypes mirror of PlLsdConfig has the C size, the ctypes signatures
of plstvo_track_stereo_images_lsd_batch / _sequence have the header's parameter counts, and examples/images_lsd_cpp.cpp
(plstvo::StereoImageHandler) compiles and links with -Wall -Werror."""
import ctypes as C
import os
import re
import subprocess

from conftest import ROOT
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import load_library

LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")


def build_lsd_example(tmp_path):
    exe = str(tmp_path / "images_lsd_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "images_lsd_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_lsd_config_struct_size(tmp_path):
    c = tmp_path / "s.c"
    c.write_text('#include <stdio.h>\n#include "plstvo.h"\nint main(void) { printf("%zu\\n", sizeof(PlLsdConfig)); return 0; }\n')
    exe = str(tmp_path / "s")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", exe], check=True)
    assert int(subprocess.run([exe], capture_output=True, text=True, check=True).stdout) == C.sizeof(T.PlLsdConfig)


def test_lsd_entry_point_signatures():
    header = open(os.path.join(ROOT, "include", "plstvo.h")).read()
    lib = load_library()
    for name, lcfg_at in (("plstvo_track_stereo_images_lsd_batch", 6), ("plstvo_track_stereo_images_lsd_sequence", 6)):
        decl = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\)\s*;", header).group(1)
        params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")]
        args = getattr(lib, name).argtypes
        assert len(args) == len(params), (name, params)
        assert params[lcfg_at].startswith("const PlLsdConfig*") and args[lcfg_at] == C.POINTER(T.PlLsdConfig), name


def test_images_lsd_example_compiles_and_links(tmp_path):
    build_lsd_example(tmp_path)
