"""Host-side checks of the stereo-images entry point: the ctypes mirror of PlStereoImages has the C size, and
examples/images_cpp.cpp (plstvo::trackStereoImages) compiles and links with -Wall -Werror."""
import ctypes as C
import os
import subprocess

from conftest import ROOT
from stvo_pl_b200 import types as T

LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")


def build_example(tmp_path):
    exe = str(tmp_path / "images_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "images_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_stereo_images_struct_size(tmp_path):
    c = tmp_path / "s.c"
    c.write_text('#include <stdio.h>\n#include "plstvo.h"\nint main(void) { printf("%zu\\n", sizeof(PlStereoImages)); return 0; }\n')
    exe = str(tmp_path / "s")
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", exe], check=True)
    assert int(subprocess.run([exe], capture_output=True, text=True, check=True).stdout) == C.sizeof(T.PlStereoImages)


def test_images_example_compiles_and_links(tmp_path):
    build_example(tmp_path)
