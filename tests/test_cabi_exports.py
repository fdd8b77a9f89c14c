"""The C-ABI library loads on a CPU-only box and exports every symbol include/plstvo.h declares; the ctypes
mirrors have the C struct sizes.  No compute call is made (there is no GPU here, and no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import EXPORTED_SYMBOLS, LIB_PATH, Engine, PlstvoError, load_library

HEADER = os.path.join(ROOT, "include", "plstvo.h")


def declared_functions():
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(plstvo_[a-z0-9_]+)\s*\(", txt)))


def test_library_is_built():
    assert os.path.exists(LIB_PATH), "run python -m stvo_pl_b200.build (driver: __graft_entry__.build())"


def test_every_declared_symbol_is_exported():
    lib = C.CDLL(LIB_PATH)
    names = declared_functions()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/plstvo.h but not exported"
    assert sorted(EXPORTED_SYMBOLS) == names          # the binding covers the whole header, nothing more
    assert load_library().plstvo_version() == 100


def test_pose_helper_layouts_match_the_header():
    """plstvo_debug_pose_helpers' record offsets in the binding are the header's PLSTVO_PH_* macros."""
    txt = open(HEADER).read()
    defs = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define PLSTVO_PH_(\w+) (\d+)", txt)}
    assert defs.pop("IN") == Engine.PH_IN_SIZE and defs.pop("OUT") == Engine.PH_OUT_SIZE
    ins = {k[3:].lower(): v for k, v in defs.items() if k.startswith("IN_")}
    outs = {k.lower(): v for k, v in defs.items() if not k.startswith("IN_")}
    assert ins == {k.lower(): off for k, (off, _) in Engine.PH_IN.items()}
    assert outs == {k.lower(): off for k, (off, _) in Engine.PH_OUT.items()}
    for layout, size in ((Engine.PH_IN, Engine.PH_IN_SIZE), (Engine.PH_OUT, Engine.PH_OUT_SIZE)):
        spans = sorted((off, off + int(np.prod(shape, dtype=np.int64))) for off, shape in layout.values())
        assert spans[0][0] == 0 and spans[-1][1] == size and all(a[1] == b[0] for a, b in zip(spans, spans[1:]))


def test_struct_layouts_match_the_header():
    src = r'''
#include <stdio.h>
#include "plstvo.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\n", sizeof(PlCamera), sizeof(PlConfig), sizeof(PlFrameBatch),
         sizeof(PlMatchedBatch), sizeof(PlPrior), sizeof(PlPoseResult));
  return 0; }'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "s.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "s")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        sizes = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    assert sizes == [C.sizeof(T.PlCamera), C.sizeof(T.PlConfig), C.sizeof(T.PlFrameBatch),
                     C.sizeof(T.PlMatchedBatch), C.sizeof(T.PlPrior), C.sizeof(T.PlPoseResult)]
    assert T.POSE_RESULT_DTYPE.itemsize == sizes[5] and T.PRIOR_DTYPE.itemsize == sizes[4]


def test_config_presets_match_the_library():
    lib = load_library()
    a, b = T.PlConfig(), T.PlConfig()
    lib.plstvo_default_config(C.byref(a))
    lib.plstvo_kitti_config(C.byref(b))
    for f, _ in T.PlConfig._fields_:
        assert getattr(a, f) == getattr(T.default_config(), f)
        assert getattr(b, f) == getattr(T.kitti_config(), f)


def test_no_cpu_fallback():
    """Without a CUDA device the product path must fail loudly, never compute on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    with pytest.raises(PlstvoError) as ei:
        Engine()
    assert ei.value.code == -4


def test_product_package_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "stvo_pl_b200")
    for dp, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".hpp")):
                txt = open(os.path.join(dp, fn), errors="ignore").read()
                assert "oracle" not in txt.lower().replace("# oracle-free", ""), f"{fn} mentions the oracle"
