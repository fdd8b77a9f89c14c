"""plstvo_stereo_session_run_keyframes without a GPU: the new calls are declared, exported and bound with the header's
signatures; PlKeyframeConfig / PlKeyframeState / PlKeyframeResult have the header's layout (offsets printed by a compiled C
program); the default config and the initial state are the reference's; KeyframeTest <-> PlKeyframeState round-trips bit for
bit in C++ and in Python; examples/run_kf_cpp.cpp compiles and links; and keyframe.cu holds no FMA nvcc formed itself."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

from conftest import ROOT
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import EXPORTED_SYMBOLS, LIB_PATH, load_library
from stvo_pl_b200.handler import KeyframeTest
from test_fp_contraction import _ptx
from test_stereo_session_host import declaration

LIBDIR = os.path.dirname(LIB_PATH)
INCLUDE = os.path.join(ROOT, "include")
CALLS = ("plstvo_stereo_session_run_keyframes", "plstvo_stereo_session_read_keyframes", "plstvo_default_keyframe_config",
         "plstvo_initial_keyframe_state")
STRUCTS = {"PlKeyframeConfig": T.KEYFRAME_CONFIG_DTYPE, "PlKeyframeState": T.KEYFRAME_STATE_DTYPE,
           "PlKeyframeResult": T.KEYFRAME_RESULT_DTYPE}


def build_run_kf_example(tmp_path):
    exe = str(tmp_path / "run_kf_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", INCLUDE, os.path.join(ROOT, "examples", "run_kf_cpp.cpp"),
                    "-L", LIBDIR, "-lplstvo_b200", f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_calls_are_declared_exported_and_bound():
    lib = C.CDLL(LIB_PATH)
    bound = load_library()
    for n in CALLS:
        assert hasattr(lib, n), n
        assert n in EXPORTED_SYMBOLS, n
        ret, params = declaration(n)
        fn = getattr(bound, n)
        assert len(fn.argtypes) == len(params), (n, params)
        for p, a in zip(params, fn.argtypes):
            if any(t in p for t in ("PlStereoSession", "PlContext", "PlPrior", "PlPoseResult", "PlKeyframe")):
                assert a is C.c_void_p, (n, p, a)
            elif "PlHandlerConfig" in p:
                assert a == C.POINTER(T.PlHandlerConfig), (n, p, a)
            elif "PlStereoImages" in p:
                assert a == C.POINTER(T.PlStereoImages), (n, p, a)
            elif "PlStereoFrameOut" in p:
                assert a == C.POINTER(T.PlStereoFrameOut), (n, p, a)
            elif "int32_t*" in p:
                assert a == T.c_int32_p, (n, p, a)
            elif p.startswith("int ") or p == "int":
                assert a is C.c_int, (n, p, a)
            else:
                raise AssertionError((n, p))
        assert fn.restype is (None if ret == "void" else C.c_int), (n, ret)
    # the run_keyframes call takes run's arguments, with the key-frame config after h and the state / tests beside results
    _, kf = declaration("plstvo_stereo_session_run_keyframes")
    _, run = declaration("plstvo_stereo_session_run")
    assert kf[:3] == run[:3] and kf[4:10] == run[3:9] and kf[11] == run[9] and kf[13:] == run[10:]


def test_struct_layouts_match_the_header(tmp_path):
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"plstvo.h\"\nint main(void) {\n"
    for s, dt in STRUCTS.items():
        src += f'  printf("{s} %zu\\n", sizeof({s}));\n'
        for f in dt.names:
            src += f'  printf("{s}.{f} %zu\\n", offsetof({s}, {f}));\n'
    src += "  return 0; }\n"
    c = tmp_path / "layout.c"
    c.write_text(src)
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", INCLUDE, str(c), "-o", exe], check=True)
    got = dict(ln.split() for ln in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.splitlines())
    for s, dt in STRUCTS.items():
        assert int(got[s]) == dt.itemsize, s
        for f in dt.names:
            assert int(got[f"{s}.{f}"]) == dt.fields[f][1], (s, f)


def test_default_config_and_initial_state():
    lib = load_library()
    k = np.zeros(1, T.KEYFRAME_CONFIG_DTYPE)
    lib.plstvo_default_keyframe_config(k.ctypes.data)     # src/config.cpp:40-42
    assert tuple(k[0]) == (0.85, 5.0, 15.0)
    s = np.full(1, 0xAB, np.uint8).repeat(T.KEYFRAME_STATE_DTYPE.itemsize).view(T.KEYFRAME_STATE_DTYPE)
    lib.plstvo_initial_keyframe_state(s.ctypes.data)      # initialize(), src/stereoFrameHandler.cpp:48-51
    assert s.tobytes() == KeyframeTest().to_state().tobytes()
    assert s["prev_f_iskf"][0] == 1 and s["N_prevKF_currF"][0] == 0 and s["entropy_first_prevKF"][0] == 0.0
    np.testing.assert_array_equal(s["T_prevKF"][0], np.eye(4))
    assert not s["cov_prevKF_currF"].any()
    lib.plstvo_default_keyframe_config(None)              # null pointers are ignored
    lib.plstvo_initial_keyframe_state(None)


def _odd_state(seed):
    rng = np.random.default_rng(seed)
    s = np.zeros(1, T.KEYFRAME_STATE_DTYPE)
    s["prev_f_iskf"], s["N_prevKF_currF"], s["entropy_first_prevKF"] = seed % 2, 7 + seed, -0.1 / 3.0 - seed
    s["T_prevKF"], s["cov_prevKF_currF"] = rng.standard_normal((4, 4)), rng.standard_normal((6, 6)) * 1e-7
    s["cov_prevKF_currF"][0, 1, 2] = -0.0
    return s


def test_state_round_trips_in_python():
    for seed in range(3):
        s = _odd_state(seed)
        assert KeyframeTest.from_state(s).to_state().tobytes() == s.tobytes()


def test_state_round_trips_in_cpp(tmp_path):
    src = tmp_path / "rt.cpp"
    src.write_text(r'''#include <cstdio>
#include <cstring>
#include "plstvo.hpp"
int main(int, char** argv) {
    PlKeyframeState s;
    FILE* f = std::fopen(argv[1], "rb");
    if (std::fread(&s, sizeof s, 1, f) != 1) return 2;
    std::fclose(f);
    const PlKeyframeState back = plstvo::KeyframeTest::fromState(s).state();
    PlKeyframeState init;
    plstvo_initial_keyframe_state(&init);
    const PlKeyframeState fresh = plstvo::KeyframeTest{}.state();
    const bool same = std::memcmp(&back, &s, sizeof s) == 0 && std::memcmp(&init, &fresh, sizeof s) == 0;
    std::puts(same ? "same" : "differs");
    return same ? 0 : 1;
}
''')
    exe = str(tmp_path / "rt")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", INCLUDE, str(src), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    for seed in range(3):
        p = tmp_path / f"s{seed}.bin"
        p.write_bytes(_odd_state(seed).tobytes())
        r = subprocess.run([exe, str(p)], capture_output=True, text=True)
        assert r.returncode == 0 and r.stdout.strip() == "same", r.stdout


def test_run_kf_example_compiles(tmp_path):
    assert os.path.exists(build_run_kf_example(tmp_path))


def _fma_per_line(ptx):
    """{source line: fma.rn count} of keyframe.cu's PTX."""
    counts, line = {}, None
    for ln in ptx.splitlines():
        m = re.match(r"^\s*\.loc\s+1\s+(\d+)", ln)
        if m:
            line = int(m.group(1))
        elif re.search(r"\bfma\.rn\.f64\b", ln):
            counts[line] = counts.get(line, 0) + 1
    return counts


def test_keyframe_kernel_has_no_compiler_formed_fma(tmp_path):
    """Every fma.rn of keyframe.cu is the same with and without -fmad=false, except inside CUDA's log: libdevice's log
    itself holds one plain multiply-add that nvcc contracts, and the header names log as one of the two operations that
    may differ from the host.  So each source line's count must agree, and a line where it does not must be a log call
    that differs by exactly one."""
    src = open(os.path.join(ROOT, "stvo_pl_b200", "csrc", "keyframe.cu")).read().splitlines()
    a = _fma_per_line(_ptx("keyframe.cu", str(tmp_path / "a.ptx"), []))
    b = _fma_per_line(_ptx("keyframe.cu", str(tmp_path / "b.ptx"), ["-fmad=false"]))
    assert a, "no fma.rn at all: the file was not compiled as expected"
    for line in set(a) | set(b):
        d = a.get(line, 0) - b.get(line, 0)
        if d:
            text = src[line - 1]
            assert d == 1 and re.search(r"\blog\(", text), (line, text, a.get(line), b.get(line))
