"""Every fused multiply-add in a byte-exact kernel is written out (CPU; needs nvcc, no GPU).

The stereo step, the lifting, LBD and ORB promise the bytes of the reference source evaluated unfused (DESIGN.md §4).  nvcc
contracts a plain `a * b + c` into an FMA unless told not to, which rounds once where the reference rounds twice and can
flip a threshold test (match_grid.cu's line direction filter once did exactly that).  So each file is compiled to PTX with
build.py's flags twice, as is and with -fmad=false: the count of fma.rn per kernel must not change, i.e. every FMA left
in the code is one the source spells (__fma_rn / fma), never one the compiler formed."""
import os
import re
import subprocess

import pytest

from stvo_pl_b200 import build as B

BYTE_EXACT = ["match_grid.cu", "lift.cu", "lbd.cu", "orb.cu"]


def _ptx(src, out, extra):
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    cmd = [B.nvcc()] + flags + extra + ["-ptx", "-o", out, os.path.join(B.CSRC, src)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    with open(out) as f:
        return f.read()


def fma_per_function(ptx: str) -> dict:
    """{kernel or device function name: number of fma.rn instructions in its body}."""
    counts, name = {}, None
    for line in ptx.splitlines():
        m = re.match(r"^\s*(?:\.visible\s+|\.weak\s+)?\.(?:entry|func)\s+(?:\([^)]*\)\s*)?([\w$]+)", line)
        if m:
            name = m.group(1)
            counts.setdefault(name, 0)
        elif name is not None and re.search(r"\bfma\.rn(\.ftz)?(\.sat)?\.f(32|64)\b", line):
            counts[name] += 1
    return counts


@pytest.mark.parametrize("src", BYTE_EXACT)
def test_no_compiler_formed_fma(src, tmp_path):
    as_is = fma_per_function(_ptx(src, str(tmp_path / "a.ptx"), []))
    unfused = fma_per_function(_ptx(src, str(tmp_path / "b.ptx"), ["-fmad=false"]))
    assert as_is, f"{src}: no kernel found in the PTX"
    assert set(as_is) == set(unfused), (src, sorted(set(as_is) ^ set(unfused)))
    diff = {k: (as_is[k], unfused[k]) for k in as_is if as_is[k] != unfused[k]}
    assert not diff, f"{src}: nvcc contracted a * b + c into an FMA in {diff} (as is, -fmad=false)"


def test_the_audit_sees_a_contraction(tmp_path):
    """The audit itself: a kernel with a plain double dot product does show up."""
    src = tmp_path / "dot.cu"
    src.write_text("__global__ void k(const double* a, double* o) { o[0] = a[0] * a[1] + a[2] * a[3]; }\n")
    flags = [f for f in B.NVCC_FLAGS if not f.startswith("--use_fast_math")]
    out = {}
    for tag, extra in (("as_is", []), ("unfused", ["-fmad=false"])):
        p = str(tmp_path / f"{tag}.ptx")
        r = subprocess.run([B.nvcc()] + flags + extra + ["-ptx", "-o", p, str(src)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        out[tag] = fma_per_function(open(p).read())
    (name,) = out["as_is"]
    assert out["as_is"][name] == 1 and out["unfused"][name] == 0
