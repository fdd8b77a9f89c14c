"""lsd.cu, like the other byte-exact kernels, holds no FMA the compiler formed (CPU; needs nvcc, no GPU): its PTX has the
same fma.rn count per function with and without -fmad=false."""
from test_fp_contraction import _ptx, fma_per_function


def test_lsd_has_no_compiler_formed_fma(tmp_path):
    as_is = fma_per_function(_ptx("lsd.cu", str(tmp_path / "a.ptx"), []))
    unfused = fma_per_function(_ptx("lsd.cu", str(tmp_path / "b.ptx"), ["-fmad=false"]))
    assert any("lsd_grow_kernel" in k for k in as_is), sorted(as_is)
    assert as_is == unfused, {k: (as_is.get(k), unfused.get(k)) for k in set(as_is) | set(unfused)
                              if as_is.get(k) != unfused.get(k)}
