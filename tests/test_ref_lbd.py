"""The LBD reference library (oracle/make_ref_lbd.py) on the CPU: its stand-in blur and Sobel equal cv2's bit for bit, it
reproduces tests/golden/lbd.npz, the golden tool regenerates that file, and the cos / sin overload it binds is the one
the library evaluates."""
import ctypes
import ctypes.util
import math
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import orb_images as I

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_lbd_golden as M  # noqa: E402

from oracle import lbd  # noqa: E402

need_ref = pytest.mark.skipif(not lbd.available(), reason="oracle/_ref/libplstvo_ref_lbd.so not built (needs the reference checkout)")
SIZES = [(w, h) for w in range(1, 9) for h in range(1, 9)] + [(9, 13), (17, 5), (63, 17), (64, 16), (65, 33), (131, 77), (640, 480)]


def _golden():
    return np.load(os.path.join(GOLDEN, "lbd.npz"))


@need_ref
@pytest.mark.parametrize("W,H", SIZES)
def test_standin_blur_sobel_equal_cv2(W, H):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(W * 1000 + H)
    for img in (rng.integers(0, 256, (H, W), dtype=np.uint8), I.make_image(W, H, W + H) if W * H > 1 else np.uint8([[7]])):
        b, dx, dy = lbd.blur_sobel(img)
        ref = cv2.GaussianBlur(img, (5, 5), 1)
        np.testing.assert_array_equal(b, ref)
        np.testing.assert_array_equal(dx, cv2.Sobel(ref, cv2.CV_16S, 1, 0, ksize=3))
        np.testing.assert_array_equal(dy, cv2.Sobel(ref, cv2.CV_16S, 0, 1, ksize=3))


@need_ref
def test_reference_equals_golden():
    g = _golden()
    for name in g["cases"]:
        images, off, seg, ang, npix, desc = M.load_case(g, str(name))
        np.testing.assert_array_equal(lbd.compute_batch(images, off, seg, ang, npix), desc, err_msg=str(name))


@need_ref
def test_golden_tool_regenerates_the_file():
    pytest.importorskip("cv2")
    g, new = _golden(), M.golden()
    assert sorted(g.files) == sorted(new.keys())
    for k in g.files:
        if k != "cv2_version":
            np.testing.assert_array_equal(g[k], new[k], err_msg=k)


@need_ref
def test_lbd_host_path_takes_the_float_trig_overload():
    """The reference's translation unit includes <math.h> (bitarray_custom.hpp:52), whose C++ form puts std::cos(float) /
    std::sin(float) into the global namespace: its unqualified cos(float) / sin(float) call the C library's cosf / sinf
    (merged into sincosf).  The stand-in reproduces that, and the host source that enqueues LBD (lbd_enqueue) evaluates the
    line direction with the same function."""
    assert lbd.trig_binding() == "float"
    csrc = os.path.join(ROOT, "stvo_pl_b200", "csrc")
    srcs = [open(os.path.join(csrc, f)).read() for f in sorted(os.listdir(csrc)) if f.endswith(".cu")]
    (host,) = [s for s in srcs if "int lbd_enqueue(" in s]
    assert "sincosf(kl_angle[k]" in host


def test_trig_binding_case_depends_on_the_binding():
    """Every line of the golden's trig_binding case has an angle where glibc's cosf / sinf differ from the double functions
    rounded to float, so a build that took the other overload fails that case."""
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.cosf.restype = libm.sinf.restype = ctypes.c_float
    libm.cosf.argtypes = libm.sinf.argtypes = [ctypes.c_float]
    angles = _golden()["trig_binding/angle_bits"].view(np.float32)
    assert len(angles) >= 5
    for a in angles:
        f = (libm.cosf(float(a)), libm.sinf(float(a)))
        d = (float(np.float32(math.cos(float(a)))), float(np.float32(math.sin(float(a)))))
        assert f != d, a


def test_reference_coefficient_tables():
    """The reference constructor's gaussCoefL_ / gaussCoefG_ are exp() in double of integer-divided centres and sigmas, the
    recipe capi_features.cu's lbd_init follows for the kernel's float tables (which the GPU goldens exercise)."""
    if not lbd.available():
        pytest.skip("oracle/_ref/libplstvo_ref_lbd.so not built (needs the reference checkout)")
    cl, cg = lbd.coefficients()
    u, s = (7 * 3 - 1) // 2, (7 * 2 + 1) // 2
    np.testing.assert_array_equal(cl, [math.exp((i - u) * (i - u) * (-1 / (2.0 * s * s))) for i in range(21)])
    u = (9 * 7 - 1) // 2
    np.testing.assert_array_equal(cg, [math.exp((i - u) * (i - u) * (-1 / (2.0 * u * u))) for i in range(63)])
