"""oracle/plot.py (plotStereoFrame's drawing) held to OpenCV: to live cv2 where it is importable, exhaustively on small
canvases (every circle centre, every segment between end points on a grid around the image, both orders), on float end
points that int() truncates toward zero, on cvtColor GRAY2BGR / BGRA2BGR, on cv2.remap of 3- and 4-channel images and on a
KITTI-size frame with 2000 points and 300 lines; and to tests/golden/plot.npz (cv2 4.13, tools/make_plot_golden.py), which
reproduces from its generator.  Also: examples/plot_cpp.cpp compiles with -Wall -Werror and the two plot calls are bound."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import color as OC
from oracle import plot as P
from stvo_pl_b200.engine import EXPORTED_SYMBOLS

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_color_golden as MC  # noqa: E402
import make_plot_golden as MP  # noqa: E402

G = np.load(os.path.join(GOLDEN, "plot.npz"))
LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")


def line_mask(w, h, p, q):
    m = np.zeros((h, w), bool)
    for x, y in P.line_pixels(p[0], p[1], q[0], q[1], w, h):
        m[y, x] = True
    return m


def circle_mask(w, h, c):
    m = np.zeros((h, w), bool)
    for x, y in P.circle_pixels(c[0], c[1], w, h):
        m[y, x] = True
    return m


# ---- the golden ----
def test_golden_grid_and_circles():
    hl = hashlib.sha256()
    for w, h in MP.GRID:
        pts = MP.grid_points(w, h, 4)
        for p in pts:
            for q in pts:
                hl.update(np.packbits(line_mask(w, h, p, q)).tobytes())
    assert hl.hexdigest() == str(G["grid_sha"])
    hc = hashlib.sha256()
    for c in MP.grid_points(9, 7, 3):
        hc.update(np.packbits(circle_mask(9, 7, c)).tobytes())
    assert hc.hexdigest() == str(G["circle_sha"])


def test_golden_kitti_frame():
    base, pl, spl, epl = MP.kitti_inputs(int(G["kitti_seed"]))
    np.testing.assert_array_equal(pl, G["kitti_pl"])
    np.testing.assert_array_equal(spl, G["kitti_spl"])
    np.testing.assert_array_equal(epl, G["kitti_epl"])
    W, H = MP.KITTI
    want = base.copy()
    want[np.unpackbits(G["kitti_mask"])[:W * H].reshape(H, W).astype(bool)] = P.COLOUR
    np.testing.assert_array_equal(P.plot_stereo_frame(base, pl, spl, epl), want)


@pytest.mark.parametrize("channels", [3, 4])
def test_golden_remap(channels):
    src = MC.color_image(int(G[f"remap{channels}_seed"]), 64, 48, channels)
    got = P.base_image(src, (G[f"remap{channels}_map1"], G[f"remap{channels}_map2"]))
    np.testing.assert_array_equal(got, G[f"remap{channels}_out"])


def test_golden_reproduces_from_its_generator():
    pytest.importorskip("cv2")
    g = MP.build()
    assert sorted(g) == sorted(G.files)
    for k in G.files:
        np.testing.assert_array_equal(g[k], G[k], err_msg=k)


# ---- live cv2 ----
def test_every_circle_centre_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    for c in MP.grid_points(9, 7, 3):
        img = np.zeros((7, 9, 3), np.uint8)
        cv2.circle(img, c, 3, P.COLOUR, 1)
        np.testing.assert_array_equal(img[..., 1] == 200, circle_mask(9, 7, c), err_msg=str(c))


@pytest.mark.parametrize("size", [(9, 7), (5, 4), (1, 1), (3, 8), (2, 1), (16, 3)])
def test_every_grid_segment_equals_cv2(size):
    cv2 = pytest.importorskip("cv2")
    w, h = size
    pts = MP.grid_points(w, h, 4)
    for p in pts:
        for q in pts:
            img = np.zeros((h, w, 3), np.uint8)
            cv2.line(img, p, q, P.COLOUR, 1)
            assert np.array_equal(img[..., 1] == 200, line_mask(w, h, p, q)), (p, q)


def test_end_point_order_matters_and_is_kept():
    """segments leaving the image: cv2's pixels depend on which end comes first, and the oracle follows both orders"""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    differ = 0
    for _ in range(3000):
        p, q = tuple(int(v) for v in rng.integers(-6, 14, 2)), tuple(int(v) for v in rng.integers(-6, 14, 2))
        a, b = line_mask(9, 7, p, q), line_mask(9, 7, q, p)
        differ += not np.array_equal(a, b)
        for s, e, m in ((p, q, a), (q, p, b)):
            img = np.zeros((7, 9, 3), np.uint8)
            cv2.line(img, s, e, P.COLOUR, 1)
            assert np.array_equal(img[..., 1] == 200, m), (s, e)
    assert differ > 0


def test_float_end_points_truncate_toward_zero():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    vals = np.concatenate([rng.uniform(-0.5, 0, 40), rng.uniform(-3, 12, 200), [-0.49999, -1e-12, -0.0, 0.999, 8.9999]])
    for _ in range(400):
        s, e, c = rng.choice(vals, 2), rng.choice(vals, 2), rng.choice(vals, 2)
        img = np.zeros((7, 9, 3), np.uint8)
        cv2.circle(img, (int(c[0]), int(c[1])), 3, P.COLOUR, 1)
        cv2.line(img, (int(s[0]), int(s[1])), (int(e[0]), int(e[1])), P.COLOUR, 1)
        got = P.plot_stereo_frame(np.zeros((7, 9, 3), np.uint8), [c], [s], [e])
        np.testing.assert_array_equal(got, img)
    assert P.trunc(-0.4) == 0 and P.trunc(-1.6) == -1 and P.trunc(2.9) == 2


def test_cvtcolor_gray2bgr_bgra2bgr():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    g = rng.integers(0, 256, (23, 37), dtype=np.uint8)
    np.testing.assert_array_equal(P.gray2bgr(g), cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))
    a = rng.integers(0, 256, (23, 37, 4), dtype=np.uint8)
    np.testing.assert_array_equal(P.bgra2bgr(a), cv2.cvtColor(a, cv2.COLOR_BGRA2BGR))
    np.testing.assert_array_equal(P.base_image(g), cv2.cvtColor(g, cv2.COLOR_GRAY2BGR))
    np.testing.assert_array_equal(P.base_image(a), cv2.cvtColor(a, cv2.COLOR_BGRA2BGR))
    np.testing.assert_array_equal(P.base_image(a[..., :3]), a[..., :3])


@pytest.mark.parametrize("channels", [1, 3, 4])
def test_base_image_remap_equals_cv2(channels):
    cv2 = pytest.importorskip("cv2")
    for w, h, seed in ((37, 23, 1), (64, 48, 2), (17, 1, 3)):
        src = MC.color_image(seed, w, h, max(channels, 3))
        if channels == 1:
            src = OC.bgr_to_gray(src)
        m1, m2 = MC.own_maps(w, h, seed)
        r = cv2.remap(src, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        want = {1: lambda x: cv2.cvtColor(x, cv2.COLOR_GRAY2BGR), 3: lambda x: x,
                4: lambda x: cv2.cvtColor(x, cv2.COLOR_BGRA2BGR)}[channels](r)
        np.testing.assert_array_equal(P.base_image(src, (m1, m2)), want)


def test_kitti_frame_equals_cv2():
    pytest.importorskip("cv2")
    base, pl, spl, epl = MP.kitti_inputs(99)
    np.testing.assert_array_equal(P.plot_stereo_frame(base, pl, spl, epl), MP.cv2_plot(base, pl, spl, epl))


# ---- bindings and the example ----
def test_plot_calls_are_bound():
    assert "plstvo_stereo_session_plot" in EXPORTED_SYMBOLS and "plstvo_stereo_session_read_plot" in EXPORTED_SYMBOLS


def test_plot_example_compiles(tmp_path):
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "plot_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200", f"-Wl,-rpath,{LIBDIR}",
                    "-o", str(tmp_path / "plot_cpp")], check=True)
