"""Host-side checks of the FLD line branch: plstvo_fld_key_lines equals the reference's own KeyLine loop
(src/stereoFrame.cpp:260-299 with sort_flines_by_length, compiled by oracle/make_ref_fld.py) byte for byte on segments with
many exact length ties, reversed endpoints, counts around n_features and endpoints on, inside and outside every border; its
numOfPixels equals cv2.clipLine's count; oracle/fld.py's RGB2GRAY equals cv2 on every 8-bit triple, with and without a
remap; the bindings of the two new calls have the header's parameter counts; and examples/fld_cpp.cpp compiles and links."""
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import fld as OF
from stvo_pl_b200.engine import EXPORTED_SYMBOLS, fld_key_lines, load_library

LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")
need_ref = pytest.mark.skipif(not OF.available(), reason="oracle/_ref/libplstvo_ref_fld.so not built (needs the reference checkout)")
KEYS = ("seg", "angle", "npix", "response", "length")


def tie_segments(rng, n, W, H):
    """n segments on a half-pixel lattice from a few (dx, dy) magnitudes, so that many lengths tie exactly; signs, the
    axis swap and the endpoint order vary, so reversed segments tie with their originals"""
    base = rng.integers(0, 24, (max(n // 6, 1), 2)) / 2.0
    out = np.zeros((n, 4), np.float32)
    for i in range(n):
        dx, dy = base[rng.integers(len(base))]
        if rng.random() < 0.5:
            dx, dy = dy, dx
        dx, dy = dx * rng.choice([-1, 1]), dy * rng.choice([-1, 1])
        x0, y0 = rng.integers(0, 2 * W) / 2.0, rng.integers(0, 2 * H) / 2.0
        s = [x0, y0, x0 + dx, y0 + dy]
        out[i] = s if rng.random() < 0.5 else s[2:] + s[:2]
    return out


def border_segments(W, H):
    """endpoints on, just inside and outside every border, and the half-pixel cases that round onto or off it"""
    xs = [-3.0, -0.75, -0.5, -0.49, 0.0, 0.49, 0.5, 1.5, W / 2, W - 1.5, W - 1.0, W - 0.51, W - 0.5, W - 0.49, W, W + 0.5, W + 4]
    ys = [-3.0, -0.75, -0.5, -0.49, 0.0, 0.5, 2.5, H / 2, H - 1.5, H - 1.0, H - 0.51, H - 0.5, H - 0.49, H, H + 0.5, H + 4]
    segs = []
    for i, x in enumerate(xs):
        for j, y in enumerate(ys):
            segs.append([x, y, xs[(i * 7 + j) % len(xs)], ys[(j * 5 + i + 3) % len(ys)]])
            segs.append([x, y, W / 3, H / 3])
            segs.append([x, y, x, ys[(j + 4) % len(ys)]])      # vertical
            segs.append([x, y, xs[(i + 5) % len(xs)], y])      # horizontal
    return np.array(segs, np.float32)


def assert_same(got, want, msg):
    for k in KEYS:
        np.testing.assert_array_equal(got[k].view(np.uint32) if got[k].dtype == np.float32 else got[k],
                                      want[k].view(np.uint32) if want[k].dtype == np.float32 else want[k], err_msg=f"{msg} {k}")


@need_ref
@pytest.mark.parametrize("W,H", [(1241, 376), (64, 48), (33, 17)])
def test_key_lines_equal_the_reference_loop(W, H):
    rng = np.random.default_rng(W * 7 + H)
    lib = load_library()
    for trial in range(40):
        n = int(rng.integers(0, 300))
        seg = tie_segments(rng, n, W, H) if trial % 2 == 0 else rng.uniform(-20, [W + 20, H + 20] * 2, (n, 4)).astype(np.float32)
        for nf in sorted({0, max(n - 1, 0), n, n + 1, max(n // 3, 1), 1}):
            want = OF.key_lines(W, H, nf, seg)
            got = fld_key_lines(W, H, nf, seg, lib)
            assert len(got["npix"]) == (n if nf == 0 else min(n, nf))
            assert_same(got, want, f"trial {trial} n {n} nf {nf}")


@need_ref
@pytest.mark.parametrize("W,H", [(1241, 376), (40, 30), (1, 1)])
def test_border_endpoints_equal_the_reference_loop(W, H):
    seg = border_segments(W, H)
    lib = load_library()
    for nf in (0, 10, len(seg)):
        assert_same(fld_key_lines(W, H, nf, seg, lib), OF.key_lines(W, H, nf, seg), f"nf {nf}")
    got = fld_key_lines(W, H, 0, seg, lib)
    assert (got["npix"] == 0).any() and (got["npix"] > 0).any()   # both sides of LineIterator's clip are exercised


def test_npix_is_cv2_cliplines_count():
    """numOfPixels on the unclamped endpoints: LineIterator rounds them (half to even), clips with clipLine where one leaves
    the image and counts max(|dx|, |dy|) + 1, or 0 when nothing is left"""
    cv2 = pytest.importorskip("cv2")
    lib = load_library()
    for W, H in ((1241, 376), (40, 30)):
        seg = np.concatenate([border_segments(W, H),
                              np.random.default_rng(3).uniform(-30, [W + 30, H + 30] * 2, (500, 4)).astype(np.float32)])
        got = fld_key_lines(W, H, 0, seg, lib)
        for s, npix in zip(seg, got["npix"]):
            p = np.rint(s).astype(np.int64)
            ok, a, b = cv2.clipLine((0, 0, W, H), (int(p[0]), int(p[1])), (int(p[2]), int(p[3])))
            want = max(abs(b[0] - a[0]), abs(b[1] - a[1])) + 1 if ok else 0
            assert npix == want, (s, npix, want)


def test_sort_only_past_n_features_and_no_clamp():
    lib = load_library()
    seg = np.array([[0, 0, 1, 0], [0, 0, 5, 0], [-4, 2, 9, 2], [0, 0, 3, 0]], np.float32)
    got = fld_key_lines(20, 10, 4, seg, lib)      # n == n_features: the caller's order, endpoints as given
    np.testing.assert_array_equal(got["seg"], seg)
    got = fld_key_lines(20, 10, 0, seg, lib)
    np.testing.assert_array_equal(got["seg"], seg)
    got = fld_key_lines(20, 10, 2, seg, lib)      # longest first, truncated
    np.testing.assert_array_equal(got["seg"], seg[[2, 1]])
    assert got["length"][0] == np.float32(13) and got["response"][0] == np.float32(13) / np.float32(20)
    np.testing.assert_array_equal(got["npix"], [10, 6])   # x -4 .. 9 clipped to 0 .. 9
    with pytest.raises(Exception):
        fld_key_lines(0, 10, 2, seg, lib)
    with pytest.raises(Exception):
        fld_key_lines(20, 10, -1, seg, lib)


def test_coordinates_outside_int_or_not_finite_are_refused():
    """cvRound leaves int (INT_MIN) where lrintf does not: such segments are refused, the edge -2^31 is kept"""
    lib = load_library()
    ok = np.array([[-2147483648.0, 5, 3, 5], [0, 0, 4, 4]], np.float32)
    assert len(fld_key_lines(20, 10, 0, ok, lib)["npix"]) == 2
    if OF.available():
        assert_same(fld_key_lines(20, 10, 0, ok, lib), OF.key_lines(20, 10, 0, ok), "edge")
    for v in (np.nan, np.inf, -np.inf, 2147483648.0, -2147483904.0, 1e30):
        bad = ok.copy()
        bad[1, 2] = v
        with pytest.raises(Exception):
            fld_key_lines(20, 10, 0, bad, lib)


# ---- the branch's fld_img of a colour frame ----
def all_triples(channels=3):
    i = np.arange(1 << 24, dtype=np.uint32)
    planes = [i & 255, (i >> 8) & 255, i >> 16] + ([(i * 2654435761) >> 24] if channels == 4 else [])
    return np.stack(planes, -1).astype(np.uint8).reshape(4096, 4096, channels)


def test_rgb2gray_equals_cv2_on_every_triple():
    cv2 = pytest.importorskip("cv2")
    for ch in (3, 4):
        img = all_triples(ch)
        want = OF.rgb_to_gray(img)
        np.testing.assert_array_equal(cv2.cvtColor(img, cv2.COLOR_RGB2GRAY), want)
        # the same fixed point as BGR2GRAY on the channel-reversed image
        np.testing.assert_array_equal(want, cv2.cvtColor(np.ascontiguousarray(img[..., 2::-1]), cv2.COLOR_BGR2GRAY))


def test_remap_then_rgb2gray_equals_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(29)
    for k in range(8):
        w, h, ch = int(rng.integers(1, 90)), int(rng.integers(1, 60)), 3 + k % 2
        mx = rng.uniform(-4, w + 3, (h, w)).astype(np.float32)
        my = rng.uniform(-4, h + 3, (h, w)).astype(np.float32)
        m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        img = rng.integers(0, 256, (h, w, ch), dtype=np.uint8)
        want = cv2.cvtColor(cv2.remap(img, m1, m2, cv2.INTER_LINEAR), cv2.COLOR_RGB2GRAY)
        np.testing.assert_array_equal(OF.remap_gray_rgb(img, m1, m2), want, err_msg=str(k))
        np.testing.assert_array_equal(OF.remap_gray_rgb(img), cv2.cvtColor(img, cv2.COLOR_RGB2GRAY))


# ---- bindings and example ----
def test_bindings_match_the_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "plstvo.h")).read(), flags=re.S)
    lib = load_library()
    for name in ("plstvo_fld_key_lines", "plstvo_stereo_session_use_fld_lines"):
        assert name in EXPORTED_SYMBOLS
        m = re.search(name + r"\s*\(([^)]*)\)", txt)
        assert m and len(getattr(lib, name).argtypes) == m.group(1).count(",") + 1, name
    assert "def use_fld_lines" in open(os.path.join(ROOT, "stvo_pl_b200", "engine.py")).read()
    hpp = open(os.path.join(ROOT, "include", "plstvo.hpp")).read()
    assert "plstvo_fld_key_lines(" in hpp and "plstvo_stereo_session_use_fld_lines(" in hpp


def test_example_compiles_and_links(tmp_path):
    exe = str(tmp_path / "fld_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "fld_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200", f"-Wl,-rpath,{LIBDIR}",
                    "-o", exe], check=True)
    assert os.path.exists(exe)
