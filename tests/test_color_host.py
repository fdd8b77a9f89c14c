"""Host-side checks of colour input: oracle/color.py equals live cv2 4.13 on every 8-bit BGR triple (and on BGRA), on remapped
3- and 4-channel images under tests/golden/color.npz's maps and a seeded sweep of rigs; the golden matches the restatement;
plstvo_rectifier_create_color's ctypes signature has the header's parameter count and the library exports it; and
examples/color_images_cpp.cpp compiles and links with -Wall -Werror."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import color as OC
from stvo_pl_b200.engine import EXPORTED_SYMBOLS, init_undistort_rectify_map, load_library

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_color_golden as MC  # noqa: E402
import make_rectify_golden as M  # noqa: E402

LIBDIR = os.path.join(ROOT, "stvo_pl_b200", "lib")
G = np.load(os.path.join(GOLDEN, "color.npz"))
GR = np.load(os.path.join(GOLDEN, "rectify.npz"))


def all_triples(channels=3, seed=None):
    """uint8[4096, 4096, channels] holding each BGR triple once (B the low byte of the pixel index), alpha seeded"""
    i = np.arange(1 << 24, dtype=np.uint32)
    planes = [i & 255, (i >> 8) & 255, i >> 16]
    if channels == 4:
        planes.append(np.random.default_rng(seed).integers(0, 256, 1 << 24, dtype=np.uint32))
    return np.stack(planes, -1).astype(np.uint8).reshape(4096, 4096, channels)


def case_maps(c):
    """(map1, map2) of golden case c, or (None, None) for the conversion alone; rectify.npz's rig maps from the library's
    builder, held to that golden's SHA-256"""
    rig = str(G[f"{c}_rig"])
    if rig == "-":
        return None, None
    if rig == "":
        return G[f"{c}_map1"], G[f"{c}_map2"]
    if f"{rig}_map1" in GR:
        return GR[f"{rig}_map1"], GR[f"{rig}_map2"]
    w, h = (int(v) for v in GR[f"{rig}_size"])
    m1, m2 = init_undistort_rectify_map(int(GR[f"{rig}_model"]), GR[f"{rig}_K"], GR[f"{rig}_D"], GR[f"{rig}_R"], GR[f"{rig}_P"],
                                        w, h)
    assert (M.sha(m1, m2) == GR[f"{rig}_map_sha"]).all(), rig
    return m1, m2


def case_image(c, seed=None):
    w, h = (int(v) for v in G[f"{c}_size"])
    return MC.color_image(int(G[f"{c}_seed"]) if seed is None else seed, w, h, int(G[f"{c}_channels"]))


def assert_golden(c, grey):
    if f"{c}_out" in G:
        np.testing.assert_array_equal(grey, G[f"{c}_out"], err_msg=c)
    else:
        assert (M.sha(grey) == G[f"{c}_out_sha"]).all(), c


def build_color_example(tmp_path):
    exe = str(tmp_path / "color_images_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "color_images_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


# ---- the conversion ----
def test_conversion_equals_cv2_on_every_triple():
    cv2 = pytest.importorskip("cv2")
    img = all_triples()
    want = OC.bgr_to_gray(img)
    use_ipp = cv2.ipp.useIPP()
    try:
        for ipp in (True, False):
            cv2.ipp.setUseIPP(ipp)
            np.testing.assert_array_equal(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), want)
    finally:
        cv2.ipp.setUseIPP(use_ipp)
    bgra = all_triples(4, seed=11)
    np.testing.assert_array_equal(OC.bgr_to_gray(bgra), want)
    np.testing.assert_array_equal(cv2.cvtColor(bgra, cv2.COLOR_BGR2GRAY), want)
    # the 14-bit coefficients quoted for BGR2GRAY give other values: the exhaustive check tells coefficient sets apart
    b, g, r = (img[..., c].astype(np.int64) for c in range(3))
    q14 = ((1868 * b + 9617 * g + 4899 * r + (1 << 13)) >> 14).astype(np.uint8)
    assert int((q14 != want).sum()) == 43864


def test_grey_replicated_into_bgr_converts_back():
    v = np.arange(256, dtype=np.uint8)
    np.testing.assert_array_equal(OC.bgr_to_gray(np.stack([v, v, v], -1)), v)
    assert OC.B2Y + OC.G2Y + OC.R2Y == 1 << OC.SHIFT


# ---- the remap, then the conversion ----
def test_remap_then_convert_equals_cv2_on_golden_maps():
    cv2 = pytest.importorskip("cv2")
    for c in G["cases"]:
        m1, m2 = case_maps(c)
        img = case_image(c, seed=5000 + len(c))
        src = img if m1 is None else cv2.remap(img, m1, m2, cv2.INTER_LINEAR)
        np.testing.assert_array_equal(OC.remap_gray(img, m1, m2), cv2.cvtColor(src, cv2.COLOR_BGR2GRAY), err_msg=c)


def test_remap_then_convert_equals_cv2_on_a_sweep():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(23)
    for k in range(12):
        w, h = int(rng.integers(1, 90)), int(rng.integers(1, 60))
        channels = 3 + k % 2
        if k % 3 == 0:   # a pinhole or fisheye rig
            model = k % 2
            K = np.array([[0.9 * w + 5, 0, w / 2 + rng.uniform(-2, 2)], [0, 0.9 * w + 5, h / 2 + rng.uniform(-2, 2)], [0, 0, 1]])
            D = rng.normal(0, 0.1, 4) * np.array([1, 0.3, 0.01, 0.01])
            P = np.hstack([K * rng.uniform(0.8, 1.2), np.zeros((3, 1))])
            P[2] = [0, 0, 1, 0]
            build = cv2.fisheye.initUndistortRectifyMap if model == 1 else cv2.initUndistortRectifyMap
            m1, m2 = build(K, D, np.eye(3), P, (w, h), cv2.CV_16SC2)
        else:
            mx = rng.uniform(-4, w + 3, (h, w)).astype(np.float32)
            my = rng.uniform(-4, h + 3, (h, w)).astype(np.float32)
            m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        img = MC.color_image(300 + k, w, h, channels)
        want = cv2.cvtColor(cv2.remap(img, m1, m2, cv2.INTER_LINEAR), cv2.COLOR_BGR2GRAY)
        np.testing.assert_array_equal(OC.remap_gray(img, m1, m2), want, err_msg=str(k))


def test_order_matters_on_the_euroc_map():
    """converting first and remapping the grey image is not what the reference does: it differs by 1 on many pixels"""
    m1, m2 = case_maps("c3_euroc_l")
    img = case_image("c3_euroc_l")
    a = OC.remap_gray(img, m1, m2)
    b = OC.R.remap(OC.bgr_to_gray(img), m1, m2)
    d = np.abs(a.astype(int) - b.astype(int))
    assert d.max() == 1 and (d > 0).sum() > 0.1 * d.size, ((d > 0).sum(), d.size)


def test_golden_matches_restatement():
    assert len(G["cases"]) > 100
    for c in G["cases"]:
        m1, m2 = case_maps(c)
        assert_golden(c, OC.remap_gray(case_image(c), m1, m2))


# ---- bindings and the example ----
def test_create_color_signature_and_export():
    header = open(os.path.join(ROOT, "include", "plstvo.h")).read()
    lib = load_library()
    decl = re.search(r"\bPlRectifier\*\s+plstvo_rectifier_create_color\s*\(([^;]*)\)\s*;", header).group(1)
    params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", decl, flags=re.S).split(",")]
    assert len(lib.plstvo_rectifier_create_color.argtypes) == len(params) == 8, params
    assert params[3] == "int channels", params
    assert "plstvo_rectifier_create_color" in EXPORTED_SYMBOLS


def test_color_example_compiles_and_links(tmp_path):
    build_color_example(tmp_path)
