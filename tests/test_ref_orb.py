"""The ORB description oracle (oracle/orb_oracle.c) stage by stage against cv2 when cv2 is importable, and always against
the committed goldens (tests/golden/orb_*.npz, written by tools/make_orb_golden.py from cv2 4.13)."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import orb_images as I

sys.path.insert(0, os.path.join(ROOT, "tools"))


@pytest.fixture(scope="module")
def orb():
    from oracle.orb import OrbOracle
    return OrbOracle()


def _cv2():
    return pytest.importorskip("cv2")


def _golden_images(name):
    import make_orb_golden as M
    return M.default_images() if name == "orb_default" else M.kitti_views()


# ---- against the goldens (no cv2 needed) ----
@pytest.mark.parametrize("name", ["orb_default", "orb_kitti"])
def test_golden_images_regenerate(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    assert [I.sha256(im) for im in _golden_images(name)] == list(z["sha256"])


@pytest.mark.parametrize("name", ["orb_default", "orb_kitti"])
def test_oracle_equals_golden(orb, name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    imgs, nl, s = _golden_images(name), int(z["n_levels"]), float(z["scale"])
    ang, desc, src, cnt = orb.compute_batch(imgs, z["det_off"], z["det_xy"], z["det_oct"], None, n_levels=nl, scale=s)
    np.testing.assert_array_equal(cnt, np.diff(z["det_off"]))                 # ORB's own key points all survive
    np.testing.assert_array_equal(ang.view(np.uint32), z["det_angle_bits"])
    np.testing.assert_array_equal(desc, z["det_desc"])
    ang, desc, src, cnt = orb.compute_batch(imgs, z["given_off"], z["given_xy"], z["given_oct"],
                                            z["given_angle_bits"].view(np.float32), n_levels=nl, scale=s, threads=2)
    np.testing.assert_array_equal(cnt, z["given_counts"])
    off = z["given_off"]
    rows = np.concatenate([np.arange(off[i], off[i] + cnt[i]) for i in range(len(cnt))])
    np.testing.assert_array_equal(src[rows], z["given_src_idx"])
    np.testing.assert_array_equal(desc[rows], z["given_desc"])
    np.testing.assert_array_equal(ang[rows].view(np.uint32), z["given_angle_bits"][off[:-1].repeat(cnt) + src[rows]])


def test_pattern_header_matches_generator_format():
    import gen_orb_pattern as G
    t = G.read_header()
    assert t.shape == (256, 4) and t.min() >= -15 and t.max() <= 15
    assert G.render(t) == open(G.HEADER).read()


# ---- stage by stage against cv2 ----
def test_pattern_rederives():
    _cv2()
    import gen_orb_pattern as G
    np.testing.assert_array_equal(G.derive(), G.read_header())


def test_level_sizes(orb):
    for W, H in [(1241, 376), (640, 480), (333, 251), (41, 39)]:
        for s in (1.2, 2.0, 1.5):
            for lvl in range(8):
                assert orb.level_size(W, H, s, lvl) == I.level_size(W, H, s, lvl)


def test_resize_equals_cv2(orb):
    cv2 = _cv2()
    rng = np.random.default_rng(0)
    for t in range(200):
        sw, sh = (int(v) for v in rng.integers(2, 260, 2))
        s = (1.2, 2.0, 1.5, 1.1)[t % 4]
        dw, dh = max(1, int(round(sw / s))), max(1, int(round(sh / s)))
        img = rng.integers(0, 256, (sh, sw), dtype=np.uint8)
        np.testing.assert_array_equal(orb.resize(img, dw, dh), cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR_EXACT))


def test_blur_equals_cv2_float_path(orb):
    """ORB blurs a sub-matrix of its pyramid buffer, so GaussianBlur takes sepFilter2D's float path; cv2.sepFilter2D with
    the same taps on a whole image takes that path too (cv2.GaussianBlur would take the fixed-point one)."""
    cv2 = _cv2()
    k = cv2.getGaussianKernel(7, 2, ktype=cv2.CV_32F)
    rng = np.random.default_rng(1)
    for _ in range(60):
        w, h = (int(v) for v in rng.integers(1, 300, 2))
        img = rng.integers(0, 256, (h, w), dtype=np.uint8)
        np.testing.assert_array_equal(orb.blur(img), cv2.sepFilter2D(img, -1, k, k, borderType=cv2.BORDER_REFLECT_101))
    img = I.make_image(400, 300, 3)
    assert not np.array_equal(orb.blur(img), cv2.GaussianBlur(img, (7, 7), 2, sigmaY=2, borderType=cv2.BORDER_REFLECT_101))


def test_fast_atan2_equals_cv2(orb):
    cv2 = _cv2()
    rng = np.random.default_rng(2)
    g = np.arange(-120, 121)
    ys, xs = np.meshgrid(g, g)
    ys = np.concatenate([ys.ravel(), rng.integers(-1_100_000, 1_100_000, 60000)])
    xs = np.concatenate([xs.ravel(), rng.integers(-1_100_000, 1_100_000, 60000)])
    a = np.array([orb.fast_atan2(float(y), float(x)) for y, x in zip(ys, xs)], np.float32)
    b = np.array([cv2.fastAtan2(float(y), float(x)) for y, x in zip(ys, xs)], np.float32)
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


CONFIGS = [(640, 480, 4, 1.2), (1241, 376, 1, 1.2), (333, 251, 4, 2.0), (301, 199, 8, 1.2), (97, 61, 2, 1.2)]


@pytest.mark.parametrize("W,H,nl,s", CONFIGS)
def test_compute_equals_cv2(orb, W, H, nl, s):
    """ORB::compute with given angles (random, and the axis / diagonal angles) and detectAndCompute (computed angles)."""
    cv2 = _cv2()
    o = cv2.ORB_create(1200, s, nl, 19, 0, 2, cv2.ORB_FAST_SCORE, 31, 20)
    for seed in (1, 2):
        img = I.make_image(W, H, seed + W)
        xy, oct_, ang = I.make_keypoints(W, H, 1200, nl, s, seed)
        ang[:24] = np.float32([0, 90, 180, 270, 359.99, 45, 44.99, 45.01, 135, 225, 315, 1e-3] * 2)
        order = np.argsort(oct_, kind="stable")
        xy, oct_, ang = xy[order], oct_[order], ang[order]
        out, d = o.compute(img, [cv2.KeyPoint(float(x), float(y), 31, float(a), 0, int(q), -1)
                                 for (x, y), a, q in zip(xy, ang, oct_)])
        a2, d2, src, cnt = orb.compute_batch(img[None], [0, len(xy)], xy, oct_, ang, n_levels=nl, scale=s)
        assert cnt[0] == len(out)
        np.testing.assert_array_equal(d2[:cnt[0]], np.asarray(d).reshape(-1, 32))
        kps, d = o.detectAndCompute(img, None)
        if not kps:
            continue
        xy = np.array([k.pt for k in kps], np.float32)
        a2, d2, src, cnt = orb.compute_batch(img[None], [0, len(xy)], xy, [k.octave for k in kps], None, n_levels=nl, scale=s)
        assert cnt[0] == len(kps)
        np.testing.assert_array_equal(a2.view(np.uint32), np.array([k.angle for k in kps], np.float32).view(np.uint32))
        np.testing.assert_array_equal(d2, d)


def test_border_filter_equals_cv2(orb):
    """runByImageBorder tests cvRound(pt): with edge 19, x = 18 and 18.5 (rounds to 18) are dropped, 18.51 and 19 kept;
    key points near the edge at every level, at angles near 45 degrees, read the unblurred border the same way."""
    cv2 = _cv2()
    import make_orb_golden as M
    W, H = 320, 240
    img = I.make_image(W, H, 9)
    xy = M.border_keypoints(W, H)
    n0 = len(xy)
    lvl_xy = [(19.0, 19.0), (19.0, H - 20.0), (W - 20.0, 19.0), (W - 20.0, H - 20.0)]
    xy = np.concatenate([xy] + [np.float32(lvl_xy)] * 4)
    oct_ = np.concatenate([np.zeros(n0, np.int32)] + [np.full(4, q, np.int32) for q in range(4)])
    for base in (0.0, 44.99, 45.0, 45.01, 134.99, 225.01):
        ang = np.full(len(xy), base, np.float32)
        o = cv2.ORB_create(1200, 1.2, 4, 19, 0, 2, cv2.ORB_FAST_SCORE, 31, 20)
        out, d = o.compute(img, [cv2.KeyPoint(float(x), float(y), 31, float(a), 0, int(q), -1) for (x, y), a, q in zip(xy, ang, oct_)])
        a2, d2, src, cnt = orb.compute_batch(img[None], [0, len(xy)], xy, oct_, ang, n_levels=4, scale=1.2)
        assert cnt[0] == len(out)
        np.testing.assert_array_equal(xy[src[:cnt[0]]], np.array([k.pt for k in out], np.float32))
        np.testing.assert_array_equal(d2[:cnt[0]], d)
