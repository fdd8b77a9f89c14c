"""The LSD restatement (oracle/lsd_oracle.cpp) on the CPU: it reproduces tests/golden/lsd.npz bit for bit (cv2 4.13's
segments and the reference's key lines), each fixed-point stage equals cv2's on its own, the seed-order decision rests on
images that separate the two candidates, and the golden tool regenerates the file."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import orb_images as I

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_lsd_golden as M  # noqa: E402

from oracle import lsd  # noqa: E402

SIZES = [(w, h) for w in range(1, 9) for h in range(1, 9)] + [(9, 13), (17, 5), (63, 17), (131, 77), (1241, 376)]
O = lsd.LsdOracle()


def _golden():
    return np.load(os.path.join(GOLDEN, "lsd.npz"))


def _cases():
    return [str(c) for c in _golden()["cases"]]


def _raw_args(P):
    return P["scale"], P["sigma_scale"], P["quant"], P["ang_th"], P["n_bins"]


@pytest.mark.parametrize("name", _cases())
def test_restatement_equals_golden(name):
    imgs, P, raw, raw_off, kl = M.load_case(_golden(), name)
    H, W = imgs.shape[1:]
    for i, img in enumerate(imgs):
        np.testing.assert_array_equal(O.segments(img, *_raw_args(P)), raw[raw_off[i]:raw_off[i + 1]], err_msg=f"{name}[{i}]")
        got = O.detect(img, *_raw_args(P), P["min_line_length"], P["n_features"])
        for f in ("seg", "angle", "npix", "response", "length"):
            np.testing.assert_array_equal(got[f], kl[f][kl["off"][i]:kl["off"][i + 1]], err_msg=f"{name}[{i}].{f}")


def test_golden_covers_the_edges():
    g = _golden()
    P = {n: M.load_case(g, n)[1] for n in _cases()}
    # every accepted parameter at a value other than the shipped one
    for k, v in lsd.SHIPPED.items():
        assert any(p[k] != v for p in P.values()), k
    assert P["other_b"]["scale"] == 1 and P["other_a"]["scale"] < 1
    assert len(g["flat/raw"]) == 0 and len(g["kitti_300/raw"]) > 600
    # ties in response decide the truncation: the first dropped line has the last kept line's response
    imgs, p, raw, raw_off, kl = M.load_case(g, "ties")
    full = O.keylines_from_segments(imgs.shape[2], imgs.shape[1], raw, p["min_line_length"], 0)
    r = np.sort(full["response"])[::-1]
    assert r[p["n_features"] - 1] == r[p["n_features"]]
    # lines along the border: endpoints within about two pixels of every side
    _, _, raw, _, _ = M.load_case(g, "border")
    xs, ys = raw[:, [0, 2]], raw[:, [1, 3]]
    assert xs.min() < 1 and xs.max() > 318 and ys.min() < 1 and ys.max() > 197
    # the clip cases: kept lines whose rounded endpoints leave the image (LineIterator clips them), and raw endpoints
    # outside the image (checkLineExtremes clamps them)
    rounded_out = clamped = 0
    for n in [c for c in _cases() if c.startswith("clip")]:
        imgs, _, raw, _, kl = M.load_case(g, n)
        H, W = imgs.shape[1:]
        r = np.rint(kl["seg"].astype(np.float64))
        rounded_out += int(((r[:, [0, 2]] >= W).any(1) | (r[:, [1, 3]] >= H).any(1)).sum())
        clamped += int(((raw[:, [0, 2]] < 0) | (raw[:, [0, 2]] >= W)).any(1).sum() + ((raw[:, [1, 3]] < 0) | (raw[:, [1, 3]] >= H)).any(1).sum())
    assert rounded_out >= 4 and clamped >= 1, (rounded_out, clamped)
    # effective blur sigmas other than 0.6 and 1.0, whose fixed-point taps need error diffusion
    assert P["other_c"]["sigma_scale"] == 0.5 and P["other_d"]["scale"] == 0.75


def test_blur_equals_cv2_over_sigmas():
    """GaussianBlur's 8-bit fixed-point taps are rounded with error diffusion (the centre takes what is left of 256): the
    restatement equals cv2 at every sigma from 0.30 to 2.99 in steps of 0.01, with LSD's kernel size for each."""
    cv2 = pytest.importorskip("cv2")
    imgs = [np.random.default_rng(3).integers(0, 256, (37, 53), dtype=np.uint8), I.make_image(64, 40, 5)]
    for k in range(30, 300):
        sigma = k / 100
        ks = 2 * int(np.ceil(sigma * np.sqrt(6 * np.log(10)))) + 1
        for img in imgs:
            np.testing.assert_array_equal(O.blur(img, sigma), cv2.GaussianBlur(img, (ks, ks), sigma), err_msg=f"sigma {sigma}")


def test_line_count_equals_cv2_line():
    """numOfPixels is cv::LineIterator's count between the rounded endpoints, clipped to the image: the pixels cv2.line
    (8-connected, which draws through LineIterator) sets, on segments pushed against and past the right and bottom edges."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    zero = clipped = 0
    for t in range(4000):
        W, H = int(rng.integers(2, 60)), int(rng.integers(2, 60))
        e = np.float32([rng.uniform(0, W), rng.uniform(0, H), rng.uniform(0, W), rng.uniform(0, H)])
        if t % 3 == 0:
            e[2 * int(rng.integers(0, 2))] = W - rng.uniform(0, 0.5)
        if t % 5 == 0:
            e[1 + 2 * int(rng.integers(0, 2))] = H - rng.uniform(0, 0.5)
        if t % 7 == 0:
            e[1] = e[3] = H - rng.uniform(0, 0.49)
        e = np.minimum(e, np.float32([W, H, W, H]) - np.float32(1e-3)).astype(np.float32)
        r = np.rint(e.astype(np.float64)).astype(int)
        canvas = np.zeros((H, W), np.uint8)
        cv2.line(canvas, (int(r[0]), int(r[1])), (int(r[2]), int(r[3])), 255, 1, cv2.LINE_8)
        want = int((canvas > 0).sum())
        assert O.line_count(W, H, e) == want, (W, H, e)
        zero += want == 0
        clipped += bool(r[0] >= W or r[2] >= W or r[1] >= H or r[3] >= H)
    assert zero > 100 and clipped > 1000


@pytest.mark.parametrize("W,H", SIZES)
def test_blur_and_resize_equal_cv2(W, H):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(W * 1000 + H)
    for img in (rng.integers(0, 256, (H, W), dtype=np.uint8), I.make_image(W, H, W + H) if W * H > 1 else np.uint8([[7]])):
        for sigma, k in ((0.6, 7), (1.0, 9)):   # the shipped blur; scale 0.8's (sigma_scale 0.8 / 0.8)
            b = O.blur(img, sigma)
            np.testing.assert_array_equal(b, cv2.GaussianBlur(img, (k, k), sigma), err_msg=f"sigma {sigma}")
            for s in (1.2, 0.8):
                np.testing.assert_array_equal(O.resize(b, s), cv2.resize(b, None, fx=s, fy=s,
                                                                         interpolation=cv2.INTER_LINEAR_EXACT))


def test_seed_order_is_raster_within_a_bin():
    """LSD grows regions from seeds in decreasing gradient bin.  Within a bin, a std::sort on the bin alone would leave
    introsort's permutation of the raster order, and that changes which regions form.  The golden's seed_order cases are
    images where the two orders give different segments: cv2 matches raster order on each, and std::sort on none."""
    g = _golden()
    names = [n for n in _cases() if n.startswith("seed_order")]
    assert len(names) >= 4
    for n in names:
        imgs, P, raw, raw_off, _ = M.load_case(g, n)
        for i, img in enumerate(imgs):
            want = raw[raw_off[i]:raw_off[i + 1]]
            np.testing.assert_array_equal(O.segments(img, *_raw_args(P), seed_order=O.STABLE), want)
            other = O.segments(img, *_raw_args(P), seed_order=O.STD_SORT)
            assert other.shape != want.shape or not np.array_equal(other, want), n


def test_restatement_equals_live_cv2():
    """240 small images under the shipped and four other parameter sets."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2024)
    for t in range(240):
        W, H = int(rng.integers(2, 48)), int(rng.integers(2, 48))
        img = rng.integers(0, 256, (H, W), dtype=np.uint8) if t % 3 == 0 else I.make_image(W, H, 1000 + t)
        P = (lsd.SHIPPED, M.OTHER_A, M.OTHER_B, M.OTHER_C, M.OTHER_D)[t % 5]
        ref = cv2.createLineSegmentDetector(0, P["scale"], P["sigma_scale"], P["quant"], P["ang_th"], 0, 0.7,
                                            P["n_bins"]).detect(img)[0]
        ref = np.zeros((0, 4), np.float32) if ref is None else ref.reshape(-1, 4)
        np.testing.assert_array_equal(O.segments(img, *_raw_args(P)), ref, err_msg=f"image {t} ({W}x{H})")


def test_npix_is_the_line_iterator_count():
    """Every golden line's numOfPixels is the number of pixels cv2.line (8-connected) draws between its rounded endpoints."""
    cv2 = pytest.importorskip("cv2")
    g = _golden()
    for name in _cases():
        imgs, _, _, _, kl = M.load_case(g, name)
        H, W = imgs.shape[1:]
        for k in range(len(kl["npix"])):
            r = [int(v) for v in np.rint(kl["seg"][k].astype(np.float64))]
            canvas = np.zeros((H, W), np.uint8)
            cv2.line(canvas, (r[0], r[1]), (r[2], r[3]), 255, 1, cv2.LINE_8)
            assert int((canvas > 0).sum()) == kl["npix"][k], (name, k)


def test_golden_tool_regenerates_the_file():
    pytest.importorskip("cv2")
    g, new = _golden(), M.golden()
    assert sorted(g.files) == sorted(new.keys())
    for k in g.files:
        if k != "cv2_version":
            np.testing.assert_array_equal(g[k], new[k], err_msg=k)
