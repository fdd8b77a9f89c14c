"""The ORB key-point selection reference (tests/ref_orb_detect.py) against the committed golden (tests/golden/orb_detect.npz,
written by tools/make_orb_detect_golden.py from cv2 4.13), and stage by stage against live cv2 when cv2 is importable."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import orb_images as I
import ref_orb_detect as R

sys.path.insert(0, os.path.join(ROOT, "tools"))

FIELDS = ("xy", "octave", "angle", "response", "desc")
CONFIGS = [(640, 480, 4, 1.2), (1241, 376, 1, 1.2), (333, 251, 4, 2.0), (301, 199, 8, 1.2), (97, 61, 2, 1.2)]


@pytest.fixture(scope="module")
def ref():
    return R.OrbDetectRef()


def _cv2():
    return pytest.importorskip("cv2")


def _bits(a):
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_same(a, b):
    for k in FIELDS:
        np.testing.assert_array_equal(_bits(np.asarray(a[k])), _bits(np.asarray(b[k])), err_msg=k)


def golden_case(z, name):
    p = z[f"{name}_params"]
    cfg = dict(n_features=int(p[0]), n_levels=int(p[1]), score_type=int(p[2]), fast_threshold=int(p[3]),
               scale=float(z[f"{name}_scale"]))
    ref = dict(off=z[f"{name}_off"], xy=z[f"{name}_xy_bits"].view(np.float32).reshape(-1, 2), octave=z[f"{name}_octave"],
               angle=z[f"{name}_angle_bits"].view(np.float32), response=z[f"{name}_response_bits"].view(np.float32),
               desc=z[f"{name}_desc"])
    return cfg, ref


# ---- against the golden (no cv2 needed) ----
def test_golden_has_ties():
    """At least one (image, level) keeps more points than its budget (FAST score ties at the cut)."""
    z = np.load(os.path.join(GOLDEN, "orb_detect.npz"))
    off, oc = z["default_fast_off"], z["default_fast_octave"]
    assert np.bincount(oc[off[0]:off[1]], minlength=4)[0] > R.level_budgets(1200, 1.2, 4)[0]


@pytest.mark.parametrize("name", ["default_fast", "default_harris", "kitti", "euroc", "th5", "th50"])
def test_reference_equals_golden(ref, name):
    import make_orb_detect_golden as G
    z = np.load(os.path.join(GOLDEN, "orb_detect.npz"))
    images, _ = G.cases()[name]
    assert [I.sha256(im) for im in images] == list(z[f"{name}_sha256"])
    cfg, want = golden_case(z, name)
    got = ref.detect_batch(images, threads=4, **cfg)
    np.testing.assert_array_equal(got["off"], want["off"])
    assert_same(got, want)


def test_level_budget_examples():
    assert R.level_budgets(1200, 1.2, 4) == [386, 322, 268, 224]
    assert R.level_budgets(2000, 1.2, 1) == [2000]
    assert R.level_budgets(0, 1.2, 4) == [0, 0, 0, 0]
    for n in (0, 1, 3, 800, 1200, 2000, 5000):
        for s in (1.2, 1.5, 2.0):
            for nl in range(1, 9):
                b = R.level_budgets(n, s, nl)
                assert len(b) == nl and min(b) >= 0 and sum(b) >= n


def test_retain_best_is_a_set_with_ties():
    r = np.float32([5, 3, 3, 3, 1, 7])
    assert R.retain_best(r, 0).sum() == 0
    assert R.retain_best(r, 6).all() and R.retain_best(r, 10).all()
    np.testing.assert_array_equal(R.retain_best(r, 2), [True, False, False, False, False, True])
    np.testing.assert_array_equal(R.retain_best(r, 3), [True, True, True, True, False, True])


# ---- against live cv2 ----
def _fast_images():
    rng = np.random.default_rng(4)
    yy, xx = np.mgrid[0:120, 0:160]
    return {"seeded": I.make_image(160, 120, 5), "flat": np.full((120, 160), 77, np.uint8),
            "saturated": np.where(rng.random((120, 160)) < 0.5, 0, 255).astype(np.uint8),
            "checker": (((yy // 4 + xx // 4) % 2) * 255).astype(np.uint8),
            "noise": rng.integers(0, 256, (120, 160), dtype=np.uint8), "tiny6": I.make_image(6, 6, 1),
            "tiny7": I.make_image(7, 9, 2), "tiny9": I.make_image(9, 8, 3)}


@pytest.mark.parametrize("th", [0, 1, 5, 20, 50, 254, 255])
def test_fast_nms_equals_cv2(th):
    cv2 = _cv2()
    for name, img in _fast_images().items():
        ys, xs, sc = R.fast_nms(img, th)
        kps = cv2.FastFeatureDetector_create(th, True).detect(img)
        want = sorted((int(k.pt[1]), int(k.pt[0]), int(k.response)) for k in kps)
        assert list(zip(ys.tolist(), xs.tolist(), sc.tolist())) == want, name


def test_level_budgets_equal_cv2(ref):
    """Per-octave counts of cv2's detectAndCompute equal the reference's selection on an image with many corners (so
    every level's budget binds), over the n_features / scale / level grid."""
    cv2 = _cv2()
    img = I.make_image(320, 240, 8)
    for n in (0, 1, 3, 800, 1200, 2000, 5000):
        for s in (1.2, 1.5, 2.0):
            for nl in range(1, 9):
                lvl, _, _, _ = ref.select(img, n_features=n, n_levels=nl, scale=s, fast_threshold=5)
                o = cv2.ORB_create(n, s, nl, 19, 0, 2, cv2.ORB_FAST_SCORE, 31, 5)
                got = np.bincount([k.octave for k in o.detect(img, None)], minlength=nl)
                np.testing.assert_array_equal(np.bincount(lvl, minlength=nl), got, err_msg=str((n, s, nl)))


def test_harris_responses_equal_cv2(ref):
    cv2 = _cv2()
    for seed, (W, H) in enumerate([(640, 480), (333, 251)]):
        img = I.make_image(W, H, 60 + seed)
        got = ref.detect(img, score_type=R.HARRIS_SCORE, describe=False)
        want = R.cv2_detect(cv2, img, score_type=R.HARRIS_SCORE)
        np.testing.assert_array_equal(got["xy"], want["xy"])
        np.testing.assert_array_equal(got["response"].view(np.uint32), want["response"].view(np.uint32))


@pytest.mark.parametrize("score_type", [R.FAST_SCORE, R.HARRIS_SCORE])
@pytest.mark.parametrize("W,H,nl,s", CONFIGS)
def test_detect_and_compute_equals_cv2(ref, W, H, nl, s, score_type):
    cv2 = _cv2()
    for seed in (1, 2):
        img = I.make_image(W, H, seed + W)
        for th in (20, 7):
            p = dict(n_levels=nl, scale=s, score_type=score_type, fast_threshold=th)
            assert_same(ref.detect(img, **p), R.cv2_detect(cv2, img, **p))


def test_golden_regenerates():
    """Running the golden tool again gives the committed arrays (the npz carries zip timestamps: compare arrays)."""
    _cv2()
    import make_orb_detect_golden as G
    z = np.load(os.path.join(GOLDEN, "orb_detect.npz"))
    rec = G.golden()
    assert sorted(rec) == sorted(z.files)
    for k, v in rec.items():
        np.testing.assert_array_equal(np.asarray(v), z[k], err_msg=k)
