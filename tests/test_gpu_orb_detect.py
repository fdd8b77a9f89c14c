"""plstvo_orb_detect_and_compute_batch on the GPU: bit-identical to cv2 (through tests/golden/orb_detect.npz) and to the
reference (tests/ref_orb_detect.py) in canonical order; edge cases, capacity and config errors; descriptors equal to
plstvo_orb_compute_batch on the detected points; and end to end, tracking fed with GPU-detected features equals tracking fed
with cv2's."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import orb_images as I
import ref_orb_detect as R
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import PlstvoError

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_orb_detect_golden as G  # noqa: E402
import make_orb_golden as M  # noqa: E402
from test_ref_orb_detect import CONFIGS, assert_same, golden_case  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    return R.OrbDetectRef()


def _cfg(n_features=1200, n_levels=4, scale=1.2, score_type=R.FAST_SCORE, fast_threshold=20):
    return T.default_orb_detect_config(n_features, n_levels, scale, score_type, fast_threshold)


def _check(engine, ref, images, fast_th=None, **p):
    n, got = engine.orb_detect_and_compute_batch(_cfg(**p), images, fast_th)
    th = p.pop("fast_threshold", 20)
    want = ref.detect_batch(images, fast_th=fast_th if fast_th is not None else [th] * len(images), threads=8, **p)
    np.testing.assert_array_equal(got["off"], want["off"])
    assert n == want["off"][-1]
    assert_same(got, want)
    return got


@pytest.mark.parametrize("name", ["default_fast", "default_harris", "kitti", "euroc", "th5", "th50"])
def test_gpu_equals_golden(engine, name):
    z = np.load(os.path.join(GOLDEN, "orb_detect.npz"))
    images, _ = G.cases()[name]
    cfg, want = golden_case(z, name)
    n, got = engine.orb_detect_and_compute_batch(_cfg(**cfg), images)
    np.testing.assert_array_equal(got["off"], want["off"])
    assert_same(got, want)


@pytest.mark.parametrize("score_type", [R.FAST_SCORE, R.HARRIS_SCORE])
@pytest.mark.parametrize("W,H,nl,s", CONFIGS)
def test_gpu_equals_reference(engine, ref, W, H, nl, s, score_type):
    imgs = np.stack([I.make_image(W, H, 300 + k) for k in range(3)])
    for th in (20, 0, 9):
        _check(engine, ref, imgs, n_levels=nl, scale=s, score_type=score_type, fast_threshold=th)
    _check(engine, ref, imgs, fast_th=[5, 40, 255], n_levels=nl, scale=s, score_type=score_type)   # per-image thresholds


@pytest.mark.parametrize("score_type", [R.FAST_SCORE, R.HARRIS_SCORE])
def test_gpu_64_images(engine, ref, score_type):
    imgs = np.stack([I.make_image(320, 240, 700 + k) for k in range(64)])
    th = [(7 * k) % 60 for k in range(64)]
    _check(engine, ref, imgs, fast_th=th, n_features=500, score_type=score_type)


def test_gpu_edge_cases(engine, ref):
    flat = np.full((2, 240, 320), 90, np.uint8)
    n, got = engine.orb_detect_and_compute_batch(_cfg(), flat)
    assert n == 0 and list(got["off"]) == [0, 0, 0]
    img = I.make_image(320, 240, 5)[None]
    for st in (R.FAST_SCORE, R.HARRIS_SCORE):
        n, got = engine.orb_detect_and_compute_batch(_cfg(n_features=0, score_type=st), img)
        assert n == 0
        _check(engine, ref, img, n_features=3, n_levels=8, score_type=st)     # budgets that round to 0 on some levels
        assert 0 in R.level_budgets(3, 1.2, 8)
    small = I.make_image(40, 36, 6)[None]                                   # every level under 2 * edge
    n, got = engine.orb_detect_and_compute_batch(_cfg(), small)
    assert n == 0
    _check(engine, ref, I.make_image(60, 50, 7)[None], n_levels=8)          # levels smaller than 7 px


def test_gpu_capacity_and_invalid(engine):
    imgs = np.stack([I.make_image(640, 480, 1), I.make_image(640, 480, 2)])
    n, full = engine.orb_detect_and_compute_batch(_cfg(), imgs)
    for st in (R.FAST_SCORE, R.HARRIS_SCORE):
        n, full = engine.orb_detect_and_compute_batch(_cfg(score_type=st), imgs)
        with pytest.raises(PlstvoError, match="TOO_LARGE"):
            engine.orb_detect_and_compute_batch(_cfg(score_type=st), imgs, capacity=n - 1)
        import ctypes as C
        off = np.zeros(3, np.int32)
        rc = engine.lib.plstvo_orb_detect_and_compute_batch(engine.ctx, C.byref(_cfg(score_type=st)), 2, 640, 480,
                                                            imgs.ctypes.data_as(T.c_uint8_p), None, n - 1,
                                                            off.ctypes.data_as(T.c_int32_p), None, None, None, None, None)
        assert rc == -2
        np.testing.assert_array_equal(off, full["off"])
        n2, again = engine.orb_detect_and_compute_batch(_cfg(score_type=st), imgs, capacity=n)
        assert n2 == n
    big = I.make_image(1500, 1200, 3)[None]                                 # more than 65535 points in one image
    with pytest.raises(PlstvoError, match="TOO_LARGE"):
        engine.orb_detect_and_compute_batch(_cfg(n_features=200000, n_levels=1, fast_threshold=0), big)
    for field, v in (("n_features", -1), ("score_type", 2)):
        cfg = _cfg()
        setattr(cfg, field, v)
        with pytest.raises(PlstvoError, match="INVALID"):
            engine.orb_detect_and_compute_batch(cfg, imgs)
    for field, v in (("patch_size", 15), ("wta_k", 3), ("n_levels", 0), ("edge_threshold", -1)):
        cfg = _cfg()
        setattr(cfg.orb, field, v)
        with pytest.raises(PlstvoError, match="INVALID"):
            engine.orb_detect_and_compute_batch(cfg, imgs)


def test_gpu_descriptors_equal_compute_batch(engine):
    imgs = np.stack([I.make_image(640, 480, 11), I.make_image(640, 480, 12)])
    for st in (R.FAST_SCORE, R.HARRIS_SCORE):
        n, got = engine.orb_detect_and_compute_batch(_cfg(score_type=st), imgs)
        ocfg = T.default_orb_config(4, float(np.float32(1.2)))
        m, out = engine.orb_compute_batch(ocfg, imgs, got["off"], got["xy"], got["octave"], None)
        assert m == n
        np.testing.assert_array_equal(out["desc"], got["desc"])
        np.testing.assert_array_equal(out["angle"].view(np.uint32), got["angle"].view(np.uint32))
    t = engine.orb_detect_kernel_times()
    assert t.shape == (4,) and (t >= 0).all() and t[0] > 0 and t[1] > 0


def test_track_stereo_with_gpu_detected_features(engine):
    """plstvo_track_stereo_batch on the KITTI-size golden frames gives identical results with GPU-detected features and with
    cv2's (golden) ones."""
    z = np.load(os.path.join(GOLDEN, "orb_detect.npz"))
    imgs = M.kitti_views()
    _, want = golden_case(z, "kitti")
    n, got = engine.orb_detect_and_compute_batch(_cfg(n_features=2000, n_levels=1), imgs)

    def frames(d):
        off, fr = d["off"], []
        for f in range(2):
            l, r = 2 * f, 2 * f + 1
            z32, zf = np.zeros((0, 32), np.uint8), np.zeros((0, 4), np.float32)
            fr.append(dict(pl_off=[0, off[l + 1] - off[l]], pr_off=[0, off[r + 1] - off[r]], kp_l=d["xy"][off[l]:off[l + 1]],
                           kp_r=d["xy"][off[r]:off[r + 1]], poct_l=d["octave"][off[l]:off[l + 1]],
                           pdesc_l=d["desc"][off[l]:off[l + 1]], pdesc_r=d["desc"][off[r]:off[r + 1]], ll_off=[0, 0],
                           lr_off=[0, 0], seg_l=zf, seg_r=zf, angle_l=np.zeros(0, np.float32), loct_l=np.zeros(0, np.int32),
                           ldesc_l=z32, ldesc_r=z32))
        return fr

    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    tc.has_lines = 0
    cam = T.kitti_camera()
    ra, na = engine.track_stereo_batch(cam, tc, mc, sc, *frames(got))
    rb, nb = engine.track_stereo_batch(cam, tc, mc, sc, *frames(want))
    assert na[0, 0] > 100 and na[0, 2] > 100, na
    np.testing.assert_array_equal(na, nb)
    assert ra.tobytes() == rb.tobytes()
