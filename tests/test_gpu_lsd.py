"""plstvo_lsd_detect_batch on the GPU: bit-identical to cv2 4.13's LineSegmentDetector and the reference's KeyLine step
(tests/golden/lsd.npz) and to the restatement (oracle/lsd.py) on ragged batches, with the capacity and error conventions of
the other batched detectors, and end to end: key lines it detects feed LBD and the tracker exactly as the golden's do."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import orb_images as I
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_lsd_golden as M  # noqa: E402

from oracle import lsd  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(GOLDEN, "lsd.npz"))
FIELDS = ("seg", "angle", "npix", "response", "length")


def _cfg(P):
    return T.default_lsd_config(**P)


def _equal(got, want, msg):
    for f in FIELDS:
        np.testing.assert_array_equal(got[f], want[f], err_msg=f"{msg}.{f}")


@pytest.mark.parametrize("name", [str(c) for c in G["cases"]])
def test_gpu_equals_golden(engine, name):
    imgs, P, _, _, kl = M.load_case(G, name)
    total, out = engine.lsd_detect_batch(_cfg(P), imgs)
    assert total == kl["off"][-1]
    np.testing.assert_array_equal(out["off"], kl["off"])
    _equal(out, kl, name)


def _oracle_batch(imgs, P):
    o = lsd.LsdOracle()
    per = [o.detect(im, P["scale"], P["sigma_scale"], P["quant"], P["ang_th"], P["n_bins"], P["min_line_length"],
                    P["n_features"]) for im in imgs]
    off = np.concatenate([[0], np.cumsum([len(d["angle"]) for d in per])]).astype(np.int32)
    return off, {f: np.concatenate([d[f] for d in per]) for f in FIELDS}


def test_ragged_batch_equals_single_calls_and_restatement(engine):
    """Flat, black, noise, textured and stereo-view images of one size in one batch (line counts 0 to hundreds), then a
    batch of 1x1 images and one of more images than the GPU has SMs."""
    W, H = 1241, 376
    imgs = np.stack([np.full((H, W), 128, np.uint8), I.make_image(W, H, 21), np.zeros((H, W), np.uint8),
                     np.random.default_rng(5).integers(0, 256, (H, W), dtype=np.uint8), I.make_image(W, H, 22),
                     M.images(W, H, "kitti_view", [1])[0]])
    for P in (lsd.SHIPPED, M.OTHER_A):
        total, out = engine.lsd_detect_batch(_cfg(P), imgs)
        off, want = _oracle_batch(imgs, P)
        np.testing.assert_array_equal(out["off"], off)
        _equal(out, want, "batch")
        assert np.diff(off)[0] == 0 and np.diff(off).max() > 0
        for i in range(len(imgs)):
            _, one = engine.lsd_detect_batch(_cfg(P), imgs[i:i + 1])
            _equal(one, {f: out[f][off[i]:off[i + 1]] for f in FIELDS}, f"image {i}")
    tiny = np.random.default_rng(7).integers(0, 256, (5, 1, 1), dtype=np.uint8)
    total, out = engine.lsd_detect_batch(_cfg(lsd.SHIPPED), tiny)
    assert total == 0 and list(out["off"]) == [0] * 6
    many = np.stack([I.make_image(96, 64, 300 + k) for k in range(141)])   # an H100 SXM has 132 SMs
    total, out = engine.lsd_detect_batch(_cfg(lsd.SHIPPED), many)
    off, want = _oracle_batch(many, lsd.SHIPPED)
    np.testing.assert_array_equal(out["off"], off)
    _equal(out, want, "many")


def test_capacity_overflow_writes_offsets(engine):
    imgs, P, _, _, kl = M.load_case(G, "kitti_300")
    cfg = _cfg(P)
    off = np.zeros(len(imgs) + 1, np.int32)
    seg = np.zeros((10, 4), np.float32)
    f = lambda a, t: a.ctypes.data_as(t)  # noqa: E731
    rc = engine.lib.plstvo_lsd_detect_batch(engine.ctx, C.byref(cfg), len(imgs), imgs.shape[2], imgs.shape[1],
                                            f(imgs, T.c_uint8_p), 10, f(off, T.c_int32_p), f(seg, T.c_float_p), None, None,
                                            None, None)
    assert rc == -2
    np.testing.assert_array_equal(off, kl["off"])
    assert not seg.any()
    total, out = engine.lsd_detect_batch(cfg, imgs, capacity=int(kl["off"][-1]))
    assert total == kl["off"][-1]
    _equal(out, kl, "exact capacity")


def test_errors_leave_the_context_usable(engine):
    imgs, P, _, _, kl = M.load_case(G, "odd_63x17")
    bad = [dict(refine=1), dict(refine=2), dict(scale=0.0), dict(scale=-1.0), dict(sigma_scale=0.0), dict(quant=-1.0),
           dict(ang_th=0.0), dict(ang_th=180.0), dict(n_bins=0), dict(n_bins=4097), dict(min_line_length=-0.1),
           dict(n_features=-1), dict(scale=0.01), dict(scale=1e6), dict(scale=0.5)]
    for kw in bad:
        with pytest.raises(PlstvoError) as e:
            engine.lsd_detect_batch(_cfg(dict(P, **kw)), imgs)
        assert e.value.code == -1, kw
    cfg = _cfg(P)
    off = np.zeros(2, np.int32)
    u8, i32 = T.c_uint8_p, T.c_int32_p
    assert engine.lib.plstvo_lsd_detect_batch(engine.ctx, C.byref(cfg), 1, 0, 17, imgs.ctypes.data_as(u8), 100,
                                              off.ctypes.data_as(i32), None, None, None, None, None) == -1
    assert engine.lib.plstvo_lsd_detect_batch(engine.ctx, C.byref(cfg), 1, 63, 17, imgs.ctypes.data_as(u8), 100, None,
                                              None, None, None, None, None) == -1
    assert engine.lib.plstvo_lsd_detect_batch(engine.ctx, C.byref(cfg), 1, 63, 17, None, 100, off.ctypes.data_as(i32),
                                              None, None, None, None, None) == -1
    assert engine.lib.plstvo_lsd_detect_batch(engine.ctx, None, 1, 63, 17, imgs.ctypes.data_as(u8), 100,
                                              off.ctypes.data_as(i32), None, None, None, None, None) == -1
    many = np.zeros((65536, 1, 1), np.uint8)   # more images than one launch's gridDim.z holds
    off_many = np.zeros(65537, np.int32)
    assert engine.lib.plstvo_lsd_detect_batch(engine.ctx, C.byref(cfg), 65536, 1, 1, many.ctypes.data_as(u8), 0,
                                              off_many.ctypes.data_as(i32), None, None, None, None, None) == -1
    total, out = engine.lsd_detect_batch(cfg, imgs)
    np.testing.assert_array_equal(out["off"], kl["off"])
    _equal(out, kl, "after errors")


def test_kernel_times(engine):
    imgs, P, _, _, _ = M.load_case(G, "kitti_300")
    engine.lsd_detect_batch(_cfg(P), imgs)
    ms = engine.lsd_kernel_times()
    assert ms.shape == (5,) and (ms >= 0).all() and ms[2] > 0


def test_fresh_context_times_before_any_call():
    e = Engine(0)
    try:
        with pytest.raises(PlstvoError):
            e.lsd_kernel_times()
    finally:
        e.close()


def test_detect_describe_track_equals_golden_lines(engine):
    """plstvo_lsd_detect_batch -> plstvo_lbd_compute_batch -> plstvo_track_stereo_batch on the KITTI stereo frames gives the
    same bytes as the same chain fed the golden (cv2) key lines."""
    imgs, P, _, _, kl = M.load_case(G, "kitti_stereo")
    total, det = engine.lsd_detect_batch(_cfg(P), imgs)

    def run(lines):
        off = lines["off"]
        desc = engine.lbd_compute_batch(imgs, off, lines["seg"], lines["angle"], lines["npix"])
        fr = []
        for f in range(2):
            l, r = 2 * f, 2 * f + 1
            z2, z32 = np.zeros((0, 2), np.float32), np.zeros((0, 32), np.uint8)
            fr.append(dict(pl_off=[0, 0], pr_off=[0, 0], kp_l=z2, kp_r=z2, poct_l=np.zeros(0, np.int32), pdesc_l=z32,
                           pdesc_r=z32, ll_off=[0, off[l + 1] - off[l]], lr_off=[0, off[r + 1] - off[r]],
                           seg_l=lines["seg"][off[l]:off[l + 1]], seg_r=lines["seg"][off[r]:off[r + 1]],
                           angle_l=lines["angle"][off[l]:off[l + 1]], loct_l=np.zeros(off[l + 1] - off[l], np.int32),
                           ldesc_l=desc[off[l]:off[l + 1]], ldesc_r=desc[off[r]:off[r + 1]]))
        mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
        tc.has_points = 0
        return desc, engine.track_stereo_batch(T.kitti_camera(), tc, mc, sc, *fr)

    da, (ra, na) = run(det)
    db, (rb, nb) = run(kl)
    assert na[0, 1] > 20 and na[0, 3] > 20, na
    np.testing.assert_array_equal(da, db)
    np.testing.assert_array_equal(na, nb)
    assert ra.tobytes() == rb.tobytes()
