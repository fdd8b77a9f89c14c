"""plstvo_track_stereo_images_lsd_batch / _sequence on the GPU: stereo images alone in, pose out.  Byte-identical to the
two-call chain they compose (plstvo_lsd_detect_batch, then plstvo_track_stereo_images_batch / _sequence fed its key lines),
and through the golden files to cv2's key points and lines; ragged batches, the config switches, context reuse, errors and
examples/images_lsd_cpp.cpp (plstvo::StereoImageHandler) against a Python loop.  Needs neither cv2 nor the reference sources."""
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from test_gpu_track_images import CAM_SMALL, assert_same, configs, frames_slice, moving_views, ragged_sets, sm_count
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError
from stvo_pl_b200.handler import HandlerConfig, update_fast_threshold

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_lbd_golden as LG  # noqa: E402
import make_lsd_golden as M  # noqa: E402
import make_orb_golden as OG  # noqa: E402

pytestmark = pytest.mark.gpu


def images_only(d):
    return dict(img_l=d["img_l"], img_r=d["img_r"], fast_th=d.get("fast_th"))


def chain(eng, cam, cfg, mc, sc, oc, lc, sets, sequence, priors=None):
    """The two-call chain: lsd_detect_batch(lc) on every image in the images call's block order ([left][right] per frame
    set), then track_stereo_images_batch / _sequence fed those key lines."""
    NF = len(sets[0]["img_l"])
    fed = [images_only(s) for s in sets]
    if cfg.has_lines:
        _, kl = eng.lsd_detect_batch(lc, np.concatenate([im for s in sets for im in (s["img_l"], s["img_r"])]))
        for j, d in enumerate(fed):
            for side, b in (("l", 2 * j), ("r", 2 * j + 1)):
                off = kl["off"][b * NF:(b + 1) * NF + 1]
                d[f"l{side}_off"] = off - off[0]
                for k in ("seg", "angle", "npix"):
                    d[f"{k}_{side}"] = kl[k][off[0]:off[-1]]
    if sequence:
        return eng.track_stereo_images_sequence(cam, cfg, mc, sc, oc, fed[0], priors)
    return eng.track_stereo_images_batch(cam, cfg, mc, sc, oc, fed[0], fed[1], priors)


def same(a, b):
    """Byte equality of two call results: (structured results, n_stereo) or (total, dict of arrays)."""
    if isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            same(a[k], b[k])
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            same(x, y)
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    else:
        assert a == b


# ---- 1. KITTI golden frames, independent of GPU LSD ----
G_LSD = np.load(os.path.join(GOLDEN, "lsd.npz"))
G_LBD = np.load(os.path.join(GOLDEN, "lbd.npz"))


def golden_line_descriptors(eng, imgs, kl):
    """LBD descriptors of lsd.npz's KITTI lines, taken from lbd.npz by matching each line (segment, angle and numOfPixels
    bits): an LBD descriptor depends only on its line and the image, and lbd.npz holds the same 300 lines per image in
    another order.  lbd.npz took the angle from a double atan2 rounded to float and numOfPixels without LineIterator's
    clipping, so some lines (a last-bit angle, a segment ending in the last half pixel) have no exact twin there; those take
    plstvo_lbd_compute_batch's descriptor, which tests/test_gpu_lbd.py holds to the reference.  Returns (desc, twins)."""
    images, off, seg, ang, npix, desc = LG.load_case(G_LBD, "kitti_stereo")
    np.testing.assert_array_equal(images, imgs)
    key = lambda s, a, n: s.tobytes() + np.float32(a).tobytes() + np.int32(n).tobytes()   # noqa: E731
    gpu = eng.lbd_compute_batch(imgs, kl["off"], kl["seg"], kl["angle"], kl["npix"])
    out, twins, moved = gpu.copy(), 0, 0
    for i in range(len(imgs)):
        table = {key(seg[k], ang[k], npix[k]): k for k in range(off[i], off[i + 1])}
        assert len(table) == off[i + 1] - off[i]
        for k in range(kl["off"][i], kl["off"][i + 1]):
            t = table.get(key(kl["seg"][k], kl["angle"][k], kl["npix"][k]))
            if t is not None:
                out[k] = desc[t]
                twins += 1
                moved += t - off[i] != k - kl["off"][i]
    assert moved > 0, "lbd.npz no longer permutes the lines: feed it directly"
    for i in range(len(imgs)):   # a line without a twin is still in lbd.npz, by its segment
        segs = {seg[k].tobytes() for k in range(off[i], off[i + 1])}
        assert all(kl["seg"][k].tobytes() in segs for k in range(kl["off"][i], kl["off"][i + 1])), i
    return out, twins


def test_kitti_golden_end_to_end(engine):
    imgs, P, _, _, kl = M.load_case(G_LSD, "kitti_stereo")
    np.testing.assert_array_equal(imgs, OG.kitti_views())
    lc = T.default_lsd_config(**P)
    mc, sc, tc, oc = configs()
    cam = T.kitti_camera()
    prev, curr = (dict(img_l=imgs[2 * f:2 * f + 1], img_r=imgs[2 * f + 1:2 * f + 2], fast_th=None) for f in range(2))
    got = engine.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, prev, curr)
    assert_same(got, chain(engine, cam, tc, mc, sc, oc, lc, [prev, curr], False))
    # cv2's key points (orb_detect.npz), cv2's lines in the reference's order (lsd.npz), the reference's descriptors
    ldesc, twins = golden_line_descriptors(engine, imgs, kl)
    assert twins >= 0.8 * len(ldesc), twins   # 251 to 266 of 300 per image
    z = np.load(os.path.join(GOLDEN, "orb_detect.npz"))
    koff, kxy, koct, kdesc = z["kitti_off"], z["kitti_xy_bits"].view(np.float32).reshape(-1, 2), z["kitti_octave"], z["kitti_desc"]
    off, seg, ang = kl["off"], kl["seg"], kl["angle"]
    feats = []
    for f in range(2):
        l, r = 2 * f, 2 * f + 1
        feats.append(dict(pl_off=[0, koff[l + 1] - koff[l]], pr_off=[0, koff[r + 1] - koff[r]], kp_l=kxy[koff[l]:koff[l + 1]],
                          kp_r=kxy[koff[r]:koff[r + 1]], poct_l=koct[koff[l]:koff[l + 1]], pdesc_l=kdesc[koff[l]:koff[l + 1]],
                          pdesc_r=kdesc[koff[r]:koff[r + 1]], ll_off=[0, off[l + 1] - off[l]], lr_off=[0, off[r + 1] - off[r]],
                          seg_l=seg[off[l]:off[l + 1]], seg_r=seg[off[r]:off[r + 1]], angle_l=ang[off[l]:off[l + 1]],
                          loct_l=np.zeros(off[l + 1] - off[l], np.int32), ldesc_l=ldesc[off[l]:off[l + 1]],
                          ldesc_r=ldesc[off[r]:off[r + 1]]))
    assert_same(got, engine.track_stereo_batch(cam, tc, mc, sc, *feats))
    n = got[1]
    assert n[0, 0] > 100 and n[0, 2] > 100 and n[0, 1] > 20 and n[0, 3] > 20, n
    ms, lsd_ms = engine.track_stereo_images_stage_times(), engine.lsd_kernel_times()
    assert (ms >= 0).all() and ms[1] > 0 and ms[2] > 0 and ms[3] > 0 and ms[4] > 0, ms
    assert lsd_ms[2] > 0, lsd_ms


# ---- 2. sequence ----
def test_sequence_equals_chain_and_batch(engine):
    fr = images_only(moving_views(9, 1241, 376, 501, 300, fast_th=[20, 0, 12, 35, 20, 5, 0, 50, 20]))
    mc, sc, tc, oc = configs(1200, 4)
    lc = T.default_lsd_config()
    cam = T.kitti_camera()
    seq = engine.track_stereo_images_lsd_sequence(cam, tc, mc, sc, oc, lc, fr)
    assert_same(seq, chain(engine, cam, tc, mc, sc, oc, lc, [fr], True))
    bat = engine.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, frames_slice(fr, 0, 8), frames_slice(fr, 1, 9))
    assert seq[0].tobytes() == bat[0].tobytes()
    np.testing.assert_array_equal(bat[1][:, :2], seq[1][:-1])
    np.testing.assert_array_equal(bat[1][:, 2:], seq[1][1:])
    assert (seq[1][:, 1] > 20).all() and (seq[1][:, 0] > 100).all(), seq[1]
    # a sequence of one frame and an empty batch run nothing
    one = engine.track_stereo_images_lsd_sequence(cam, tc, mc, sc, oc, lc, frames_slice(fr, 0, 1))
    assert one[0].size == 0 and (one[1] == 0).all()
    empty = frames_slice(fr, 0, 0)
    assert engine.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, empty, empty)[0].size == 0


# ---- 3. ragged batches ----
MODES = ["fast", "harris", "lines_only", "points_only", "lsd_scale_1", "lsd_all_lines", "lsd_100"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("size", ["9", "37", "sms+5"])
def test_ragged_batch_equals_chain(mode, size):
    """ragged_sets: flat images (no lines), lines on one side only, thresholds 0 and 255.  9 pairs (36 images, fewer than
    SMs) take the path where LSD runs before ORB; 37 and SMs + 5 pairs the one where they overlap."""
    B = {"9": 9, "37": 37}.get(size, sm_count() + 5)
    prev, curr = (images_only(d) for d in ragged_sets(B, 8100 + B))
    mc, sc, tc, oc = configs(500, 4, T.ORB_HARRIS_SCORE if mode == "harris" else T.ORB_FAST_SCORE)
    lc = T.default_lsd_config(**{"lsd_scale_1": dict(scale=1.0), "lsd_all_lines": dict(n_features=0),
                                 "lsd_100": dict(n_features=100)}.get(mode, {}))
    if mode == "lines_only":
        tc.has_points = 0
    if mode == "points_only":
        tc.has_lines = 0
        lc = None
    priors = np.zeros(B, T.PRIOR_DTYPE)
    priors["Tfw"] = priors["DT"] = np.eye(4)
    e = Engine()
    l0 = e.launches
    got = e.track_stereo_images_lsd_batch(CAM_SMALL, tc, mc, sc, oc, lc, prev, curr, priors)
    l1 = e.launches
    ms = e.track_stereo_images_stage_times()
    want = chain(e, CAM_SMALL, tc, mc, sc, oc, lc, [prev, curr], False, priors)
    l2 = e.launches
    assert_same(got, want)
    assert l1 - l0 == l2 - l1, (l1 - l0, l2 - l1)     # the same kernels, once each
    if mode != "points_only":
        assert ms[2] > 0, ms
    if mode == "lines_only":
        assert ms[1] == 0 and ms[2] > 0 and (got[1][:, 0::2] == 0).all(), ms
    if mode == "points_only":
        assert ms[2] == 0 and ms[1] > 0, ms
    e.close()


# ---- 4. context reuse ----
def test_context_reuse():
    kv = OG.kitti_views()
    kp, kc = (dict(img_l=kv[2 * f:2 * f + 1], img_r=kv[2 * f + 1:2 * f + 2], fast_th=None) for f in range(2))
    sp, scu = ragged_sets(9, 9300)
    mc, sc, tc, oc = configs()
    mc2, sc2, tc2, oc2 = configs(500, 4)
    lc, lc2 = T.default_lsd_config(), T.default_lsd_config(100, scale=1.0)
    cam = T.kitti_camera()
    imgs = np.stack([M.images(640, 480, "make", [s])[0] for s in (1, 2)])
    calls = {
        "lsd_big": lambda e: e.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, kp, kc),
        "lsd_small": lambda e: e.track_stereo_images_lsd_batch(CAM_SMALL, tc2, mc2, sc2, oc2, lc2, images_only(sp),
                                                               images_only(scu)),
        "lsd_detect": lambda e: e.lsd_detect_batch(lc, imgs),
        "images": lambda e: e.track_stereo_images_batch(CAM_SMALL, tc2, mc2, sc2, oc2, sp, scu),
        "orb": lambda e: e.orb_detect_and_compute_batch(T.default_orb_detect_config(), imgs),
    }
    fresh = {}
    for k, f in calls.items():
        e = Engine()
        fresh[k] = f(e)
        e.close()
    e = Engine()
    for k in ("lsd_big", "lsd_detect", "lsd_small", "images", "orb", "lsd_big", "images", "lsd_small", "lsd_detect", "orb",
              "lsd_small"):
        same(calls[k](e), fresh[k])
    e.close()


# ---- 5. errors ----
CAM_TINY = T.PlCamera(fx=10.0, fy=10.0, cx=4.0, cy=4.0, b=0.2, width=8, height=8)


def _call(e, cam, tc, mc, sc, oc, lc, prev, curr, sequence=False, msg=None):
    """The raw C call; with msg, the return code and plstvo_last_error's text (that names the check that failed)."""
    ps, kp = T.stereo_images_as_c(prev)
    res = np.zeros(max(ps.B, 1), T.POSE_RESULT_DTYPE)
    lcp = None if lc is None else C.byref(lc)
    if sequence:
        rc = e.lib.plstvo_track_stereo_images_lsd_sequence(e.ctx, C.byref(cam), C.byref(tc), C.byref(mc), C.byref(sc),
                                                           C.byref(oc), lcp, C.byref(ps), None, res.ctypes.data, None)
    else:
        cs, kc = T.stereo_images_as_c(curr)
        rc = e.lib.plstvo_track_stereo_images_lsd_batch(e.ctx, C.byref(cam), C.byref(tc), C.byref(mc), C.byref(sc), C.byref(oc),
                                                        lcp, C.byref(ps), C.byref(cs), None, res.ctypes.data, None)
    return rc, (e.lib.plstvo_last_error(e.ctx) or b"").decode()


def test_errors_leave_the_context_usable():
    with_lines = ragged_sets(6, 9500)
    prev, curr = (images_only(d) for d in with_lines)
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e = Engine()
    want = e.track_stereo_images_lsd_batch(CAM_SMALL, tc, mc, sc, oc, lc, prev, curr)
    e.close()
    e = Engine()

    def check(got, rc, text):
        assert got[0] == rc and text in got[1], (got, rc, text)
        assert_same(e.track_stereo_images_lsd_batch(CAM_SMALL, tc, mc, sc, oc, lc, prev, curr), want)

    lines_given = "key-line fields must be null"
    check(_call(e, CAM_SMALL, tc, mc, sc, oc, lc, with_lines[0], curr), -1, lines_given)
    for k in ("ll_off", "npix_r"):
        bad = dict(curr)
        bad[k] = with_lines[1][k]
        check(_call(e, CAM_SMALL, tc, mc, sc, oc, lc, prev, bad), -1, lines_given)
    check(_call(e, CAM_SMALL, tc, mc, sc, oc, None, prev, curr), -1, "null lsd config")
    for kw, text in ((dict(refine=1), "lsd refine"), (dict(scale=0.5), "lsd scale 0.5"), (dict(n_bins=0), "lsd parameter out of range"),
                     (dict(ang_th=180.0), "lsd parameter out of range")):
        check(_call(e, CAM_SMALL, tc, mc, sc, oc, T.default_lsd_config(**kw), prev, curr), -1, text)
    big_cam = T.PlCamera(fx=300.0, fy=300.0, cx=160.0, cy=120.0, b=0.2, width=640, height=240)
    check(_call(e, big_cam, tc, mc, sc, oc, lc, prev, curr), -5, "image size differs from the camera's")
    check(_call(e, CAM_SMALL, tc, mc, sc, oc, lc, prev, frames_slice(curr, 0, 5)), -5, "different numbers of frames")
    # more than 65535 images in one call: 4 B for a batch, 2 B for a sequence
    tiny = lambda n: dict(img_l=np.zeros((n, 8, 8), np.uint8), img_r=np.zeros((n, 8, 8), np.uint8))   # noqa: E731
    too_many = "more than 65535 images in one call"
    check(_call(e, CAM_TINY, tc, mc, sc, oc, lc, tiny(16384), tiny(16384)), -1, too_many)
    check(_call(e, CAM_TINY, tc, mc, sc, oc, lc, tiny(32768), None, sequence=True), -1, too_many)
    with pytest.raises(PlstvoError, match="lsd refine"):
        e.track_stereo_images_lsd_batch(CAM_SMALL, tc, mc, sc, oc, T.default_lsd_config(refine=1), prev, curr)
    e.close()


# ---- 6. StereoImageHandler (examples/images_lsd_cpp.cpp) against a Python loop ----
def test_handler_example_equals_python_loop(engine, tmp_path):
    NF, W, H = 9, 1241, 376
    fr = moving_views(NF, W, H, 601, 300)
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iii", W, H, NF))
        for k in range(NF):
            f.write(np.ascontiguousarray(fr["img_l"][k]).tobytes())
            f.write(np.ascontiguousarray(fr["img_r"][k]).tobytes())
    from test_track_images_lsd_host import build_lsd_example
    out = subprocess.run([build_lsd_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout
    rows = [line.split() for line in out.strip().splitlines()]
    assert len(rows) == NF - 1
    # the loop: B = 1 calls, thresholds from update_fast_threshold, priors by StereoFrameHandler.f2fTracking's rule
    mc, sc, tc, oc = configs(1200, 4)
    lc, hc, cam = T.default_lsd_config(), HandlerConfig(), T.kitti_camera()
    th = prev_th = hc.orb_fast_th
    state = dict(Tfw=np.eye(4), Tfw_cov=np.eye(6), DT=np.eye(4), DT_cov=np.zeros((6, 6)), err_norm=-1.0)
    ths = []
    for k in range(1, NF):
        pri = np.zeros(1, T.PRIOR_DTYPE)
        for key, v in state.items():
            pri[key][0] = v
        prev = dict(img_l=fr["img_l"][k - 1:k], img_r=fr["img_r"][k - 1:k], fast_th=[prev_th])
        curr = dict(img_l=fr["img_l"][k:k + 1], img_r=fr["img_r"][k:k + 1], fast_th=[th])
        res, ns = engine.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, prev, curr, pri)
        r, row = res[0], rows[k - 1]
        assert row[:2] == ["frame", str(k)] and row[2] == "th" and int(row[3]) == th, (row[:4], th)
        assert [int(x) for x in row[5:9]] == list(ns[0]), (row[5:9], ns[0])
        assert int(row[10]) == r["good"]
        np.testing.assert_array_equal(np.float64(row[12:28]).reshape(4, 4), r["DT"])
        ths.append(th)
        state = dict(Tfw=r["Tfw"], Tfw_cov=r["Tfw_cov"], DT=r["DT"], DT_cov=r["DT_cov"], err_norm=float(r["err_norm"]))
        prev_th, th = th, update_fast_threshold(hc, th, r["DT"], float(r["err_norm"]), int(r["n_inliers_pt"]))
    assert len(set(ths)) > 1, ths    # the adaptive threshold moved along the sequence
