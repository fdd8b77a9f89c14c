"""Rectification on the GPU: plstvo_rectify_batch against tests/golden/rectify.npz (cv2 4.13) and oracle/rectify.py bit for
bit, and plstvo_track_stereo_raw_images_batch / _sequence against plstvo_rectify_batch followed by the _lsd_ call byte for
byte; rect == NULL, reuse, errors, and a distorted sequence tracked from its raw images.  Needs neither cv2 nor the
reference sources."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from test_gpu_track_images import CAM_SMALL, assert_same, configs, frames_slice, moving_views, ragged_sets, sm_count
from test_gpu_track_images_lsd import images_only, same
from oracle import rectify as R
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError, init_undistort_rectify_map

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_orb_golden as OG  # noqa: E402
import make_rectify_golden as M  # noqa: E402

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(GOLDEN, "rectify.npz"))


def case_args(c):
    w, h = (int(v) for v in G[f"{c}_size"])
    return int(G[f"{c}_model"]), G[f"{c}_K"], G[f"{c}_D"], G[f"{c}_R"], G[f"{c}_P"], w, h


def case_maps(c):
    m1, m2 = init_undistort_rectify_map(*case_args(c))
    assert (M.sha(m1, m2) == G[f"{c}_map_sha"]).all(), c
    return m1, m2


def rig(name):
    """(rectified PlCamera, rectifier maps (m1l, m2l, m1r, m2r)) of a golden rig"""
    if name == "euroc":
        l, r = case_maps("euroc_l"), case_maps("euroc_r")
        fx, fy, cx, cy, b = G["euroc_l_cam"]
        return T.PlCamera(fx=fx, fy=fy, cx=cx, cy=cy, b=b, width=752, height=480), (*l, *r)
    m = case_maps("kitti_d0")
    return T.kitti_camera(), (*m, *m)


# ---- 1. remap against the golden and the restatement ----
@pytest.mark.parametrize("size", ["1", "37", "sms+5"])
def test_rectify_batch_equals_golden_and_restatement(engine, size):
    B = {"1": 1, "37": 37}.get(size, sm_count() + 5)
    m1l, m2l, m1r, m2r = case_maps("euroc_l") + case_maps("euroc_r")
    rect = engine.rectifier_create(m1l, m2l, m1r, m2r)
    W, H = 752, 480
    il = np.stack([M.image(int(G["euroc_l_seed"]) if b == 0 else 3000 + b, W, H) for b in range(B)])
    ir = np.stack([M.image(int(G["euroc_r_seed"]) if b == 0 else 6000 + b, W, H) for b in range(B)])
    ol, orr = engine.rectify_batch(rect, il, ir)
    assert (M.sha(ol[0]) == G["euroc_l_out_sha"]).all() and (M.sha(orr[0]) == G["euroc_r_out_sha"]).all()
    for b in sorted({0, B // 2, B - 1}):
        np.testing.assert_array_equal(ol[b], R.remap(il[b], m1l, m2l))
        np.testing.assert_array_equal(orr[b], R.remap(ir[b], m1r, m2r))
    assert engine.rectify_kernel_times() > 0
    engine.rectifier_destroy(rect)


def test_every_golden_case(engine):
    """Each map case on its seeded image (one side, both sides given the same maps), each remap case on its maps."""
    for c in list(G["map_cases"]) + list(G["remap_cases"]):
        w, h = (int(v) for v in G[f"{c}_size"])
        m1, m2 = (G[f"{c}_map1"], G[f"{c}_map2"]) if f"{c}_map1" in G else case_maps(c)
        img = M.image(int(G[f"{c}_seed"]), w, h)
        rect = engine.rectifier_create(m1, m2)
        ol, orr = engine.rectify_batch(rect, img[None], img[None])
        want = G[f"{c}_out"] if f"{c}_out" in G else None
        if want is not None:
            np.testing.assert_array_equal(ol[0], want, err_msg=c)
        else:
            assert (M.sha(ol[0]) == G[f"{c}_out_sha"]).all(), c
        np.testing.assert_array_equal(orr[0], ol[0])
        engine.rectifier_destroy(rect)


def test_more_than_65535_images(engine):
    c = "remap_8x8"
    rect = engine.rectifier_create(G[f"{c}_map1"], G[f"{c}_map2"])
    B = 33000   # 66000 images: two grid slices
    rng = np.random.default_rng(5)
    il = rng.integers(0, 256, (B, 8, 8), dtype=np.uint8)
    ir = rng.integers(0, 256, (B, 8, 8), dtype=np.uint8)
    ol, orr = engine.rectify_batch(rect, il, ir)
    for b in (0, 1, 32767, 32768, B - 1):
        np.testing.assert_array_equal(ol[b], R.remap(il[b], G[f"{c}_map1"], G[f"{c}_map2"]))
        np.testing.assert_array_equal(orr[b], R.remap(ir[b], G[f"{c}_map1"], G[f"{c}_map2"]))
    engine.rectifier_destroy(rect)


def test_identity_map_copies(engine):
    for W, H in ((752, 480), (13, 7), (1, 1)):
        y, x = np.mgrid[0:H, 0:W]
        m1 = np.stack([x, y], -1).astype(np.int16)
        m2 = np.zeros((H, W), np.uint16)
        rect = engine.rectifier_create(m1, m2)
        il = np.stack([M.image(s, W, H) for s in (1, 2, 3)])
        ir = np.stack([M.image(s, W, H) for s in (4, 5, 6)])
        ol, orr = engine.rectify_batch(rect, il, ir)
        np.testing.assert_array_equal(ol, il)
        np.testing.assert_array_equal(orr, ir)
        engine.rectifier_destroy(rect)


# ---- 2. raw images in, pose out ----
def rectified_chain(e, rect, cam, tc, mc, sc, oc, lc, sets, sequence, priors=None):
    """plstvo_rectify_batch on every pair, then the _lsd_ call on the rectified images"""
    fed = []
    for s in sets:
        ol, orr = e.rectify_batch(rect, s["img_l"], s["img_r"])
        fed.append(dict(img_l=ol, img_r=orr, fast_th=s.get("fast_th")))
    if sequence:
        return e.track_stereo_images_lsd_sequence(cam, tc, mc, sc, oc, lc, fed[0], priors)
    return e.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, fed[0], fed[1], priors)


def test_kitti_golden_frames_cam_d0(engine):
    cam, maps = rig("kitti")
    rect = engine.rectifier_create(*maps)
    kv = OG.kitti_views()
    prev, curr = (dict(img_l=kv[2 * f:2 * f + 1], img_r=kv[2 * f + 1:2 * f + 2], fast_th=None) for f in range(2))
    mc, sc, tc, oc = configs()
    lc = T.default_lsd_config()
    got = engine.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, rect, prev, curr)
    assert_same(got, rectified_chain(engine, rect, cam, tc, mc, sc, oc, lc, [prev, curr], False))
    assert got[1][0, 0] > 50 and got[1][0, 1] > 10, got[1]
    ms = engine.track_stereo_images_stage_times()
    assert ms[0] > 0 and engine.rectify_kernel_times() > 0, ms
    # rect == NULL is the _lsd_ call
    assert_same(engine.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, None, prev, curr),
                engine.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, prev, curr))
    engine.rectifier_destroy(rect)


def test_euroc_sequence_and_batch(engine):
    cam, maps = rig("euroc")
    rect = engine.rectifier_create(*maps)
    fr = images_only(moving_views(9, 752, 480, 811, 200, fast_th=[20, 0, 12, 35, 20, 5, 0, 50, 20]))
    mc, sc, tc, oc = configs(1200, 4)
    lc = T.default_lsd_config()
    seq = engine.track_stereo_raw_images_sequence(cam, tc, mc, sc, oc, lc, rect, fr)
    assert_same(seq, rectified_chain(engine, rect, cam, tc, mc, sc, oc, lc, [fr], True))
    prev, curr = frames_slice(fr, 0, 8), frames_slice(fr, 1, 9)
    bat = engine.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, rect, prev, curr)
    assert_same(bat, rectified_chain(engine, rect, cam, tc, mc, sc, oc, lc, [prev, curr], False))
    assert seq[0].tobytes() == bat[0].tobytes()
    assert (seq[1][:, 0] > 0).all(), seq[1]   # few: the rig's rectification warps the fronto-parallel texture
    engine.rectifier_destroy(rect)


MODES = ["both", "points_only", "lines_only"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("size", ["9", "sms+5"])
def test_ragged_batch_equals_rectify_then_lsd(mode, size):
    """9 pairs take the path where LSD runs before ORB, SMs + 5 the one where they overlap; both on the remap's copy."""
    B = {"9": 9}.get(size, sm_count() + 5)
    prev, curr = (images_only(d) for d in ragged_sets(B, 8700 + B))
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    if mode == "points_only":
        tc.has_lines = 0
    if mode == "lines_only":
        tc.has_points = 0
    rng = np.random.default_rng(B)
    mx = (np.arange(320)[None, :] + rng.uniform(-2, 2, (240, 320))).astype(np.float32)
    my = (np.arange(240)[:, None] + rng.uniform(-2, 2, (240, 320))).astype(np.float32)
    # a convertMaps-style map built in NumPy: round(x * 32), integer part and fraction
    ix, iy = np.rint(mx * 32).astype(np.int64), np.rint(my * 32).astype(np.int64)
    m1 = np.stack([ix >> 5, iy >> 5], -1).astype(np.int16)
    m2 = ((iy & 31) * 32 + (ix & 31)).astype(np.uint16)
    e = Engine()
    rect = e.rectifier_create(m1, m2, m1[::-1].copy(), m2[::-1].copy())
    got = e.track_stereo_raw_images_batch(CAM_SMALL, tc, mc, sc, oc, lc, rect, prev, curr)
    assert_same(got, rectified_chain(e, rect, CAM_SMALL, tc, mc, sc, oc, lc, [prev, curr], False))
    e.close()


def test_reuse_with_a_rectifier_destroyed_between():
    cam, maps = rig("kitti")
    kv = OG.kitti_views()
    kp, kc = (dict(img_l=kv[2 * f:2 * f + 1], img_r=kv[2 * f + 1:2 * f + 2], fast_th=None) for f in range(2))
    sp, scu = (images_only(d) for d in ragged_sets(9, 9300))
    mc, sc, tc, oc = configs()
    mc2, sc2, tc2, oc2 = configs(500, 4)
    lc = T.default_lsd_config()
    small = M.image(9, 320, 240)
    y, x = np.mgrid[0:240, 0:320]
    sm1 = np.stack([x[:, ::-1], y], -1).astype(np.int16)   # a mirror
    sm2 = np.zeros((240, 320), np.uint16)

    def run(e, rects):
        return [e.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, rects["kitti"], kp, kc),
                e.track_stereo_raw_images_batch(CAM_SMALL, tc2, mc2, sc2, oc2, lc, rects["mirror"], sp, scu),
                e.rectify_batch(rects["mirror"], small[None], small[None]),
                e.track_stereo_images_lsd_batch(CAM_SMALL, tc2, mc2, sc2, oc2, lc, sp, scu)]

    e = Engine()
    fresh = run(e, dict(kitti=e.rectifier_create(*maps), mirror=e.rectifier_create(sm1, sm2)))
    e.close()
    e = Engine()
    k = e.rectifier_create(*maps)
    first = run(e, dict(kitti=k, mirror=e.rectifier_create(sm1, sm2)))
    e.rectifier_destroy(k)
    second = run(e, dict(kitti=e.rectifier_create(*maps), mirror=e.rectifier_create(sm1, sm2)))
    same(first, fresh)
    same(second, fresh)
    np.testing.assert_array_equal(first[2][0][0], small[:, ::-1])
    e.close()


def test_errors_leave_the_context_usable():
    prev, curr = (images_only(d) for d in ragged_sets(6, 9500))
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    y, x = np.mgrid[0:240, 0:320]
    m1, m2 = np.stack([x, y], -1).astype(np.int16), np.zeros((240, 320), np.uint16)
    e = Engine()
    rect = e.rectifier_create(m1, m2)
    want = e.track_stereo_raw_images_batch(CAM_SMALL, tc, mc, sc, oc, lc, rect, prev, curr)
    assert_same(want, e.track_stereo_images_lsd_batch(CAM_SMALL, tc, mc, sc, oc, lc, prev, curr))   # identity maps

    def call(r, cam=CAM_SMALL, lcfg=lc, sequence=False):
        ps, kp = T.stereo_images_as_c(prev)
        cs, kc = T.stereo_images_as_c(curr)
        res = np.zeros(ps.B, T.POSE_RESULT_DTYPE)
        lcp = None if lcfg is None else C.byref(lcfg)
        if sequence:
            rc = e.lib.plstvo_track_stereo_raw_images_sequence(e.ctx, C.byref(cam), C.byref(tc), C.byref(mc), C.byref(sc),
                                                               C.byref(oc), lcp, r, C.byref(ps), None, res.ctypes.data, None)
        else:
            rc = e.lib.plstvo_track_stereo_raw_images_batch(e.ctx, C.byref(cam), C.byref(tc), C.byref(mc), C.byref(sc),
                                                            C.byref(oc), lcp, r, C.byref(ps), C.byref(cs), None,
                                                            res.ctypes.data, None)
        return rc, (e.lib.plstvo_last_error(e.ctx) or b"").decode()

    def check(got, rc, text):
        assert got[0] == rc and text in got[1], (got, rc, text)
        assert_same(e.track_stereo_raw_images_batch(CAM_SMALL, tc, mc, sc, oc, lc, rect, prev, curr), want)

    small = e.rectifier_create(m1[:120, :160].copy(), m2[:120, :160].copy())
    check(call(small.handle), -5, "rectifier size differs from the camera's")
    check(call(small.handle, sequence=True), -5, "rectifier size differs from the camera's")
    other = Engine()
    foreign = other.rectifier_create(m1, m2)
    check(call(foreign.handle), -1, "the rectifier belongs to another context")
    ol = np.zeros((1, 240, 320), np.uint8)
    u8 = ol.ctypes.data_as(T.c_uint8_p)
    rc = e.lib.plstvo_rectify_batch(e.ctx, foreign.handle, 1, u8, u8, u8, u8)
    assert rc == -1 and b"another context" in e.lib.plstvo_last_error(e.ctx)
    check(call(rect.handle, lcfg=T.default_lsd_config(refine=1)), -1, "lsd refine")
    check(call(rect.handle, lcfg=None), -1, "null lsd config")
    big_cam = T.PlCamera(fx=300.0, fy=300.0, cx=160.0, cy=120.0, b=0.2, width=640, height=240)
    big = e.rectifier_create(np.zeros((240, 640, 2), np.int16), np.zeros((240, 640), np.uint16))
    check(call(big.handle, cam=big_cam), -5, "image size differs from the camera's")
    with pytest.raises(PlstvoError, match="width and height must be 1..32767"):
        e.rectifier_create(np.zeros((1, 40000, 2), np.int16), np.zeros((1, 40000), np.uint16))
    assert e.lib.plstvo_rectifier_create(e.ctx, 320, 240, None, None, None, None) is None
    assert "null map" in e.lib.plstvo_last_error(e.ctx).decode()
    with pytest.raises(PlstvoError, match="null rectifier"):
        e._ck(e.lib.plstvo_rectify_batch(e.ctx, None, 1, None, None, None, None))
    other.close()
    e.close()


# ---- 3. a distorted sequence tracked from its raw images ----
EUROC_D = np.array(M.EUROC_DL)


def distort(img, K, D):
    """What a camera with intrinsics K and radial-tangential D records of the undistorted view img (pinhole K): for each raw
    pixel the undistorted point by fixed-point iteration (as cv::undistortPoints), sampled bilinearly; outside: 0."""
    H, W = img.shape
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    xd, yd = (u - cx) / fx, (v - cy) / fy
    x, y = xd.copy(), yd.copy()
    k1, k2, p1, p2 = D
    for _ in range(20):
        r2 = x * x + y * y
        kr = 1 + (k2 * r2 + k1) * r2
        x = (xd - (2 * p1 * x * y + p2 * (r2 + 2 * x * x))) / kr
        y = (yd - (p1 * (r2 + 2 * y * y) + 2 * p2 * x * y)) / kr
    su, sv = x * fx + cx, y * fy + cy
    x0, y0 = np.floor(su).astype(np.int64), np.floor(sv).astype(np.int64)
    ax, ay = su - x0, sv - y0
    f = img.astype(np.float64)

    def tap(xx, yy):
        ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        return np.where(ok, f[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], 0.0)

    out = ((1 - ax) * (1 - ay) * tap(x0, y0) + ax * (1 - ay) * tap(x0 + 1, y0) + (1 - ax) * ay * tap(x0, y0 + 1)
           + ax * ay * tap(x0 + 1, y0 + 1))
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def test_distorted_sequence_recovers_the_motion(engine):
    """The 9-frame sequence rendered through EuRoC's distortion on KITTI's intrinsics (cam_d0 form: R = I, P = K): the raw
    call on the distorted images against the _lsd_ call on the undistorted ones.  Not a byte contract (interpolation moves
    the features); the bar was set from the first H100 run, DESIGN.md records the numbers."""
    cam = T.kitti_camera()
    K = np.array([[cam.fx, 0, cam.cx], [0, cam.fy, cam.cy], [0, 0, 1]])
    P = np.hstack([K, np.zeros((3, 1))])
    m1, m2 = init_undistort_rectify_map(T.RECTIFY_PINHOLE, K, EUROC_D, np.eye(3), P, cam.width, cam.height)
    fr = images_only(moving_views(9, cam.width, cam.height, 501, 300))
    raw = dict(img_l=np.stack([distort(i, K, EUROC_D) for i in fr["img_l"]]),
               img_r=np.stack([distort(i, K, EUROC_D) for i in fr["img_r"]]), fast_th=None)
    mc, sc, tc, oc = configs(1200, 4)
    lc = T.default_lsd_config()
    rect = engine.rectifier_create(m1, m2)
    got, n_got = engine.track_stereo_raw_images_sequence(cam, tc, mc, sc, oc, lc, rect, raw)
    ref, n_ref = engine.track_stereo_images_lsd_sequence(cam, tc, mc, sc, oc, lc, fr)
    dt = np.array([np.linalg.norm(g[:3, 3] - r[:3, 3]) for g, r in zip(got["DT"], ref["DT"])])
    ang = []
    for g, r in zip(got["DT"], ref["DT"]):
        Dm = g[:3, :3] @ r[:3, :3].T
        ang.append(np.arccos(np.clip((np.trace(Dm) - 1) / 2, -1, 1)))
    step = np.array([np.linalg.norm(r[:3, 3]) for r in ref["DT"]])
    print("distorted sequence: |dt| max %.3e m (ref step %.3e m), rotation max %.3e rad, good %s, stereo pts %s vs %s"
          % (dt.max(), step.mean(), max(ang), list(got["good"]), list(n_got[:, 0]), list(n_ref[:, 0])))
    assert (got["good"] == 1).all()
    assert dt.max() < 0.1 * step.mean() + 1e-3 and max(ang) < 5e-3, (dt, ang)
    engine.rectifier_destroy(rect)


# ---- 4. StereoImageHandler with a Rectifier (examples/raw_images_cpp.cpp) against a Python loop ----
def test_handler_example_equals_python_loop(engine, tmp_path):
    import struct
    import subprocess
    from stvo_pl_b200.handler import HandlerConfig, update_fast_threshold
    from test_rectify_host import build_raw_example
    NF, cam = 9, T.kitti_camera()
    d = (-0.2, 0.05, 0.001, -0.0008)   # cam_d0 .. cam_d3: the example stores them in float, as the reference does
    fr = images_only(moving_views(NF, cam.width, cam.height, 601, 300))
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iii", cam.width, cam.height, NF))
        f.write(struct.pack("<9d", cam.fx, cam.fy, cam.cx, cam.cy, cam.b, *d))
        for k in range(NF):
            f.write(np.ascontiguousarray(fr["img_l"][k]).tobytes())
            f.write(np.ascontiguousarray(fr["img_r"][k]).tobytes())
    out = subprocess.run([build_raw_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout
    rows = [line.split() for line in out.strip().splitlines()]
    assert len(rows) == NF - 1
    # StereoRectification::camD0: K, D, P in float, P's fy = fx, R = I, one map for both sides
    f32 = lambda v: float(np.float32(v))   # noqa: E731
    K = np.array([[f32(cam.fx), 0, f32(cam.cx)], [0, f32(cam.fy), f32(cam.cy)], [0, 0, 1]])
    P = np.array([[f32(cam.fx), 0, f32(cam.cx), 0], [0, f32(cam.fx), f32(cam.cy), 0], [0, 0, 1, 0]])
    m1, m2 = init_undistort_rectify_map(T.RECTIFY_PINHOLE, K, [f32(v) for v in d] + [0.0], np.eye(3), P, cam.width, cam.height)
    rcam = T.PlCamera(fx=P[0, 0], fy=P[1, 1], cx=P[0, 2], cy=P[1, 2], b=cam.b, width=cam.width, height=cam.height)
    rect = engine.rectifier_create(m1, m2)
    mc, sc, tc, oc = configs(1200, 4)
    lc, hc = T.default_lsd_config(), HandlerConfig()
    th = prev_th = hc.orb_fast_th
    state = dict(Tfw=np.eye(4), Tfw_cov=np.eye(6), DT=np.eye(4), DT_cov=np.zeros((6, 6)), err_norm=-1.0)
    for k in range(1, NF):
        pri = np.zeros(1, T.PRIOR_DTYPE)
        for key, v in state.items():
            pri[key][0] = v
        prev = dict(img_l=fr["img_l"][k - 1:k], img_r=fr["img_r"][k - 1:k], fast_th=[prev_th])
        curr = dict(img_l=fr["img_l"][k:k + 1], img_r=fr["img_r"][k:k + 1], fast_th=[th])
        res, ns = engine.track_stereo_raw_images_batch(rcam, tc, mc, sc, oc, lc, rect, prev, curr, pri)
        r, row = res[0], rows[k - 1]
        assert row[:2] == ["frame", str(k)] and row[2] == "th" and int(row[3]) == th, (row[:4], th)
        assert [int(x) for x in row[5:9]] == list(ns[0]), (row[5:9], ns[0])
        assert int(row[10]) == r["good"]
        np.testing.assert_array_equal(np.float64(row[12:28]).reshape(4, 4), r["DT"])
        state = dict(Tfw=r["Tfw"], Tfw_cov=r["Tfw_cov"], DT=r["DT"], DT_cov=r["DT_cov"], err_norm=float(r["err_norm"]))
        prev_th, th = th, update_fast_threshold(hc, th, r["DT"], float(r["err_norm"]), int(r["n_inliers_pt"]))
    engine.rectifier_destroy(rect)
