"""Colour input on the GPU: plstvo_rectify_batch with colour rectifiers against oracle/color.py on every BGR triple and
against tests/golden/color.npz (cv2 4.13) bit for bit; the raw-images calls and sessions with colour rectifiers against
plstvo_rectify_batch (colour) followed by the _lsd_ call, byte for byte; grey frames replicated into BGR / BGRA against the
_lsd_ call on the grey frames; errors; and examples/color_images_cpp.cpp against a Python loop.  Needs neither cv2 nor the
reference sources."""
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import color as OC
from test_color_host import G, all_triples, assert_golden, build_color_example, case_image, case_maps
from test_gpu_rectify import rig
from test_gpu_stereo_session import Mirror, fresh, frames_of, stream_frames
from test_gpu_track_images import CAM_SMALL, assert_same, configs, frames_slice, moving_views, ragged_sets, sm_count
from test_gpu_track_images_lsd import images_only
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError, init_undistort_rectify_map

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_orb_golden as OG  # noqa: E402

pytestmark = pytest.mark.gpu


def colorize(g, channels, seed):
    """Colour images whose grey differs from each channel but keeps the grey texture: B = 255 - g (+-3 of seeded noise),
    G = g, R = g^2 / 255, seeded alpha."""
    rng = np.random.default_rng(seed)
    g16 = np.asarray(g).astype(np.int32)
    planes = [np.clip(255 - g16 + rng.integers(-3, 4, g16.shape), 0, 255), g16, g16 * g16 // 255]
    if channels == 4:
        planes.append(rng.integers(0, 256, g16.shape))
    return np.stack(planes, -1).astype(np.uint8)


def colorize_frames(d, channels, seed):
    out = dict(d)
    out["img_l"] = colorize(d["img_l"], channels, seed)
    out["img_r"] = colorize(d["img_r"], channels, seed + 1)
    return out


def color_rectifier(e, W, H, channels, maps=None):
    return e.rectifier_create_color(W, H, channels, *(maps or ()))


def color_chain(e, rect, cam, tc, mc, sc, oc, lc, sets, sequence, priors=None):
    """plstvo_rectify_batch (colour) on every pair, then the _lsd_ call on the grey images"""
    fed = []
    for s in sets:
        ol, orr = e.rectify_batch(rect, s["img_l"], s["img_r"])
        fed.append(dict(img_l=ol, img_r=orr, fast_th=s.get("fast_th")))
    if sequence:
        return e.track_stereo_images_lsd_sequence(cam, tc, mc, sc, oc, lc, fed[0], priors)
    return e.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, fed[0], fed[1], priors)


# ---- 1. the conversion on every BGR triple ----
@pytest.mark.parametrize("channels", [3, 4])
def test_exhaustive_conversion(engine, channels):
    img = all_triples(channels, seed=31)
    want = OC.bgr_to_gray(img)
    rect = engine.rectifier_create_color(4096, 4096, channels)
    ol, orr = engine.rectify_batch(rect, img, img[::-1].copy())
    np.testing.assert_array_equal(ol[0], want)
    np.testing.assert_array_equal(orr[0], want[::-1])
    assert engine.rectify_kernel_times() > 0
    engine.rectifier_destroy(rect)


# ---- 2. remap then convert: every golden case, batched ----
@pytest.mark.parametrize("size", ["1", "37", "sms+5"])
def test_every_golden_case(engine, size):
    B = {"1": 1, "37": 37}.get(size, sm_count() + 5)
    for c in G["cases"]:
        w, h = (int(v) for v in G[f"{c}_size"])
        channels = int(G[f"{c}_channels"])
        m1, m2 = case_maps(c)
        rect = engine.rectifier_create_color(w, h, channels, *(() if m1 is None else (m1, m2)))
        if B == 1:
            il, ir = case_image(c)[None], case_image(c)[None]
        else:   # the golden image first on the left and last on the right, seeded noise images between
            rng = np.random.default_rng(B + len(c))
            il = rng.integers(0, 256, (B, h, w, channels), dtype=np.uint8)
            ir = rng.integers(0, 256, (B, h, w, channels), dtype=np.uint8)
            il[0] = ir[-1] = case_image(c)
        ol, orr = engine.rectify_batch(rect, il, ir)
        assert_golden(c, ol[0])
        assert_golden(c, orr[-1])
        if B > 1:
            np.testing.assert_array_equal(ol[B // 2], OC.remap_gray(il[B // 2], m1, m2), err_msg=c)
            np.testing.assert_array_equal(orr[1], OC.remap_gray(ir[1], m1, m2), err_msg=c)
        engine.rectifier_destroy(rect)


def test_both_sides_own_maps(engine):
    """The EuRoC rig's two sides in one rectifier, 3 and 4 channels: each side's golden through its own maps."""
    for channels in (3, 4):
        cl, cr = f"c{channels}_euroc_l", f"c{channels}_euroc_r"
        rect = engine.rectifier_create_color(752, 480, channels, *case_maps(cl), *case_maps(cr))
        ol, orr = engine.rectify_batch(rect, case_image(cl)[None], case_image(cr)[None])
        assert_golden(cl, ol[0])
        assert_golden(cr, orr[0])
        engine.rectifier_destroy(rect)


# ---- 3. pipeline contract: raw-images calls on colour images ----
def kitti_maps():
    m1, m2 = case_maps("c3_kitti_d0")
    return m1, m2


@pytest.mark.parametrize("score", ["fast", "harris"])
@pytest.mark.parametrize("maps", [False, True])
def test_kitti_colour_batch_and_sequence(score, maps):
    cam = T.kitti_camera()
    fr = colorize_frames(images_only(moving_views(9, cam.width, cam.height, 711, 300, fast_th=[20, 0, 12, 35, 20, 5, 0, 50, 20])),
                         3, 50)
    mc, sc, tc, oc = configs(1200, 4, T.ORB_HARRIS_SCORE if score == "harris" else T.ORB_FAST_SCORE)
    lc = T.default_lsd_config()
    e = Engine()
    rect = color_rectifier(e, cam.width, cam.height, 3, kitti_maps() if maps else None)
    seq = e.track_stereo_raw_images_sequence(cam, tc, mc, sc, oc, lc, rect, fr)
    assert_same(seq, color_chain(e, rect, cam, tc, mc, sc, oc, lc, [fr], True))
    prev, curr = frames_slice(fr, 0, 8), frames_slice(fr, 1, 9)
    bat = e.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, rect, prev, curr)
    assert_same(bat, color_chain(e, rect, cam, tc, mc, sc, oc, lc, [prev, curr], False))
    assert seq[0].tobytes() == bat[0].tobytes()
    assert (seq[1][:, 0] > 50).all() and (seq[1][:, 1] > 10).all(), seq[1]
    ms = e.track_stereo_images_stage_times()
    assert ms[0] > 0 and e.rectify_kernel_times() > 0, ms
    e.close()


def test_euroc_rig_bgra():
    cam, maps = rig("euroc")
    fr = colorize_frames(images_only(moving_views(5, 752, 480, 812, 200)), 4, 60)
    mc, sc, tc, oc = configs(1200, 4)
    lc = T.default_lsd_config()
    e = Engine()
    rect = e.rectifier_create_color(752, 480, 4, *maps)
    seq = e.track_stereo_raw_images_sequence(cam, tc, mc, sc, oc, lc, rect, fr)
    assert_same(seq, color_chain(e, rect, cam, tc, mc, sc, oc, lc, [fr], True))
    assert (seq[1][:, 0] > 0).all(), seq[1]
    e.close()


MODES = ["both", "points_only", "lines_only"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("size", ["9", "37", "sms+5"])
def test_ragged_colour_batch_equals_rectify_then_lsd(mode, size):
    """9 pairs take the path where LSD runs before ORB, SMs + 5 the one where they overlap; with and without maps."""
    B = {"9": 9, "37": 37}.get(size, sm_count() + 5)
    channels = 3
    prev, curr = (colorize_frames(images_only(d), channels, 90 + 2 * B + 2 * j) for j, d in enumerate(ragged_sets(B, 8800 + B)))
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    if mode == "points_only":
        tc.has_lines = 0
    if mode == "lines_only":
        tc.has_points = 0
    rng = np.random.default_rng(B)
    mx = (np.arange(320)[None, :] + rng.uniform(-2, 2, (240, 320))).astype(np.float32)
    my = (np.arange(240)[:, None] + rng.uniform(-2, 2, (240, 320))).astype(np.float32)
    ix, iy = np.rint(mx * 32).astype(np.int64), np.rint(my * 32).astype(np.int64)
    m1 = np.stack([ix >> 5, iy >> 5], -1).astype(np.int16)
    m2 = ((iy & 31) * 32 + (ix & 31)).astype(np.uint16)
    e = Engine()
    for maps in (None, (m1, m2, m1[::-1].copy(), m2[::-1].copy())):
        rect = color_rectifier(e, 320, 240, channels, maps)
        got = e.track_stereo_raw_images_batch(CAM_SMALL, tc, mc, sc, oc, lc, rect, prev, curr)
        assert_same(got, color_chain(e, rect, CAM_SMALL, tc, mc, sc, oc, lc, [prev, curr], False))
        e.rectifier_destroy(rect)
    e.close()


# ---- 4. grey replicated into BGR / BGRA: the colour path on the chain pinned to cv2 ----
@pytest.mark.parametrize("channels", [3, 4])
def test_replicated_grey_equals_the_lsd_call(engine, channels):
    kv = OG.kitti_views()
    cam = T.kitti_camera()
    prev, curr = (dict(img_l=kv[2 * f:2 * f + 1], img_r=kv[2 * f + 1:2 * f + 2], fast_th=None) for f in range(2))
    rng = np.random.default_rng(channels)

    def rep(g):
        planes = [g, g, g] + ([rng.integers(0, 256, g.shape).astype(np.uint8)] if channels == 4 else [])
        return np.stack(planes, -1)

    cp, cc = ({**d, "img_l": rep(d["img_l"]), "img_r": rep(d["img_r"])} for d in (prev, curr))
    mc, sc, tc, oc = configs()
    lc = T.default_lsd_config()
    rect = engine.rectifier_create_color(cam.width, cam.height, channels)
    got = engine.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, rect, cp, cc)
    want = engine.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, prev, curr)
    assert_same(got, want)
    assert got[1][0, 0] > 50 and got[1][0, 1] > 10, got[1]
    engine.rectifier_destroy(rect)


# ---- 5. sessions: colour inserts equal the colour batch call ----
def scribble(frames, rng):
    for k in ("img_l", "img_r"):
        frames[k][...] = rng.integers(0, 256, frames[k].shape, np.uint8)


@pytest.mark.parametrize("maps", [False, True])
def test_one_stream_session(maps):
    cam, rmaps = rig("euroc") if maps else (T.kitti_camera(), None)
    fr = colorize_frames(images_only(moving_views(7, cam.width, cam.height, 613, 200, fast_th=[20, 0, 12, 35, 20, 5, 0])),
                         4 if maps else 3, 70)
    mc, sc, tc, oc = configs(1200, 4)
    lc = T.default_lsd_config()
    e = Engine()
    rect = color_rectifier(e, cam.width, cam.height, 4 if maps else 3, rmaps)
    ss = e.stereo_session_create(cam, tc, mc, sc, oc, lc, rect, 1)
    rng = np.random.default_rng(9)
    m = Mirror()
    f0 = fresh(frames_slice(fr, 0, 1))
    ss.initialize([0], f0)
    m.keep([0], frames_slice(fr, 0, 1))
    scribble(f0, rng)
    for k in range(1, 7):
        cur = frames_slice(fr, k, k + 1)
        given = fresh(cur)
        got = ss.insert([0], given)
        scribble(given, rng)
        assert_same(got, m.batch(e, cam, tc, mc, sc, oc, lc, rect, [0], cur))
        m.keep([0], cur)
    assert got[1][0, 1] > 0, got[1]
    with pytest.raises(ValueError, match="channels"):
        ss.insert([0], images_only(moving_views(2, cam.width, cam.height, 5, 0)))   # grey frames on a colour session
    e.close()


def test_many_streams_uneven_arrival():
    S, NF = 37, 6
    st = [colorize_frames(d, 3, 400 + s) for s, d in enumerate(stream_frames(S, NF, 4900))]
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e = Engine()
    rect = e.rectifier_create_color(320, 240, 3)
    ss = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, rect, S)
    rng = np.random.default_rng(S)
    m = Mirror()
    pos = {i: 0 for i in range(S)}
    order = rng.permutation(S)
    for ids in (order[:S // 3], order[S // 3:]):
        fr = frames_of(st, ids, pos)
        given = fresh(fr)
        ss.initialize(ids, given)
        scribble(given, rng)
        m.keep(ids, fr)
    for n in (S, 5, S // 2, 9):
        pool = [i for i in range(S) if pos[i] + 1 < NF]
        ids = np.int32(rng.permutation(pool)[:n])
        for i in ids:
            pos[int(i)] += 1
        fr = frames_of(st, ids, pos)
        given = fresh(fr)
        got = ss.insert(ids, given)
        scribble(given, rng)
        assert_same(got, m.batch(e, CAM_SMALL, tc, mc, sc, oc, lc, rect, ids, fr))
        m.keep(ids, fr)
    e.close()


# ---- 6. errors ----
def test_errors_leave_the_context_usable():
    prev, curr = (colorize_frames(images_only(d), 3, 95 + 2 * j) for j, d in enumerate(ragged_sets(6, 9600)))
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e = Engine()
    rect = e.rectifier_create_color(320, 240, 3)
    want = e.track_stereo_raw_images_batch(CAM_SMALL, tc, mc, sc, oc, lc, rect, prev, curr)
    i16p, u16p = C.POINTER(C.c_int16), C.POINTER(C.c_uint16)
    m1, m2 = np.zeros((240, 320, 2), np.int16), np.zeros((240, 320), np.uint16)
    p1, p2 = m1.ctypes.data_as(i16p), m2.ctypes.data_as(u16p)
    n1, n2 = C.cast(None, i16p), C.cast(None, u16p)

    def create(w, h, ch, a=n1, b=n2, c=n1, d=n2):
        r = e.lib.plstvo_rectifier_create_color(e.ctx, w, h, ch, a, b, c, d)
        return r, (e.lib.plstvo_last_error(e.ctx) or b"").decode()

    def still_usable():
        assert_same(e.track_stereo_raw_images_batch(CAM_SMALL, tc, mc, sc, oc, lc, rect, prev, curr), want)

    for ch in (0, 1, 2, 5):
        r, msg = create(320, 240, ch)
        assert r is None and "channels must be 3 (BGR) or 4 (BGRA)" in msg, (ch, msg)
    for w, h in ((0, 240), (320, 32768), (-1, 1)):
        r, msg = create(w, h, 3)
        assert r is None and "width and height must be 1..32767" in msg, (w, h, msg)
    for maps in ((p1, n2, n1, n2), (p1, p2, n1, n2), (p1, p2, p1, n2), (n1, n2, n1, p2)):
        r, msg = create(320, 240, 4, *maps)
        assert r is None and "maps must be all four or none" in msg, msg
    still_usable()

    def call(r, cam=CAM_SMALL):
        ps, kp = T.stereo_images_as_c(prev)
        cs, kc = T.stereo_images_as_c(curr)
        res = np.zeros(ps.B, T.POSE_RESULT_DTYPE)
        rc = e.lib.plstvo_track_stereo_raw_images_batch(e.ctx, C.byref(cam), C.byref(tc), C.byref(mc), C.byref(sc),
                                                        C.byref(oc), C.byref(lc), r, C.byref(ps), C.byref(cs), None,
                                                        res.ctypes.data, None)
        return rc, (e.lib.plstvo_last_error(e.ctx) or b"").decode()

    other = Engine()
    foreign = other.rectifier_create_color(320, 240, 3)
    rc, msg = call(foreign.handle)
    assert rc == -1 and "the rectifier belongs to another context" in msg, (rc, msg)
    still_usable()
    small = e.rectifier_create_color(160, 120, 3)
    rc, msg = call(small.handle)
    assert rc == -5 and "rectifier size differs from the camera's" in msg, (rc, msg)
    still_usable()
    with pytest.raises(PlstvoError, match="rectifier size differs"):
        e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, small, 2)
    still_usable()
    with pytest.raises(ValueError, match="channels"):
        e.rectify_batch(rect, prev["img_l"][..., 0], prev["img_r"][..., 0])
    with pytest.raises(ValueError, match="channels"):
        e.track_stereo_raw_images_batch(CAM_SMALL, tc, mc, sc, oc, lc, rect, images_only(ragged_sets(6, 1)[0]), curr)
    still_usable()
    other.close()
    e.close()


# ---- 7. StereoImageHandler with a colour Rectifier (examples/color_images_cpp.cpp) against a Python loop ----
@pytest.mark.parametrize("maps", [False, True])
def test_color_example_equals_python_loop(engine, tmp_path, maps):
    from stvo_pl_b200.handler import HandlerConfig, update_fast_threshold
    NF, cam, channels = 8, T.kitti_camera(), 3
    d = (-0.2, 0.05, 0.001, -0.0008) if maps else (0.0, 0.0, 0.0, 0.0)
    fr = colorize_frames(images_only(moving_views(NF, cam.width, cam.height, 602, 300)), channels, 80)
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiiii", cam.width, cam.height, NF, channels, int(maps)))
        f.write(struct.pack("<9d", cam.fx, cam.fy, cam.cx, cam.cy, cam.b, *d))
        for k in range(NF):
            f.write(np.ascontiguousarray(fr["img_l"][k]).tobytes())
            f.write(np.ascontiguousarray(fr["img_r"][k]).tobytes())
    out = subprocess.run([build_color_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout
    rows = [line.split() for line in out.strip().splitlines()]
    assert len(rows) == NF - 1
    if maps:   # StereoRectification::camD0: K, D, P in float, P's fy = fx, R = I, one map for both sides
        f32 = lambda v: float(np.float32(v))   # noqa: E731
        K = np.array([[f32(cam.fx), 0, f32(cam.cx)], [0, f32(cam.fy), f32(cam.cy)], [0, 0, 1]])
        P = np.array([[f32(cam.fx), 0, f32(cam.cx), 0], [0, f32(cam.fx), f32(cam.cy), 0], [0, 0, 1, 0]])
        m1, m2 = init_undistort_rectify_map(T.RECTIFY_PINHOLE, K, [f32(v) for v in d] + [0.0], np.eye(3), P, cam.width,
                                            cam.height)
        rcam = T.PlCamera(fx=P[0, 0], fy=P[1, 1], cx=P[0, 2], cy=P[1, 2], b=cam.b, width=cam.width, height=cam.height)
        rect = engine.rectifier_create_color(cam.width, cam.height, channels, m1, m2)
    else:
        rcam = cam
        rect = engine.rectifier_create_color(cam.width, cam.height, channels)
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
