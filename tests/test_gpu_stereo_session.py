"""plstvo_stereo_session_* on the GPU: each stream's previous frame kept in HBM.  Every insert equals, byte for byte in results
and n_stereo, plstvo_track_stereo_raw_images_batch (rect NULL: the _lsd_ batch call) on (each named stream's kept images at
the threshold they were detected with, the new images) in the same order.  One stream with and without a rectifier and under
the config switches; many streams with uneven arrival across both sides of the LSD-first rule and of the K2 / streamed
policy; caller buffers overwritten after every call; errors; reuse beside other calls; and examples/streams_cpp.cpp
(plstvo::StereoStreamsHandler) against a Python loop of the handler rules.  Needs neither cv2 nor the reference sources."""
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

from test_gpu_track_images import CAM_SMALL, assert_same, configs, frames_slice, moving_views, sm_count
from test_gpu_track_images_lsd import images_only, same
from test_gpu_rectify import rig
from stvo_pl_b200 import synth
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError
from stvo_pl_b200.handler import HandlerConfig, KeyframeTest, update_fast_threshold

pytestmark = pytest.mark.gpu


class Mirror:
    """The test's own record of each stream's kept images and threshold: what the batch call is fed as prev."""

    def __init__(self):
        self.kept = {}

    def batch(self, e, cam, tc, mc, sc, oc, lc, rect, ids, curr, priors=None):
        prev = dict(img_l=np.stack([self.kept[i][0] for i in ids]), img_r=np.stack([self.kept[i][1] for i in ids]),
                    fast_th=np.int32([self.kept[i][2] for i in ids]))
        return e.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, rect, prev, curr, priors)

    def keep(self, ids, frames):
        th = frames.get("fast_th")
        for k, i in enumerate(ids):
            self.kept[i] = (frames["img_l"][k].copy(), frames["img_r"][k].copy(), 0 if th is None else int(th[k]))


def fresh(frames):
    """Copies the session call is given; they are overwritten with noise after the call."""
    return {k: None if v is None else np.array(v) for k, v in frames.items()}


def scribble(frames, rng):
    for k in ("img_l", "img_r"):
        frames[k][...] = rng.integers(0, 256, frames[k].shape, np.uint8)


# ---- 1. one stream: every insert equals the batch call on (kept images, new images) ----
MODES = ["fast", "harris", "no_points", "no_lines", "rectifier"]


@pytest.mark.parametrize("mode", MODES)
def test_one_stream_equals_batch(mode):
    rect_rig = mode == "rectifier"
    W, H = (752, 480) if rect_rig else (1241, 376)
    th = [20, 0, 12, 35, 20, 5, 0, 50, 20]
    fr = images_only(moving_views(9, W, H, 611, 200, fast_th=th))
    mc, sc, tc, oc = configs(1200, 4, T.ORB_HARRIS_SCORE if mode == "harris" else T.ORB_FAST_SCORE)
    lc = T.default_lsd_config()
    if mode == "no_points":
        tc.has_points = 0
    if mode == "no_lines":
        tc.has_lines = 0
        lc = None
    e = Engine()
    rect = None
    cam = T.kitti_camera()
    if rect_rig:
        cam, maps = rig("euroc")
        rect = e.rectifier_create(*maps)
    ss = e.stereo_session_create(cam, tc, mc, sc, oc, lc, rect, 1)
    rng = np.random.default_rng(5)
    m = Mirror()
    f0 = fresh(frames_slice(fr, 0, 1))
    n0 = ss.initialize([0], f0)
    m.keep([0], frames_slice(fr, 0, 1))
    scribble(f0, rng)
    prev_n = n0[0]
    for k in range(1, 9):
        cur = frames_slice(fr, k, k + 1)
        pri = None
        if k % 2:
            pri = np.zeros(1, T.PRIOR_DTYPE)
            pri["Tfw"] = pri["DT"] = np.eye(4)
            pri["Tfw_cov"] = np.eye(6)
        given = fresh(cur)
        got = ss.insert([0], given, pri)
        scribble(given, rng)
        want = m.batch(e, cam, tc, mc, sc, oc, lc, rect, [0], cur, pri)
        assert_same(got, want)
        np.testing.assert_array_equal(got[1][0, :2], prev_n)   # the kept frame's counts are its own
        prev_n = got[1][0, 2:]
        m.keep([0], cur)
    if mode == "no_points":
        assert (got[1][:, 0::2] == 0).all()
    if mode == "no_lines":
        assert (got[1][:, 1::2] == 0).all()
    else:
        assert got[1][0, 1] > 0, got[1]
    ms = e.track_stereo_images_stage_times()
    assert ms[3] > 0 and ms[4] > 0, ms
    e.close()


# ---- 2. many streams, uneven arrival; 3. the caller's buffers are not read again ----
def stream_frames(S, NF, seed, W=320, H=240):
    """Per stream NF frames of its own moving scene (different seeds); a few flat frames (no lines, no points)."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(S):
        d = images_only(moving_views(NF, W, H, seed + 17 * s, 0))
        d["fast_th"] = rng.choice([0, 5, 12, 20, 35], NF).astype(np.int32)
        if s % 7 == 3:
            d["img_l"][1] = 90
            d["img_r"][1] = 90
        if s % 11 == 5:
            d["img_r"][2] = 40
        out.append(d)
    return out


def frames_of(streams, ids, pos):
    return dict(img_l=np.stack([streams[i]["img_l"][pos[i]] for i in ids]),
                img_r=np.stack([streams[i]["img_r"][pos[i]] for i in ids]),
                fast_th=np.int32([streams[i]["fast_th"][pos[i]] for i in ids]))


@pytest.mark.parametrize("size", ["37", "sms+5"])
def test_many_streams_uneven_arrival(size):
    S = 37 if size == "37" else sm_count() + 5
    NF = 8
    sms = sm_count()
    st = stream_frames(S, NF, 4200 + S)
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e = Engine()
    ss = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)
    rng = np.random.default_rng(S)
    m = Mirror()
    pos = {i: 0 for i in range(S)}
    order = rng.permutation(S)
    first, rest = order[:S // 3], order[S // 3:]
    for ids in (first, rest):   # two initialize calls over disjoint subsets
        fr = frames_of(st, ids, pos)
        ss.initialize(ids, fresh(fr))
        m.keep(ids, fr)
    idle = int(order[0])
    sizes = [S, 5, S // 2, S, 9, S - 2]
    seen_images, seen_solvers = set(), set()
    for rnd, n in enumerate(sizes):
        pool = [i for i in range(S) if not (i == idle and rnd < 3) and pos[i] + 1 < NF]
        ids = np.int32(rng.permutation(pool)[:n])
        if rnd == 2:   # one stream starts over while the others continue
            again = np.int32([ids[-1]])
            ids = ids[:-1]
            pos[int(again[0])] += 1
            fr = frames_of(st, again, pos)
            ss.initialize(again, fresh(fr))
            m.keep(again, fr)
        for i in ids:
            pos[int(i)] += 1
        fr = frames_of(st, ids, pos)
        pri = None
        if rnd % 2:
            pri = np.zeros(len(ids), T.PRIOR_DTYPE)
            pri["Tfw"] = pri["DT"] = np.eye(4)
            pri["Tfw_cov"] = np.eye(6)
        given = fresh(fr)
        got = ss.insert(ids, given, pri)
        scribble(given, rng)
        want = m.batch(e, CAM_SMALL, tc, mc, sc, oc, lc, None, ids, fr, pri)
        assert_same(got, want)
        m.keep(ids, fr)
        seen_images.add(2 * len(ids) < sms)
        seen_solvers.add(len(ids) > sms)
    if size != "37":   # S = 37 has fewer images than SMs in every call; SMs + 5 streams reach both sides of both rules
        assert seen_images == {True, False}, "both sides of the LSD-first rule"
        assert seen_solvers == {True, False}, "both sides of the K2 / streamed policy"
    assert ss.device_bytes > 0
    e.close()


# ---- 4. errors ----
def _raw(e, ss, track, ids, frames, priors=None):
    ids = np.ascontiguousarray(ids, np.int32)
    fs, keep = T.stereo_images_as_c(frames)
    res = np.zeros(max(len(ids), 1), T.POSE_RESULT_DTYPE)
    ns = np.zeros((max(len(ids), 1), 4), np.int32)
    ip = ids.ctypes.data_as(T.c_int32_p)
    if track:
        rc = e.lib.plstvo_stereo_session_insert(e.ctx, ss.handle, len(ids), ip, C.byref(fs), None, res.ctypes.data,
                                                ns.ctypes.data_as(T.c_int32_p))
    else:
        rc = e.lib.plstvo_stereo_session_initialize(e.ctx, ss.handle, len(ids), ip, C.byref(fs), ns.ctypes.data_as(T.c_int32_p))
    return rc, (e.lib.plstvo_last_error(e.ctx) or b"").decode()


def test_errors_leave_the_session_unchanged():
    S = 6
    st = stream_frames(S, 20, 9900)
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e, other = Engine(), Engine()
    ss = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)
    m = Mirror()
    pos = {i: 0 for i in range(S)}
    ids0 = np.int32([0, 1, 2, 3])
    fr = frames_of(st, ids0, pos)
    ss.initialize(ids0, fr)
    m.keep(ids0, fr)
    step = {"k": 0}

    def check(got, rc, text):
        assert got[0] == rc and text in got[1], (got, rc, text)
        ids = np.int32([3, 1, 0]) if step["k"] % 2 else np.int32([2, 0])
        step["k"] += 1
        for i in ids:
            pos[int(i)] += 1
        f = frames_of(st, ids, pos)
        assert_same(ss.insert(ids, f), m.batch(e, CAM_SMALL, tc, mc, sc, oc, lc, None, ids, f))
        m.keep(ids, f)

    nxt = lambda ids: frames_of(st, ids, {i: pos[i] + 1 for i in range(S)})   # noqa: E731
    check(_raw(e, ss, True, [1, 6], nxt([1, 0])), -1, "stream id outside [0, n_streams)")
    check(_raw(e, ss, True, [-1], nxt([1])), -1, "stream id outside [0, n_streams)")
    check(_raw(e, ss, True, [1, 1], nxt([1, 1])), -1, "duplicate stream id")
    check(_raw(e, ss, False, [4, 4], nxt([4, 4])), -1, "duplicate stream id")
    check(_raw(e, ss, True, [0, 4], nxt([0, 4])), -1, "insert on a stream with no frame")
    check(_raw(other, ss, True, [0], nxt([0])), -1, "the session belongs to another context")
    check(_raw(e, ss, True, [0, 1], nxt([0])), -5, "frames->B differs from n")
    bad = nxt([0, 1])
    bad["ll_off"] = np.zeros(3, np.int32)
    check(_raw(e, ss, True, [0, 1], bad), -1, "key-line fields must be null")
    wide = dict(img_l=np.zeros((1, 240, 330), np.uint8), img_r=np.zeros((1, 240, 330), np.uint8))
    check(_raw(e, ss, True, [0], wide), -5, "image size differs from the camera's")
    # more than 65535 images in one call (2 n)
    tiny_cam = T.PlCamera(fx=10.0, fy=10.0, cx=4.0, cy=4.0, b=0.2, width=8, height=8)
    tiny = e.stereo_session_create(tiny_cam, tc, mc, sc, oc, lc, None, 32768)
    z = np.zeros((32768, 8, 8), np.uint8)
    got = _raw(e, tiny, False, np.arange(32768), dict(img_l=z, img_r=z))
    tiny.close()
    check(got, -1, "more than 65535 images in one call")
    # creation errors: a rectifier of another context, a bad config
    cam, maps = rig("euroc")
    r_other = other.rectifier_create(*maps)
    with pytest.raises(PlstvoError, match="the rectifier belongs to another context"):
        e.stereo_session_create(cam, tc, mc, sc, oc, lc, r_other, 2)
    with pytest.raises(PlstvoError, match="lsd refine"):
        e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, T.default_lsd_config(refine=1), None, 2)
    with pytest.raises(PlstvoError, match="n_streams must be at least 1"):
        e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, 0)
    check(_raw(e, ss, True, [5], nxt([5])), -1, "insert on a stream with no frame")   # and the session still tracks
    other.close()
    e.close()


# ---- 5. reuse: other calls between inserts, two sessions interleaved, destroy and recreate ----
def test_reuse_beside_other_calls():
    S = 5
    st = stream_frames(S, 8, 7300)
    st2 = stream_frames(3, 8, 7400)
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    ids_seq = [np.int32([0, 1, 2, 3, 4]), np.int32([4, 2]), np.int32([1, 3, 0]), np.int32([2, 4, 1])]

    def run(e, others):
        out = []
        a = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)
        b = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, 3)
        pa, pb = {i: 0 for i in range(S)}, {i: 0 for i in range(3)}
        a.initialize(np.arange(S), frames_of(st, range(S), pa))
        b.initialize([2, 0, 1], frames_of(st2, [2, 0, 1], pb))
        for r, ids in enumerate(ids_seq):
            for i in ids:
                pa[int(i)] += 1
            if others:
                others[r % len(others)](e)
            out.append(a.insert(ids, frames_of(st, ids, pa)))
            bids = np.int32([r % 3])
            pb[r % 3] += 1
            out.append(b.insert(bids, frames_of(st2, bids, pb)))
        a.close()
        b.close()
        return out

    prev, curr, _, cam = synth.make_batch("kitti", 2)
    kv = moving_views(2, 320, 240, 77, 50)
    imgs = np.concatenate([kv["img_l"], kv["img_r"]])
    n0 = int(kv["ll_off"][1])   # image 0's key lines
    others = [
        lambda e: e.track_batch(cam, T.kitti_config(), prev, curr),
        lambda e: e.track_stereo_images_lsd_batch(CAM_SMALL, tc, mc, sc, oc, lc, images_only(frames_slice(kv, 0, 1)),
                                                  images_only(frames_slice(kv, 1, 2))),
        lambda e: e.orb_detect_and_compute_batch(T.default_orb_detect_config(), imgs),
        lambda e: e.lsd_detect_batch(lc, imgs),
        lambda e: e.lbd_compute_batch(imgs, np.int32([0, n0, n0, n0, n0]), kv["seg_l"][:n0], kv["angle_l"][:n0],
                                      kv["npix_l"][:n0]),
    ]
    e0 = Engine()
    want = run(e0, [])
    e0.close()
    e = Engine()
    same(run(e, others), want)
    same(run(e, others[::-1]), want)   # destroyed and recreated on the same context: a fresh result
    # the pure session results equal the batch call, too
    m = Mirror()
    ss = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)
    pa = {i: 0 for i in range(S)}
    ss.initialize(np.arange(S), frames_of(st, range(S), pa))
    m.keep(np.arange(S), frames_of(st, range(S), pa))
    ids = ids_seq[1]
    for i in ids:
        pa[int(i)] += 1
    f = frames_of(st, ids, pa)
    assert_same(ss.insert(ids, f), m.batch(e, CAM_SMALL, tc, mc, sc, oc, lc, None, ids, f))
    e.close()


# ---- 6. StereoStreamsHandler (examples/streams_cpp.cpp) against a Python loop of the handler rules ----
def test_streams_example_equals_python_loop(tmp_path):
    W, H, S = 640, 376, 4
    NF = 7
    scenes = [images_only(moving_views(NF, W, H, 900 + 31 * s, 0)) for s in range(S)]
    scenes[3]["img_l"][3] = 90   # stream 3's fourth frame: flat, the pair fails
    scenes[3]["img_r"][3] = 90
    rounds = [[2, 0, 1, 3], [0, 1], [1, 3, 0, 2], [3, 2], [3, 0], [2, 1, 3], [0, 3, 2, 1], [3, 2, 0], [1, 0, 3, 2],
              [2, 3, 1], [1], [0, 1]]
    pos = {s: 0 for s in range(S)}
    path = tmp_path / "streams.bin"
    events = []
    with open(path, "wb") as f:
        f.write(struct.pack("<iiii", W, H, S, len(rounds)))
        for rnd in rounds:
            rnd = [s for s in rnd if pos[s] < NF]
            f.write(struct.pack("<i", len(rnd)))
            for s in rnd:
                f.write(struct.pack("<i", s))
                f.write(np.ascontiguousarray(scenes[s]["img_l"][pos[s]]).tobytes())
                f.write(np.ascontiguousarray(scenes[s]["img_r"][pos[s]]).tobytes())
                events.append((s, pos[s]))
                pos[s] += 1
    from test_stereo_session_host import build_streams_example
    out = subprocess.run([build_streams_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout
    rows = [line.split() for line in out.strip().splitlines()]
    # the loop: one handler per stream, B = 1 calls of the _lsd_ batch call on (previous images, new images)
    mc, sc, tc, oc = configs(1200, 4)
    oc.fast_threshold = 0
    lc, hc, cam = T.default_lsd_config(), HandlerConfig(), T.kitti_camera()
    cam = T.PlCamera(fx=cam.fx, fy=cam.fy, cx=cam.cx, cy=cam.cy, b=cam.b, width=W, height=H)
    e = Engine()
    state, th, prev_th, kft = {}, {}, {}, {}
    r = 0
    ths = {s: [] for s in range(S)}
    fails = 0
    for s, k in events:
        if k == 0:
            th[s] = prev_th[s] = hc.orb_fast_th
            state[s] = dict(Tfw=np.eye(4), Tfw_cov=np.eye(6), DT=np.eye(4), DT_cov=np.zeros((6, 6)), err_norm=-1.0)
            kft[s] = KeyframeTest()
            continue
        pri = np.zeros(1, T.PRIOR_DTYPE)
        for key, v in state[s].items():
            pri[key][0] = v
        sc_ = scenes[s]
        prev = dict(img_l=sc_["img_l"][k - 1:k], img_r=sc_["img_r"][k - 1:k], fast_th=[prev_th[s]])
        curr = dict(img_l=sc_["img_l"][k:k + 1], img_r=sc_["img_r"][k:k + 1], fast_th=[th[s]])
        res, ns = e.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, prev, curr, pri)
        x, row = res[0], rows[r]
        r += 1
        assert row[:6] == ["stream", str(s), "frame", str(k), "th", str(th[s])], (row[:6], s, k, th[s])
        assert [int(v) for v in row[7:11]] == list(ns[0]), (row[7:11], ns[0])
        assert int(row[12]) == x["good"]
        fails += int(x["good"]) == 0
        np.testing.assert_array_equal(np.float64(row[14:30]).reshape(4, 4), x["DT"])
        np.testing.assert_array_equal(np.float64(row[31:47]).reshape(4, 4), x["Tfw"])
        kf = kft[s].needNewKF(hc, x["Tfw"], x["DT"], x["DT_cov"])
        assert int(row[48]) == int(kf), (s, k, row[48], kf)
        ths[s].append(th[s])
        Tfw, Tfw_cov = (np.eye(4), np.eye(6)) if kf else (x["Tfw"], x["Tfw_cov"])
        if kf:
            kft[s].T_prevKF, kft[s].cov_prevKF_currF = np.eye(4), np.zeros((6, 6))
            kft[s].prev_f_iskf, kft[s].N_prevKF_currF = True, 0
        state[s] = dict(Tfw=Tfw, Tfw_cov=Tfw_cov, DT=x["DT"], DT_cov=x["DT_cov"], err_norm=float(x["err_norm"]))
        prev_th[s], th[s] = th[s], update_fast_threshold(hc, th[s], x["DT"], float(x["err_norm"]), int(x["n_inliers_pt"]))
    assert r == len(rows)
    assert fails >= 1, "a stream with a failed pair"
    assert any(len(set(v)) > 1 for v in ths.values()), ths   # a stream whose threshold moved
    e.close()
