"""plstvo_stereo_session_run on the GPU: T steps of the handler's loop in one call.  Every check compares a run with the
per-frame loop of plstvo_stereo_session_insert on a twin session, driven by handler.update_fast_threshold and by priors
built from the previous results as plstvo.hpp's priorOf builds them: results, n_stereo and the threshold rows byte for byte,
then read() after the last step and a follow-up insert on both sessions.  Sessions plain, with a camera per stream and
grey rigs (one NULL entry), and BGR rectifiers with and without maps; S = 1, 37 and SMs + 5 streams, T = 1, 2 and 9; the
config switches; a subset run; a split run; T = 0; run / insert / run on one session; the branches of the rule; errors."""
import ctypes as C
import subprocess
from collections import Counter

import numpy as np
import pytest

from test_gpu_track_images import CAM_SMALL, configs, sm_count
from test_gpu_stereo_session import stream_frames
from test_gpu_session_cams import colour, perturbed_maps, three_cams
from test_gpu_rectify import rig
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError
from stvo_pl_b200.handler import HandlerConfig, update_fast_threshold

pytestmark = pytest.mark.gpu


def scenes(S, NF, seed, W=320, H=240):
    """Per stream NF frames: dense, medium and sparse texture (contrast cut towards mid grey), a flat frame in some streams
    (no features: the solve fails and DT stays I)."""
    st = stream_frames(S, NF, seed, W, H)
    for s, d in enumerate(st):
        cut = (1, 2, 6)[s % 3]
        for k in ("img_l", "img_r"):
            d[k] = ((d[k].astype(np.int16) - 128) // cut + 128).astype(np.uint8)
        if s % 5 == 2 and NF > 2:
            d["img_l"][2] = 70
            d["img_r"][2] = 70
    return st


def step_major(st, ids, t0, T_):
    """Frames t0 .. t0 + T_ - 1 of streams ids, step-major (no fast_th)."""
    return dict(img_l=np.concatenate([np.stack([st[i]["img_l"][t] for i in ids]) for t in range(t0, t0 + T_)]),
                img_r=np.concatenate([np.stack([st[i]["img_r"][t] for i in ids]) for t in range(t0, t0 + T_)]))


def priors_of(res):
    """priorOf(publishPose(r)) per row."""
    p = np.zeros(len(res), T.PRIOR_DTYPE)
    for k in ("Tfw", "Tfw_cov", "DT", "DT_cov", "err_norm"):
        p[k] = res[k]
    return p


BRANCHES = Counter()


def rule(h, th, r):
    """update_fast_threshold, counting the branch it took and the clamps."""
    want = update_fast_threshold(h, th, r["DT"], float(r["err_norm"]), int(r["n_inliers_pt"]))
    n, inc, feat = int(r["n_inliers_pt"]), h.fast_inc_th, h.fast_feat_th
    if not h.adaptative_fast:
        b, dec = "off", None
    elif np.array_equal(r["DT"], np.eye(4)):
        b, dec = "identity", 2 * inc
    elif float(r["err_norm"]) > float(np.float32(h.fast_err_th)):
        b, dec = "err_norm", 2 * inc
    elif n < feat:
        b, dec = "lt_feat", 2 * inc
    elif n < 2 * feat:
        b, dec = "lt_2feat", inc
    elif n > 3 * feat:
        b, dec = "gt_3feat", None
        if th + inc > h.fast_max_th:
            BRANCHES["clamp_max"] += 1
    else:
        b, dec = "keep", None
    if dec is not None and th - dec < h.fast_min_th:
        BRANCHES["clamp_min"] += 1
    BRANCHES[b] += 1
    return want


def loop(ss, h, oc, ids, frames, T_, th0=None, priors=None):
    """The per-frame insert loop the run must equal: (results [T, n], thresholds [T + 1, n], n_stereo [T, n, 4])."""
    n = len(ids)
    th = np.full(n, oc.fast_threshold, np.int32) if th0 is None else np.where(np.int32(th0) == 0, oc.fast_threshold, th0)
    th = np.int32(th)
    rows, res_all, ns_all, pri = [th.copy()], [], [], priors
    for t in range(T_):
        fr = dict(img_l=frames["img_l"][t * n:(t + 1) * n], img_r=frames["img_r"][t * n:(t + 1) * n], fast_th=th.copy())
        res, ns = ss.insert(ids, fr, pri)
        th = np.int32([rule(h, int(th[k]), res[k]) for k in range(n)])
        rows.append(th.copy())
        res_all.append(res.copy())
        ns_all.append(ns.copy())
        pri = priors_of(res)
    if T_ == 0:
        return np.zeros((0, n), T.POSE_RESULT_DTYPE), np.stack(rows), np.zeros((0, n, 4), np.int32)
    return np.stack(res_all), np.stack(rows), np.stack(ns_all)


def same_read(a, b):
    for x, y in zip(a.read(), b.read()):
        if isinstance(x, dict):
            assert x.keys() == y.keys()
            for k in x:
                assert x[k].tobytes() == y[k].tobytes(), k
        else:
            assert (x is None and y is None) or x.tobytes() == y.tobytes()


def same_run(got, want):
    (r1, t1, n1), (r2, t2, n2) = got, want
    np.testing.assert_array_equal(t1, t2)
    np.testing.assert_array_equal(n1, n2)
    assert r1.tobytes() == r2.tobytes()


def follow_up(A, B, ids, fr, pri):
    """One more insert on both sessions: the kept frames are the same bytes either way."""
    a, b = A.insert(ids, fr, pri), B.insert(ids, fr, pri)
    assert a[0].tobytes() == b[0].tobytes()
    np.testing.assert_array_equal(a[1], b[1])


class Twins:
    """Two identical sessions: A runs, B loops."""

    def __init__(self, e, kind, S):
        self.e = e
        mc, sc, tc, oc = configs(500, 2)
        lc = T.default_lsd_config()
        self.W, self.H, cam, rects, self.bgr = 320, 240, CAM_SMALL, None, False
        cams = None
        if kind == "motion_solver1":
            tc.use_motion_model, tc.solver_mode = 1, 1
        elif kind == "no_points":
            tc.has_points = 0
        elif kind == "no_lines":
            tc.has_lines, lc = 0, None
        elif kind == "cams":
            cams = [three_cams(CAM_SMALL)[s % 3] for s in range(S)]
        elif kind in ("cams_grey_rigs", "bgr_maps", "bgr_nomaps"):
            cam, maps = rig("euroc")
            self.W, self.H = cam.width, cam.height
            if kind == "cams_grey_rigs":
                rs = [e.rectifier_create(*maps), e.rectifier_create(*perturbed_maps(1)), None]
            elif kind == "bgr_maps":
                rs = [e.rectifier_create_color(self.W, self.H, 3, *maps), e.rectifier_create_color(self.W, self.H, 3,
                                                                                               *perturbed_maps(2))]
                self.bgr = True
            else:
                rs = [e.rectifier_create_color(self.W, self.H, 3)]
                self.bgr = True
            rects = [rs[s % len(rs)] for s in range(S)]
            cams = [three_cams(cam)[s % 3] for s in range(S)]
        self.oc = oc
        self.h = HandlerConfig(fast_feat_th=20)
        if kind == "not_adaptive":
            self.h.adaptative_fast = False
        if kind == "tiny_err":
            self.h.fast_err_th = 1e-6
        if kind == "low_max":   # dense frames climb into the upper clamp
            self.h.fast_max_th = 12
        mk = (lambda: e.stereo_session_create(cam, tc, mc, sc, oc, lc, None, S)) if cams is None else \
            (lambda: e.stereo_session_create_cams(cams, tc, mc, sc, oc, lc, rects, S))
        self.A, self.B = mk(), mk()
        for s in (self.A, self.B):
            s.retain(True)

    def frames(self, S, NF, seed):
        st = scenes(S, NF, seed, self.W, self.H)
        if self.bgr:
            st = [colour(d, s) for s, d in enumerate(st)]
        return st

    def init(self, st, ids, t=0):
        fr = dict(img_l=np.stack([st[i]["img_l"][t] for i in ids]), img_r=np.stack([st[i]["img_r"][t] for i in ids]))
        self.A.initialize(ids, fr)
        self.B.initialize(ids, fr)

    def compare(self, ids, frames, T_, th0=None, priors=None):
        got = self.A.run(self.h, ids, T_, frames, th0, priors)
        want = loop(self.B, self.h, self.oc, ids, frames, T_, th0, priors)
        same_run(got, want)
        if T_ > 0:
            same_read(self.A, self.B)
        return got


def th0_for(n, seed):
    """Starting thresholds at and near both clamps and 0 (the configured threshold)."""
    return np.random.default_rng(seed).choice([0, 1, 5, 7, 12, 20, 46, 50, 200, 255], n).astype(np.int32)


def check(kind, S, T_, seed):
    e = Engine()
    tw = Twins(e, kind, S)
    st = tw.frames(S, T_ + 2, seed)
    ids = np.int32(np.random.default_rng(seed).permutation(S))
    tw.init(st, ids)
    th0 = th0_for(S, seed)
    pri = priors_of(np.zeros(S, T.POSE_RESULT_DTYPE))
    pri["Tfw"] = pri["DT"] = np.eye(4)
    pri["Tfw_cov"] = np.eye(6)
    res, rows, _ = tw.compare(ids, step_major(st, ids, 1, T_), T_, th0, pri if seed % 2 else None)
    last = dict(img_l=np.stack([st[i]["img_l"][T_ + 1] for i in ids]), img_r=np.stack([st[i]["img_r"][T_ + 1] for i in ids]),
                fast_th=rows[-1])
    follow_up(tw.A, tw.B, ids, last, priors_of(res[-1]))
    ms = e.track_stereo_images_stage_times()
    assert (ms >= 0).all() and ms[4] > 0, ms
    e.close()


@pytest.mark.parametrize("S,T_", [(1, 9), (37, 2), ("sms+5", 1), ("sms+5", 9)])
def test_sizes(S, T_):
    check("plain", sm_count() + 5 if S == "sms+5" else S, T_, 100 + T_)


@pytest.mark.parametrize("kind", ["cams", "motion_solver1", "no_points", "no_lines", "not_adaptive", "tiny_err"])
def test_configs(kind):
    check(kind, 11, 4, 300 + len(kind))


@pytest.mark.parametrize("kind", ["cams_grey_rigs", "bgr_maps", "bgr_nomaps"])
def test_rectifiers(kind):
    check(kind, 5, 3, 400 + len(kind))


def test_every_branch_fires():
    """The rule's branches over a run of textured, sparse and flat frames from thresholds at both clamps, a tiny fast_err_th
    and a low fast_max_th: each fires, and the run agrees with the loop throughout."""
    BRANCHES.clear()
    check("plain", 37, 9, 71)
    check("tiny_err", 9, 3, 72)
    check("low_max", 11, 4, 73)
    fired = set(BRANCHES)
    want = {"identity", "err_norm", "lt_feat", "lt_2feat", "gt_3feat", "keep", "clamp_min", "clamp_max"}
    assert want <= fired, (want - fired, dict(BRANCHES))


def test_subset_split_empty_and_interleaving():
    e = Engine()
    S = 13
    tw = Twins(e, "plain", S)
    st = tw.frames(S, 16, 900)
    all_ids = np.int32(range(S))
    tw.init(st, all_ids)
    # a subset runs 7 steps on A, one call of 7 against the loop; the others keep their frames
    sub = np.int32([3, 0, 9, 5, 12])
    res, rows, _ = tw.compare(sub, step_major(st, sub, 1, 7), 7)
    # T = 0: nothing happens, read() still gives the last step
    r0, t0, n0 = tw.A.run(tw.h, sub, 0, dict(img_l=np.zeros((0, tw.H, tw.W), np.uint8),
                                            img_r=np.zeros((0, tw.H, tw.W), np.uint8)))
    assert r0.shape == (0, len(sub)) and t0.shape == (1, len(sub)) and n0.shape == (0, len(sub), 4)
    np.testing.assert_array_equal(t0[0], tw.oc.fast_threshold)   # row T = row 0: no fast_th0, the configured threshold
    same_read(tw.A, tw.B)
    # an insert on every stream: the untouched ones are tracked against their initial frames on both
    pos = {i: (8 if i in sub else 1) for i in range(S)}
    fr = dict(img_l=np.stack([st[i]["img_l"][pos[i]] for i in all_ids]), img_r=np.stack([st[i]["img_r"][pos[i]] for i in all_ids]))
    follow_up(tw.A, tw.B, all_ids, fr, None)
    # run, insert, run again on one session: the second run starts at the thresholds and priors the caller gives
    res2, rows2, _ = tw.compare(all_ids, step_major(st, all_ids, 9, 2), 2, np.int32([20] * S), None)
    fr = dict(img_l=np.stack([st[i]["img_l"][11] for i in all_ids]), img_r=np.stack([st[i]["img_r"][11] for i in all_ids]),
              fast_th=rows2[-1])
    follow_up(tw.A, tw.B, all_ids, fr, priors_of(res2[-1]))
    tw.compare(all_ids, step_major(st, all_ids, 12, 2), 2, rows2[-1], None)
    e.close()
    # split: run(7) equals run(3) then run(4) from row 3 and the last priors
    e = Engine()
    tw = Twins(e, "plain", 6)
    st = tw.frames(6, 8, 901)
    ids = np.int32([5, 1, 4, 0, 2, 3])
    tw.init(st, ids)
    th0 = th0_for(6, 9)
    whole = tw.B.run(tw.h, ids, 7, step_major(st, ids, 1, 7), th0)
    a = tw.A.run(tw.h, ids, 3, step_major(st, ids, 1, 3), th0)
    b = tw.A.run(tw.h, ids, 4, step_major(st, ids, 4, 4), a[1][-1], priors_of(a[0][-1]))
    assert np.concatenate([a[0], b[0]]).tobytes() == whole[0].tobytes()
    np.testing.assert_array_equal(np.concatenate([a[1][:-1], b[1]]), whole[1])
    np.testing.assert_array_equal(np.concatenate([a[2], b[2]]), whole[2])
    same_read(tw.A, tw.B)
    e.close()


def _raw_run(e, ss, h, ids, T_, frames, th0=None, results=True, null_ids=False):
    ids = np.ascontiguousarray(ids, np.int32)
    fs, keep = T.stereo_images_as_c(frames)
    n = len(ids)
    res = np.zeros(max(T_ * n, 1), T.POSE_RESULT_DTYPE)
    th = None if th0 is None else np.ascontiguousarray(th0, np.int32)
    rc = e.lib.plstvo_stereo_session_run(e.ctx, ss.handle, None if h is None else C.byref(h), n,
                                         None if null_ids else ids.ctypes.data_as(T.c_int32_p), T_, C.byref(fs),
                                         None if th is None else th.ctypes.data_as(T.c_int32_p), None,
                                         res.ctypes.data if results else None, None, None)
    del keep
    return rc, (e.lib.plstvo_last_error(e.ctx) or b"").decode()


class Untouched:
    """A session that meets the errors and its twin that does not: after every error the first reads nothing and gives the
    twin's next insert, byte for byte."""

    def __init__(self, A, B, ids, st):
        self.A, self.B, self.ids, self.st, self.k = A, B, ids, st, 0

    def check(self):
        with pytest.raises(PlstvoError):
            self.A.read()
        self.k += 1
        t = 1 + self.k % 3
        fr = dict(img_l=np.stack([self.st[i]["img_l"][t] for i in self.ids]),
                  img_r=np.stack([self.st[i]["img_r"][t] for i in self.ids]), fast_th=np.int32([20] * len(self.ids)))
        follow_up(self.A, self.B, self.ids, fr, None)


def test_errors_leave_the_session_usable():
    e = Engine()
    S = 3
    tw = Twins(e, "plain", S)
    st = tw.frames(S, 4, 77)
    ids = np.int32([0, 1, 2])
    tw.init(st, ids)
    u = Untouched(tw.A, tw.B, ids, st)
    fr = step_major(st, ids, 1, 2)
    good = e.handler_config()
    assert (good.fast_min_th, good.fast_max_th, good.fast_inc_th, good.fast_feat_th, good.fast_err_th) == (5, 50, 5, 50, 0.5)
    k = e.handler_config(kitti=True)
    assert (k.adaptative_fast, k.fast_min_th, k.fast_max_th) == (1, 7, 30)

    def bad_h(**kw):
        h = e.handler_config()
        for f, v in kw.items():
            setattr(h, f, v)
        return h

    with_th = dict(fr, fast_th=np.zeros(6, np.int32))
    with_lines = dict(fr, ll_off=np.zeros(7, np.int32))
    empty = dict(img_l=np.zeros((0, 240, 320), np.uint8), img_r=np.zeros((0, 240, 320), np.uint8))
    many = dict(img_l=np.zeros((32769, 1, 1), np.uint8), img_r=np.zeros((32769, 1, 1), np.uint8))
    out_of_range = "handler config out of range"
    cases = [
        (dict(h=None), -1, "null handler config"),
        (dict(h=bad_h(fast_min_th=0)), -1, out_of_range),
        (dict(h=bad_h(fast_min_th=60)), -1, out_of_range),
        (dict(h=bad_h(fast_max_th=256)), -1, out_of_range),
        (dict(h=bad_h(fast_inc_th=-1)), -1, out_of_range),
        (dict(h=bad_h(fast_feat_th=-1)), -1, out_of_range),
        (dict(h=bad_h(fast_err_th=float("nan"))), -1, out_of_range),
        (dict(h=bad_h(fast_err_th=float("inf"))), -1, out_of_range),
        (dict(h=bad_h(fast_err_th=float("-inf"))), -1, out_of_range),
        (dict(frames=with_th), -1, "must be null"),
        (dict(frames=with_lines), -1, "must be null"),
        (dict(T_=-1, frames=empty), -1, "negative T"),
        (dict(T_=3), -5, "frames->B differs from T * n"),
        (dict(th0=np.int32([0, 256, 5])), -1, "fast_th0 outside [0, 255]"),
        (dict(th0=np.int32([0, -1, 5])), -1, "fast_th0 outside [0, 255]"),
        (dict(null_ids=True), -1, "null ids or results"),
        (dict(results=False), -1, "null ids or results"),
        (dict(T_=10923, frames=many), -1, "more than 65535 images"),   # 2 n T > 65535, checked before anything is read
        (dict(ids=np.int32([0, 1, 3])), -1, "stream id outside"),
        (dict(ids=np.int32([0, 1, 1])), -1, "duplicate stream id"),
    ]
    for kw, code, msg in cases:
        a = dict(h=good, ids=ids, T_=2, frames=fr)
        a.update(kw)
        rc, err = _raw_run(e, tw.A, a.pop("h"), a.pop("ids"), a.pop("T_"), a.pop("frames"), **a)
        assert rc == code and msg in err, (msg, rc, err)
        u.check()
    # the Python binding checks the per-stream arrays' lengths before the call
    with pytest.raises(ValueError):
        tw.A.run(good, ids, 2, fr, fast_th0=np.int32([20, 20]))
    with pytest.raises(ValueError):
        tw.A.run(good, ids, 2, fr, priors=np.zeros(4, T.PRIOR_DTYPE))
    # checks that need a session of their own, each against its twin
    init = dict(img_l=fr["img_l"][:3], img_r=fr["img_r"][:3])
    mc, sc, tc, oc = configs(500, 2)
    fresh = [e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, T.default_lsd_config(), None, S) for _ in range(2)]
    rc, err = _raw_run(e, fresh[0], good, ids, 2, fr)
    assert rc == -1 and "initialize it first" in err, err
    for ss in fresh:
        ss.initialize(ids, init)
    Untouched(fresh[0], fresh[1], ids, st).check()
    mc, sc, tc, oc = configs(70000, 2)   # n_features beyond the per-frame limit
    huge = [e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, T.default_lsd_config(), None, S) for _ in range(2)]
    for ss in huge:
        ss.initialize(ids, init)
    rc, err = _raw_run(e, huge[0], good, ids, 2, fr)
    assert rc == -1 and "n_features exceeds" in err, err
    Untouched(huge[0], huge[1], ids, st).check()
    mc, sc, tc, oc = configs(500, 2)   # an ORB fast_threshold outside [0, 255] where fast_th0 leaves it
    oc.fast_threshold = 300
    hot = [e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, T.default_lsd_config(), None, S) for _ in range(2)]
    for ss in hot:
        ss.initialize(ids, dict(init, fast_th=np.int32([20] * S)))
    rc, err = _raw_run(e, hot[0], good, ids, 2, fr, th0=np.int32([0, 20, 20]))
    assert rc == -1 and "ocfg->fast_threshold outside" in err, err
    Untouched(hot[0], hot[1], ids, st).check()
    # and after them all, a run still equals the loop
    tw.compare(ids, step_major(st, ids, 2, 2), 2)
    e.close()


def bars(W, H):
    """Dark 3 x 24 bars on a light ground every 8 x 32 pixels: at scale 1 with no length floor LSD finds both long edges of
    every bar, 73 728 key lines on 4096 x 2304 (the LSD restatement, oracle/lsd.py, gives that count)."""
    img = np.full((H, W), 200, np.uint8)
    for y in range(2, H - 26, 32):
        for x in range(2, W - 5, 8):
            img[y:y + 24, x:x + 3] = 30
    return img


def test_key_line_limit_before_step_0():
    """More than 65535 key lines in one image of step 1: PLSTVO_E_TOO_LARGE before step 0 runs, the session untouched."""
    W, H = 4096, 2304
    cam = T.PlCamera(fx=2000.0, fy=2000.0, cx=W / 2, cy=H / 2, b=0.2, width=W, height=H)
    mc, sc, tc, oc = configs(500, 2)
    lc = T.default_lsd_config(0, scale=1.0, min_line_length=0.0)
    e = Engine()
    A, B = (e.stereo_session_create(cam, tc, mc, sc, oc, lc, None, 1) for _ in range(2))
    for ss in (A, B):
        ss.retain(True)
    flat = np.full((1, H, W), 120, np.uint8)
    for ss in (A, B):
        ss.initialize([0], dict(img_l=flat, img_r=flat))
    fr = dict(img_l=np.stack([flat[0], bars(W, H)]), img_r=np.stack([flat[0], flat[0]]))
    h = e.handler_config()
    with pytest.raises(PlstvoError) as ex:
        A.run(h, [0], 2, fr)
    assert ex.value.code == -2 and "65535 key lines" in str(ex.value), ex.value
    # step 0 (a flat frame) did not run: the next insert equals the twin's
    nxt = dict(img_l=flat, img_r=flat, fast_th=np.int32([20]))
    follow_up(A, B, np.int32([0]), nxt, None)
    e.close()


def test_run_example(tmp_path):
    """examples/run_cpp.cpp: StereoStreamsHandler::insertStereoSequences against the per-frame loop, byte for byte."""
    from test_session_run_host import build_run_example
    r = subprocess.run([build_run_example(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "run equals the per-frame loop" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
