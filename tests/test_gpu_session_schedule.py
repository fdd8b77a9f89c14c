"""plstvo_stereo_session_run_schedule on the GPU: runs over uneven streams (steps where a stream has no frame, streams that
start or restart inside the call) against the chain it must equal, driven on a twin session with handler.py's rules: per
step one _initialize on the step's code-2 entries, then one _insert on its code-1 entries, each stream's threshold, prior
and key-frame state carried by handler.ScheduleStreams.  Results, n_stereo and the threshold rows byte for byte, key-frame
decisions exactly and their diagnostics and states to the last ulps (the host test is numpy's), then _read, _read_keyframes
and a following insert on both sessions.  A dense schedule equals _run and _run_keyframes byte for byte.  Seeded drop
patterns on 1, 8 and SMs + 5 streams; a stream absent for the whole call, one starting inside it, one re-initialised on a
step where others insert, empty steps and T = 0; plain, camera-per-stream, colour and FLD sessions; retention on and off,
with and without the test; a second call continuing the first; and every error, each leaving the session usable."""
import numpy as np
import pytest

from test_gpu_session_fld import line_fields
from test_gpu_session_run import Twins, same_read
from test_gpu_track_images import sm_count
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError
from stvo_pl_b200.handler import KeyframeTest, ScheduleStreams, schedule_frames, schedule_groups, take_frames

E_INVALID, E_SIZE = -1, -5   # PLSTVO_E_INVALID, PLSTVO_E_SIZE

pytestmark = pytest.mark.gpu


def frame_source(tw, st, ids, fld_lc=None):
    """frame_of(t, k) for schedule_frames: stream ids[k]'s frame t (+1: frame 0 initialised the streams), with its key lines
    on the FLD branch"""
    def frame_of(t, k):
        i = ids[k]
        d = dict(img_l=st[i]["img_l"][t + 1][None], img_r=st[i]["img_r"][t + 1][None])
        if fld_lc is not None:
            d.update(line_fields(tw.e, fld_lc, d["img_l"], d["img_r"]))
        return d
    return frame_of


def chain(tw, ss, ids, sched, frames, th0=None, priors=None, kcfg=None, kf_state=None):
    """The chain the scheduled run must equal, on session ss: (results, kf or None, fast_th, n_stereo, kf_state or None,
    the records each insert retained by step)"""
    n, T_ = len(ids), len(sched)
    oc, h = tw.oc, tw.h
    th = np.int32([oc.fast_threshold] * n) if th0 is None else np.where(np.int32(th0) == 0, oc.fast_threshold, th0)
    m = ScheduleStreams(h, th, priors, kf_state if kcfg is not None else None)
    results = np.zeros((T_, n), T.POSE_RESULT_DTYPE)
    kf = np.zeros((T_, n), T.KEYFRAME_RESULT_DTYPE) if kcfg is not None else None
    fast_th = np.zeros((T_ + 1, n), np.int32)
    n_stereo = np.zeros((T_, n, 4), np.int32)
    reads = {}
    by_step = {g[0]: g for g in schedule_groups(sched)}
    for t in range(T_):
        fast_th[t] = m.th
        if t not in by_step:
            continue
        _, init, ins, bi, bn = by_step[t]
        if init:
            fr = take_frames(frames, bi)
            given = fr.get("fast_th")
            thr = np.int32([g if g else oc.fast_threshold for g in (given if given is not None else [0] * len(init))])
            fr["fast_th"] = thr
            ns = ss.initialize(ids[init], fr)
            n_stereo[t, init, 2:] = ns
            for k, v in zip(init, thr):
                m.initialize(k, int(v))
                fast_th[t, k] = v
        if ins:
            fr = take_frames(frames, bn)
            fr["fast_th"] = m.th[ins].copy()
            res, ns = ss.insert(ids[ins], fr, m.prior[ins].copy())
            results[t, ins] = res
            n_stereo[t, ins] = ns
            if tw_retains(ss):
                reads[t] = (ss.read(), ns.copy())
            for k, r in zip(ins, res):
                state, new = None, False
                if kcfg is not None:
                    test = KeyframeTest.from_state(m.kf[k])
                    new = test.needNewKF(tw.h, r["Tfw"], r["DT"], r["DT_cov"])
                    kf[t, k] = (int(new), test.N_prevKF_currF, test.entropy_curr, test.entropy_ratio, test.t, test.r)
                    if new:
                        test.currFrameIsKF(_Frame())
                    state = test.to_state()[0]
                m.inserted(k, r, state, new)
    fast_th[T_] = m.th
    return results, kf, fast_th, n_stereo, m.kf, reads


class _Frame:
    Tfw = Tfw_cov = None


def tw_retains(ss):
    return getattr(ss, "_retains", True)


def same(got, want, kcfg=None, kf_state=None):
    if kcfg is None:
        r1, t1, n1 = got
    else:
        r1, k1, t1, n1 = got
    r2, k2, t2, n2, s2, _ = want
    np.testing.assert_array_equal(t1, t2)
    np.testing.assert_array_equal(n1, n2)
    assert r1.tobytes() == r2.tobytes()
    if kcfg is not None:
        np.testing.assert_array_equal(k1["new_kf"], k2["new_kf"])
        np.testing.assert_array_equal(k1["N_prevKF_currF"], k2["N_prevKF_currF"])
        for f in ("entropy_curr", "entropy_ratio", "t", "r"):
            np.testing.assert_allclose(k1[f], k2[f], rtol=1e-9, atol=1e-9)
        np.testing.assert_array_equal(kf_state["prev_f_iskf"], s2["prev_f_iskf"])
        np.testing.assert_array_equal(kf_state["N_prevKF_currF"], s2["N_prevKF_currF"])
        for f in ("entropy_first_prevKF", "T_prevKF", "cov_prevKF_currF"):
            np.testing.assert_allclose(kf_state[f], s2[f], rtol=1e-9, atol=1e-9)


def same_keyframes(A, want, ids, sched):
    """_read_keyframes of A against the records the chain's inserts retained; returns the number of key frames"""
    rows, pt, ls = A.read_keyframes()
    at_pt = at_ls = 0
    for t, sid, npt, nls in rows:
        (p2, l2, *_), ns = want[5][int(t)]
        ins = [k for k in range(len(ids)) if sched[t, k] == 1]
        j = ins.index(int(np.nonzero(np.asarray(ids) == sid)[0][0]))
        o_pt, o_ls = int(ns[:j, 2].sum()), int(ns[:j, 3].sum())
        assert (npt, nls) == (ns[j, 2], ns[j, 3])
        for key in (x for x in pt if x != "counts"):   # per-frame counts: checked above
            assert pt[key][at_pt:at_pt + npt].tobytes() == p2[key][o_pt:o_pt + npt].tobytes(), key
        for key in (x for x in ls if x != "counts"):
            assert ls[key][at_ls:at_ls + nls].tobytes() == l2[key][o_ls:o_ls + nls].tobytes(), key
        at_pt += npt
        at_ls += nls
    return len(rows)


def make(kind, S, fld=False, retain=True):
    e = Engine()
    tw = Twins(e, "plain" if kind == "fld" else kind, S)
    lc = None
    if kind == "fld":
        lc = T.default_lsd_config()
        for s in (tw.A, tw.B):
            s.use_fld_lines(True)
    for s in (tw.A, tw.B):
        s.retain(retain)
        s._retains = retain
    return tw, lc


def start(tw, S, NF, seed, ids, held, lc=None):
    """Frames of S streams; streams `held` initialised on both sessions with frame 0"""
    st = tw.frames(S, NF, seed)
    if len(held):
        fr = dict(img_l=np.stack([st[i]["img_l"][0] for i in held]), img_r=np.stack([st[i]["img_r"][0] for i in held]))
        if lc is not None:
            fr.update(line_fields(tw.e, lc, fr["img_l"], fr["img_r"]))
        tw.A.initialize(held, fr)
        tw.B.initialize(held, fr)
    return st


def drops(S, T_, rate, seed, reinit=0.08):
    rng = np.random.default_rng(seed)
    sched = np.where(rng.random((T_, S)) < rate, 0, 1).astype(np.uint8)
    sched[rng.random((T_, S)) < reinit] = 2
    return sched


def compare(tw, ids, sched, frames, kcfg=None, th0=None, priors=None, kf_state=None):
    ids = np.int32(ids)
    ks = None if kcfg is None else kf_state.copy()
    got = tw.A.run_schedule(tw.h, ids, sched, frames, th0, priors, kcfg, ks)
    want = chain(tw, tw.B, ids, sched, frames, th0, priors, kcfg, kf_state)
    same(got, want, kcfg, ks)
    if sched.any() and tw_retains(tw.A):
        same_read(tw.A, tw.B)
    return got, want, ks


def follow_up(tw, st, ids, t):
    """one more insert of every stream on both sessions: the kept frames are the same bytes"""
    fr = dict(img_l=np.stack([st[i]["img_l"][t] for i in ids]), img_r=np.stack([st[i]["img_r"][t] for i in ids]))
    a, b = tw.A.insert(ids, fr), tw.B.insert(ids, fr)
    assert a[0].tobytes() == b[0].tobytes()
    np.testing.assert_array_equal(a[1], b[1])


@pytest.mark.parametrize("keyframes", [False, True])
def test_dense_schedule_is_the_run(keyframes):
    S, T_ = 4, 3
    tw, _ = make("plain", S)
    ids = np.int32([2, 0, 3, 1])
    st = start(tw, S, T_ + 2, 5, ids, ids)
    sched = np.ones((T_, S), np.uint8)
    frames = schedule_frames(sched, frame_source(tw, st, ids))
    th0 = np.int32([0, 7, 30, 12])
    if keyframes:
        k = tw.e.keyframe_config()
        s1, s2 = tw.e.initial_keyframe_state(S), tw.e.initial_keyframe_state(S)
        got = tw.A.run_schedule(tw.h, ids, sched, frames, th0, None, k, s1)
        want = tw.B.run_keyframes(tw.h, k, ids, T_, frames, s2, th0)
        for x, y in zip(got, want):
            assert x.tobytes() == y.tobytes()
        assert s1.tobytes() == s2.tobytes()
        r1, r2 = tw.A.read_keyframes(), tw.B.read_keyframes()
        for x, y in zip(r1[1:], r2[1:]):
            for key in x:
                assert x[key].tobytes() == y[key].tobytes()
        np.testing.assert_array_equal(r1[0], r2[0])
    else:
        got = tw.A.run_schedule(tw.h, ids, sched, frames, th0)
        want = tw.B.run(tw.h, ids, T_, frames, th0)
        for x, y in zip(got, want):
            assert x.tobytes() == y.tobytes()
    same_read(tw.A, tw.B)
    follow_up(tw, st, ids, T_ + 1)


@pytest.mark.parametrize("S,T_,rate", [(1, 6, 0.2), (8, 5, 0.05), (8, 5, 0.2), (8, 4, 0.5), ("sm+5", 2, 0.2)])
def test_random_drops(S, T_, rate):
    S = sm_count() + 5 if S == "sm+5" else S
    tw, _ = make("plain", S)
    ids = np.int32(np.random.default_rng(S + T_).permutation(S))
    st = start(tw, S, T_ + 2, 11 + S, ids, ids)
    sched = drops(S, T_, rate, 100 * S + T_)
    frames = schedule_frames(sched, frame_source(tw, st, ids))
    compare(tw, ids, sched, frames)
    follow_up(tw, st, ids, T_ + 1)


@pytest.mark.parametrize("keyframes", [False, True])
@pytest.mark.parametrize("retain", [True, False])
def test_late_absent_reinitialised_and_continued(keyframes, retain):
    """stream 0 absent throughout; stream 1 holds no frame at the start and starts at step 2; stream 2 re-initialised at step
    3 while the others insert; step 1 empty.  Then a second call continues from the returned state."""
    S, T_ = 5, 5
    tw, _ = make("plain", S, retain=retain)
    ids = np.int32([0, 1, 2, 3, 4])
    st = start(tw, S, 2 * T_ + 2, 21, ids, np.int32([0, 2, 3, 4]))
    sched = np.uint8([[0, 0, 1, 1, 1],
                      [0, 0, 0, 0, 0],
                      [0, 2, 1, 0, 1],
                      [0, 1, 2, 1, 1],
                      [0, 1, 1, 1, 0]])
    frames = schedule_frames(sched, frame_source(tw, st, ids))
    frames["fast_th"] = np.where(sched[sched != 0] == 2, 9, 0).astype(np.int32)   # the initialize entries' thresholds
    k = tw.e.keyframe_config() if keyframes else None
    s0 = tw.e.initial_keyframe_state(S) if keyframes else None
    got, want, ks = compare(tw, ids, sched, frames, k, kf_state=s0)
    fast_th = got[-2]
    assert (fast_th[2, 1], fast_th[3, 2]) == (9, 9)
    if keyframes and retain:
        same_keyframes(tw.A, want, ids, sched)
    # the second call: fast_th0 = row T, priors and kf_state from the chain's mirror
    m_pri = ScheduleStreams(tw.h, fast_th[-1])
    res = want[0]
    for t in range(T_):
        for kk in range(S):
            if sched[t, kk] == 2:
                m_pri.initialize(kk, int(fast_th[t, kk]))
            elif sched[t, kk] == 1:
                new = keyframes and bool(got[1][t, kk]["new_kf"])
                m_pri.inserted(kk, res[t, kk], None, new)
    sched2 = np.uint8([[1, 1, 1, 0, 1], [2, 1, 0, 1, 1]])
    frames2 = schedule_frames(sched2, lambda t, kk: frame_source(tw, st, ids)(t + T_, kk))
    compare(tw, ids, sched2, frames2, k, fast_th[-1], m_pri.prior, ks if keyframes else None)
    follow_up(tw, st, ids, 2 * T_ + 1)


@pytest.mark.parametrize("kind", ["cams", "bgr_maps", "fld"])
def test_session_kinds(kind):
    S, T_ = 4, 4
    tw, lc = make(kind, S)
    ids = np.int32([3, 1, 0, 2])
    st = start(tw, S, T_ + 2, 31, ids, ids[:3], lc)
    sched = np.uint8([[1, 0, 1, 2], [1, 1, 0, 1], [2, 1, 1, 0], [0, 0, 0, 0]])
    frames = schedule_frames(sched, frame_source(tw, st, ids, lc))
    compare(tw, ids, sched, frames)
    k = tw.e.keyframe_config()
    sched2 = np.uint8([[1, 1, 0, 1]])
    frames2 = schedule_frames(sched2, lambda t, kk: frame_source(tw, st, ids, lc)(t + T_, kk))
    compare(tw, ids, sched2, frames2, k, kf_state=tw.e.initial_keyframe_state(S))


def test_empty_calls():
    S = 3
    tw, _ = make("plain", S)
    ids = np.int32([0, 1, 2])
    st = start(tw, S, 4, 41, ids, ids)
    sched = np.ones((1, S), np.uint8)
    compare(tw, ids, sched, schedule_frames(sched, frame_source(tw, st, ids)))
    # T = 0, and a call where every stream idles: fast_th's rows are row 0, and _read still returns the last call's frames
    for T_ in (0, 3):
        sched = np.zeros((T_, S), np.uint8)
        empty = dict(img_l=np.zeros((0, tw.H, tw.W), np.uint8), img_r=np.zeros((0, tw.H, tw.W), np.uint8))
        res, fast_th, ns = tw.A.run_schedule(tw.h, ids, sched, empty, np.int32([0, 9, 40]))
        assert fast_th.shape == (T_ + 1, S) and (fast_th == np.int32([tw.oc.fast_threshold, 9, 40])).all()
        assert not res.tobytes().strip(b"\0") and not ns.any()
        same_read(tw.A, tw.B)
    follow_up(tw, st, ids, 3)


def test_errors_leave_the_session_usable():
    S = 3
    tw, _ = make("plain", S)
    ids = np.int32([0, 1, 2])
    st = start(tw, S, 5, 51, ids, np.int32([0, 1]))
    fs = frame_source(tw, st, ids)
    ok = np.uint8([[1, 1, 2]])
    A = tw.A

    def refused(code, msg, sched, frames=None, **kw):
        frames = frames if frames is not None else schedule_frames(np.where(sched > 2, 1, sched), fs)
        with pytest.raises(PlstvoError) as ei:
            A.run_schedule(tw.h, ids, sched, frames, **kw)
        assert ei.value.code == code and msg in str(ei.value), str(ei.value)

    refused(E_INVALID, "schedule value outside {0, 1, 2}", np.uint8([[1, 3, 1]]))
    refused(E_INVALID, "schedule value outside {0, 1, 2}", np.uint8([[1, 1, 2], [255, 0, 0]]))
    for wide in (256, -1):   # the binding refuses what uint8 would wrap (256 would read as 0, an idle entry)
        with pytest.raises(ValueError, match="schedule"):
            A.run_schedule(tw.h, ids, np.int64([[1, 1, wide]]), schedule_frames(np.uint8([[1, 1, 0]]), fs))
    refused(E_SIZE, "frames->B differs", ok, schedule_frames(np.uint8([[1, 1, 0]]), fs))
    refused(E_INVALID, "insert on a stream with no frame", np.uint8([[1, 1, 1]]))            # at the call's start
    refused(E_INVALID, "insert on a stream with no frame", np.uint8([[1, 1, 0], [0, 0, 1], [0, 0, 2]]))
    bad = schedule_frames(ok, fs)
    bad["fast_th"] = np.int32([5, 0, 0])
    refused(E_INVALID, "fast_th of an insert entry", ok, bad)
    bad["fast_th"] = np.int32([0, 0, 256])
    refused(E_INVALID, "initialize entry's threshold", ok, bad)
    refused(E_INVALID, "fast_th0 outside", ok, fast_th0=np.int32([0, -1, 0]))
    kbad = tw.e.initial_keyframe_state(S)
    kbad["prev_f_iskf"][1] = 2
    refused(E_INVALID, "prev_f_iskf", ok, kcfg=tw.e.keyframe_config(), kf_state=kbad)
    with pytest.raises(PlstvoError) as ei:   # the image limit counts the present images only
        big = np.ones((10923, S), np.uint8)   # 2 x 32769 present images
        one = dict(img_l=np.zeros((32769, 1, 1), np.uint8), img_r=np.zeros((32769, 1, 1), np.uint8))
        A.run_schedule(tw.h, ids, big, one)
    assert ei.value.code == E_INVALID and "65535 images" in str(ei.value)
    big = np.zeros((11000, S), np.uint8)   # T n far beyond, present frames within: passes the limit, fails on the size
    big[:2, :2] = 1
    with pytest.raises(PlstvoError) as ei:
        A.run_schedule(tw.h, ids, big, dict(img_l=np.zeros((4, 1, 1), np.uint8), img_r=np.zeros((4, 1, 1), np.uint8)))
    assert ei.value.code == E_SIZE and "image size" in str(ei.value)
    # every refusal left the session usable: the schedule then equals the chain
    compare(tw, ids, ok, schedule_frames(ok, fs))
    follow_up(tw, st, ids, 3)


def test_dense_schedule_launches_the_run_plus_two_per_step():
    """The dense schedule is the run's steps, each with one slot gather and one slot update more; the run itself keeps its
    launches (its host path is the parent's, and session.cu / keyframe.cu's existing kernels compile to the same SASS)."""
    S, T_ = 3, 3
    tw, _ = make("plain", S, retain=False)
    ids = np.int32([1, 2, 0])
    st = start(tw, S, T_ + 2, 61, ids, ids)
    sched = np.ones((T_, S), np.uint8)
    frames = schedule_frames(sched, frame_source(tw, st, ids))
    e = tw.e
    l0 = e.launches
    got = tw.A.run_schedule(tw.h, ids, sched, frames)
    l1 = e.launches
    want = tw.B.run(tw.h, ids, T_, frames)
    l2 = e.launches
    for x, y in zip(got, want):
        assert x.tobytes() == y.tobytes()
    assert (l1 - l0) - (l2 - l1) == 2 * T_, (l1 - l0, l2 - l1)


def test_handler_example_equals_the_per_frame_calls(tmp_path):
    """examples/schedule_cpp.cpp: StereoStreamsHandler::insertStereoSequences with a schedule leaves every stream's handler
    state as the per-frame initialize / insertStereoPairs / optimizePose / needNewKF / currFrameIsKF / updateFrame calls do,
    with and without the key-frame test: a late camera, drops, an empty round, a stream re-initialised and then tracked, one
    whose last entry re-initialises it after an insert, and a flat frame whose pair fails."""
    import struct
    import subprocess
    from test_gpu_track_images import moving_views
    from test_gpu_track_images_lsd import images_only
    from test_session_schedule_host import build_schedule_example
    W, H, S = 640, 376, 4
    NF = 8
    scenes = [images_only(moving_views(NF, W, H, 700 + 31 * s, 0)) for s in range(S)]
    scenes[0]["img_l"][4] = 90   # stream 0's fifth frame: flat, the pair fails
    scenes[0]["img_r"][4] = 90
    # per round the named streams (-(id + 1): re-initialise); stream 3 comes online at round 3, stream 1 is re-initialised
    # at round 3 and tracked after it, stream 2's last entry re-initialises it after an insert in the round before
    rounds = [[0, 1, 2], [0, 2], [], [0, 1, 2, 3], [0, -2, 2, 3], [0, 1, 3], [1, 2, 3], [0, 1, -3, 3]]
    pos = {s: 0 for s in range(S)}
    path = tmp_path / "schedule.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiii", W, H, S, len(rounds)))
        for rnd in rounds:
            f.write(struct.pack("<i", len(rnd)))
            for x in rnd:
                s = x if x >= 0 else -x - 1
                f.write(struct.pack("<i", x))
                f.write(np.ascontiguousarray(scenes[s]["img_l"][pos[s]]).tobytes())
                f.write(np.ascontiguousarray(scenes[s]["img_r"][pos[s]]).tobytes())
                pos[s] += 1
    exe = build_schedule_example(tmp_path)
    for extra in ([], ["no-kf"]):
        one, loop = (subprocess.run([exe, str(path)] + extra + mode, capture_output=True, text=True, check=True).stdout
                     .strip().splitlines() for mode in ([], ["per-frame"]))
        assert len(one) == len(loop)
        fails = 0
        for a, b in zip(one, loop):
            if a.startswith("kfstate"):   # the device's test rounds log like CUDA: its doubles agree to the last ulps
                x, y = a.split(), b.split()
                assert x[1] == y[1]
                np.testing.assert_allclose(np.float64(x[2:]), np.float64(y[2:]), rtol=1e-9, atol=1e-12)
            else:
                assert a == b, (extra, a[:120], b[:120])
                fails += a.startswith("round") and a.split()[5] == "0"
        assert fails >= 1, "a failed pair"
        states = [line for line in one if line.startswith("stream")]
        assert len(states) == S and all(" has_prev 1 " in line for line in states)
