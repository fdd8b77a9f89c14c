"""plstvo_stereo_session_run_keyframes on the GPU: the run with the key-frame test against the per-frame insert loop on a twin
session driven by the host test (handler.KeyframeTest per stream, and currFrameIsKF's reset of the next prior): results,
n_stereo and threshold rows byte for byte, decisions and counters equal, diagnostics within the host bar, the final state,
and a follow-up insert.  Decisions are also checked against plstvo.hpp's KeyframeTest compiled on the host.  Sizes S = 1,
37, SMs + 5 and T = 1, 4, 13; the session kinds of test_gpu_session_run.py; every branch of needNewKF; continuation and
subsets; a config that cannot fire against the plain run; retention; errors; and examples/run_kf_cpp.cpp."""
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

from conftest import ROOT
from test_gpu_session_run import Twins, follow_up, priors_of, rule, same_read, step_major
from test_gpu_track_images import sm_count
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError
from stvo_pl_b200.handler import KeyframeTest

pytestmark = pytest.mark.gpu

INF = float("inf")
BRANCHES = Counter()
MARGIN = [INF]   # the smallest relative distance of a compared quantity to the threshold it was compared with


def kcfg(ratio=0.85, t=5.0, r=15.0):
    return np.array([(ratio, t, r)], T.KEYFRAME_CONFIG_DTYPE)


def kf_test(kt, k, r):
    """needNewKF of the host test on one result, counting every criterion that holds, and the decision's row."""
    first = kt.prev_f_iskf
    fire = kt.needNewKF(_Cfg(k), r["Tfw"], r["DT"], r["DT_cov"])
    ratio = kt.entropy_ratio
    if first and kt.entropy_first_prevKF == -999999999.99:
        BRANCHES["first_det_zero"] += 1
    if ratio < k["min_entropy_ratio"][0]:
        BRANCHES["ratio"] += 1
    if not np.isfinite(ratio):
        BRANCHES["nan_inf"] += 1
    if not r["DT_cov"].any() and np.array_equal(r["DT"], np.eye(4)):
        BRANCHES["failed_solve"] += 1
    if kt.t > k["max_kf_t_dist"][0]:
        BRANCHES["t"] += 1
    if kt.r > k["max_kf_r_dist"][0]:
        BRANCHES["r"] += 1
    if fire and kt.N_prevKF_currF > 10:
        BRANCHES["counter"] += 1
    for v, th in ((ratio, k["min_entropy_ratio"][0]), (kt.t, k["max_kf_t_dist"][0]), (kt.r, k["max_kf_r_dist"][0])):
        if np.isfinite(v) and np.isfinite(th) and th != 0:
            MARGIN[0] = min(MARGIN[0], abs(v - th) / abs(th))
    row = (int(fire), kt.N_prevKF_currF, kt.entropy_curr, kt.entropy_ratio, kt.t, kt.r)
    if fire:
        kt.currFrameIsKF(_Frame())
    return row


class _Cfg:
    def __init__(self, k):
        self.min_entropy_ratio, self.max_kf_t_dist, self.max_kf_r_dist = (float(k[f][0]) for f in k.dtype.names)


class _Frame:
    pass


def kf_loop(ss, h, oc, k, ids, frames, T_, state, th0=None, priors=None):
    """The per-frame loop with the host test: (results, rows, n_stereo, kf rows [T][n] as tuples, final states)."""
    n = len(ids)
    kts = [KeyframeTest.from_state(state[i]) for i in range(n)]
    th = np.int32(np.full(n, oc.fast_threshold) if th0 is None else np.where(np.int32(th0) == 0, oc.fast_threshold, th0))
    rows, res_all, ns_all, kfs, pri = [th.copy()], [], [], [], priors
    for t in range(T_):
        fr = dict(img_l=frames["img_l"][t * n:(t + 1) * n], img_r=frames["img_r"][t * n:(t + 1) * n], fast_th=th.copy())
        res, ns = ss.insert(ids, fr, pri)
        th = np.int32([rule(h, int(th[i]), res[i]) for i in range(n)])
        kfs.append([kf_test(kts[i], k, res[i]) for i in range(n)])
        pri = reset_priors(res, [x[0] for x in kfs[-1]])
        rows.append(th.copy())
        res_all.append(res.copy())
        ns_all.append(ns.copy())
    return np.stack(res_all), np.stack(rows), np.stack(ns_all), kfs, np.concatenate([x.to_state() for x in kts])


def reset_priors(res, new_kf):
    p = priors_of(res)
    for i, f in enumerate(new_kf):
        if f:
            p["Tfw"][i], p["Tfw_cov"][i] = np.eye(4), np.eye(6)
    return p


def agree(got_kf, want_kf):
    """Decisions and counters equal, diagnostics within test_handler_state.py's bar for the host implementations."""
    for t, row in enumerate(want_kf):
        for i, w in enumerate(row):
            g = got_kf[t, i]
            assert (int(g["new_kf"]), int(g["N_prevKF_currF"])) == w[:2], (t, i, g, w)
            for j, f in enumerate(("entropy_curr", "entropy_ratio", "t", "r")):
                x, y = float(g[f]), w[2 + j]
                if np.isfinite(x) or np.isfinite(y):
                    assert x == pytest.approx(y, rel=1e-9, abs=1e-12), (t, i, f, x, y)


def same_state(got, want):
    for f in ("prev_f_iskf", "N_prevKF_currF"):
        np.testing.assert_array_equal(got[f], want[f])
    for f in ("T_prevKF", "cov_prevKF_currF", "entropy_first_prevKF"):
        np.testing.assert_allclose(got[f], want[f], rtol=1e-9, atol=1e-12)


CPP_HELPER = r'''#include <cstdio>
#include "plstvo.hpp"
// stdin: PlKeyframeConfig, PlKeyframeState, int32 T, then T records of Tfw [16], DT [16], DT_cov [36]; prints each test
int main() {
    PlKeyframeConfig k;
    PlKeyframeState s;
    int32_t T;
    if (std::fread(&k, sizeof k, 1, stdin) != 1 || std::fread(&s, sizeof s, 1, stdin) != 1 || std::fread(&T, 4, 1, stdin) != 1)
        return 2;
    plstvo::HandlerConfig hc;
    hc.min_entropy_ratio = k.min_entropy_ratio; hc.max_kf_t_dist = k.max_kf_t_dist; hc.max_kf_r_dist = k.max_kf_r_dist;
    plstvo::KeyframeTest kt = plstvo::KeyframeTest::fromState(s);
    for (int t = 0; t < T; ++t) {
        double rec[68];
        if (std::fread(rec, sizeof rec, 1, stdin) != 1) return 2;
        plstvo::StereoFrame f;
        std::copy(rec, rec + 16, f.Tfw.begin());
        std::copy(rec + 16, rec + 32, f.DT.begin());
        std::copy(rec + 32, rec + 68, f.DT_cov.begin());
        const bool kf = kt.needNewKF(hc, f);
        std::printf("%d %d\n", kf ? 1 : 0, kt.N_prevKF_currF);
        if (kf) kt.currFrameIsKF(f);
    }
    return 0;
}
'''


@pytest.fixture(scope="module")
def cpp_kf(tmp_path_factory):
    d = tmp_path_factory.mktemp("kfcpp")
    (d / "kf.cpp").write_text(CPP_HELPER)
    exe = str(d / "kf")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(d / "kf.cpp"),
                    "-o", exe], check=True)
    return exe


def check_cpp(exe, k, state, res, kf):
    """Per stream, plstvo.hpp's KeyframeTest over the run's results gives the run's decisions and counters."""
    for i in range(res.shape[1]):
        blob = k.tobytes() + state[i:i + 1].tobytes() + np.int32(res.shape[0]).tobytes()
        for t in range(res.shape[0]):
            r = res[t, i]
            blob += np.concatenate([r["Tfw"].ravel(), r["DT"].ravel(), r["DT_cov"].ravel()]).astype(np.float64).tobytes()
        out = subprocess.run([exe], input=blob, capture_output=True, check=True).stdout.decode().split()
        got = np.int32(out).reshape(-1, 2)
        np.testing.assert_array_equal(got[:, 0], kf["new_kf"][:, i])
        np.testing.assert_array_equal(got[:, 1], kf["N_prevKF_currF"][:, i])


def check(kind, S, T_, seed, k, exe=None, follow=True):
    e = Engine()
    tw = Twins(e, kind, S)
    st = tw.frames(S, T_ + 2, seed)
    ids = np.int32(np.random.default_rng(seed).permutation(S))
    tw.init(st, ids)
    state = e.initial_keyframe_state(S)
    fr = step_major(st, ids, 1, T_)
    want = kf_loop(tw.B, tw.h, tw.oc, k, ids, fr, T_, state)
    s0 = state.copy()
    res, kf, rows, ns = tw.A.run_keyframes(tw.h, k, ids, T_, fr, state)
    assert res.tobytes() == want[0].tobytes()
    np.testing.assert_array_equal(rows, want[1])
    np.testing.assert_array_equal(ns, want[2])
    agree(kf, want[3])
    same_state(state, want[4])
    if exe:
        check_cpp(exe, k, s0, res, kf)
    same_read(tw.A, tw.B)
    if follow:
        last = dict(img_l=np.stack([st[i]["img_l"][T_ + 1] for i in ids]),
                    img_r=np.stack([st[i]["img_r"][T_ + 1] for i in ids]), fast_th=rows[-1])
        follow_up(tw.A, tw.B, ids, last, reset_priors(res[-1], kf["new_kf"][-1]))
    e.close()
    return kf


@pytest.mark.parametrize("S,T_", [(1, 13), (37, 4), ("sms+5", 1), ("sms+5", 13)])
def test_sizes(S, T_, cpp_kf):
    check("plain", sm_count() + 5 if S == "sms+5" else S, T_, 500 + T_, kcfg(0.95, 0.3, 2.0), cpp_kf)
    print(f"smallest relative margin to a threshold: {MARGIN[0]:.3g}")


@pytest.mark.parametrize("kind", ["cams", "bgr_maps", "no_points", "no_lines"])
def test_configs(kind, cpp_kf):
    check(kind, 7, 4, 600 + len(kind), kcfg(0.9, 0.2, 1.0), cpp_kf)


def test_every_branch_fires(cpp_kf):
    BRANCHES.clear()
    check("plain", 11, 4, 71, kcfg(0.999, INF, INF), cpp_kf)    # the entropy ratio
    check("plain", 11, 4, 72, kcfg(-INF, 1e-3, INF), cpp_kf)    # t
    check("plain", 11, 4, 73, kcfg(-INF, INF, 1e-3), cpp_kf)    # r
    kf = check("plain", 5, 13, 74, kcfg(-INF, INF, INF), cpp_kf)   # the counter, and the flat frames of scenes()
    assert kf["new_kf"].any()
    want = {"ratio", "nan_inf", "failed_solve", "t", "r", "counter", "first_det_zero"}
    assert want <= set(BRANCHES), (want - set(BRANCHES), dict(BRANCHES))
    print(dict(BRANCHES), f"smallest relative margin: {MARGIN[0]:.3g}")


def test_no_key_frame_equals_the_plain_run():
    """A config that cannot fire over T <= 11 steps of textured frames: the plain run's bytes, one launch more per step."""
    e = Engine()
    S, T_ = 2, 8
    tw = Twins(e, "plain", S)
    # scenes()' medium texture: the densest one can give a covariance whose determinant is negative (a NaN ratio fires), the
    # sparse one holds a flat frame (a failed solve fires); both streams view it
    st = [tw.frames(2, T_ + 1, 81)[1]] * S
    ids = np.int32(np.arange(S))
    tw.A.retain(False)
    tw.B.retain(False)
    tw.init(st, ids)
    fr = step_major(st, ids, 1, T_)
    state = e.initial_keyframe_state(S)
    l0 = e.launches
    res, kf, rows, ns = tw.A.run_keyframes(tw.h, kcfg(-INF, INF, INF), ids, T_, fr, state)
    l1 = e.launches
    want = tw.B.run(tw.h, ids, T_, fr)
    l2 = e.launches
    assert not kf["new_kf"].any() and state["N_prevKF_currF"].tolist() == [T_] * S
    assert res.tobytes() == want[0].tobytes()
    np.testing.assert_array_equal(rows, want[1])
    np.testing.assert_array_equal(ns, want[2])
    assert (l1 - l0) - (l2 - l1) == T_, (l1 - l0, l2 - l1)
    e.close()


def test_continuation_and_subsets():
    e = Engine()
    S, T1, T2 = 6, 3, 4
    tw = Twins(e, "plain", S)
    st = tw.frames(S, T1 + T2 + 1, 91)
    ids = np.int32([4, 1, 5, 0, 2, 3])
    tw.init(st, ids)
    k = kcfg(0.95, 0.2, 1.0)
    sa, sb = e.initial_keyframe_state(S), e.initial_keyframe_state(S)
    whole = tw.B.run_keyframes(tw.h, k, ids, T1 + T2, step_major(st, ids, 1, T1 + T2), sb)
    r1, k1, th1, _ = tw.A.run_keyframes(tw.h, k, ids, T1, step_major(st, ids, 1, T1), sa)
    r2, k2, th2, _ = tw.A.run_keyframes(tw.h, k, ids, T2, step_major(st, ids, 1 + T1, T2), sa, th1[-1],
                                        reset_priors(r1[-1], k1["new_kf"][-1]))
    assert np.concatenate([r1, r2]).tobytes() == whole[0].tobytes()
    assert np.concatenate([k1, k2]).tobytes() == whole[1].tobytes()
    assert sa.tobytes() == sb.tobytes()
    assert k1["new_kf"].any() or k2["new_kf"].any()
    # a subset: the unnamed streams keep their frames, and their state is the caller's
    sub = np.int32([5, 2])
    ssub = sa[[list(ids).index(i) for i in sub]].copy()
    frs = step_major(st, sub, T1 + T2, 1)
    tw.A.run_keyframes(tw.h, k, sub, 1, frs, ssub)
    tw.B.run_keyframes(tw.h, k, sub, 1, frs, sb[[list(ids).index(i) for i in sub]].copy())
    others = np.int32([i for i in ids if i not in sub])
    fo = dict(img_l=np.stack([st[i]["img_l"][T1 + T2] for i in others]), img_r=np.stack([st[i]["img_r"][T1 + T2] for i in others]))
    follow_up(tw.A, tw.B, others, fo, None)
    e.close()


def test_retention():
    """read_keyframes equals, row for row, what read returns after the key frame's own insert; read still gives the last step;
    a failed call and any other call discard the key frames; device bytes as the header states them."""
    e = Engine()
    S, T_ = 5, 5
    tw = Twins(e, "plain", S)
    st = tw.frames(S, T_ + 1, 101)
    ids = np.int32([3, 0, 4, 1, 2])
    tw.init(st, ids)
    k = kcfg(0.95, 0.2, 1.0)
    fr = step_major(st, ids, 1, T_)
    b0 = tw.A.device_bytes
    res, kf, rows, ns = tw.A.run_keyframes(tw.h, k, ids, T_, fr, e.initial_keyframe_state(S))
    grown = tw.A.device_bytes - b0
    per_step = [int(ns[t, :, 2].sum()) * 96 + int(ns[t, :, 3].sum()) * 176 for t in range(T_)]
    assert grown >= sum(per_step), (grown, per_step)
    kr, kpt, kls = tw.A.read_keyframes()
    want_rows = [(t, int(ids[i]), int(ns[t, i, 2]), int(ns[t, i, 3])) for t in range(T_) for i in range(S) if kf["new_kf"][t, i]]
    assert [tuple(r) for r in kr] == want_rows and len(want_rows) > 0
    # the loop on the twin, reading after each insert
    kts = [KeyframeTest() for _ in ids]
    th, pri, p0, l0, j = np.int32(np.full(S, tw.oc.fast_threshold)), None, 0, 0, 0
    for t in range(T_):
        f = dict(img_l=fr["img_l"][t * S:(t + 1) * S], img_r=fr["img_r"][t * S:(t + 1) * S], fast_th=th.copy())
        r, n_s = tw.B.insert(ids, f, pri)
        pt, ls = tw.B.read()[:2]
        fire = [kf_test(kts[i], k, r[i])[0] for i in range(S)]
        th = np.int32([rule(tw.h, int(th[i]), r[i]) for i in range(S)])
        pri = reset_priors(r, fire)
        op, ol = np.concatenate([[0], np.cumsum(n_s[:, 2])]), np.concatenate([[0], np.cumsum(n_s[:, 3])])
        for i in range(S):
            if not fire[i]:
                continue
            npt, nls = int(n_s[i, 2]), int(n_s[i, 3])
            for key in pt:
                if key != "counts":
                    assert kpt[key][p0:p0 + npt].tobytes() == pt[key][op[i]:op[i] + npt].tobytes(), (t, i, key)
            for key in ls:
                if key != "counts":
                    assert kls[key][l0:l0 + nls].tobytes() == ls[key][ol[i]:ol[i] + nls].tobytes(), (t, i, key)
            p0, l0, j = p0 + npt, l0 + nls, j + 1
    assert j == len(want_rows)
    same_read(tw.A, tw.B)   # both hold the last step
    # a failed call discards them, and frees their chunks
    full = tw.A.device_bytes
    with pytest.raises(PlstvoError):
        tw.A.run_keyframes(tw.h, kcfg(np.nan), ids, 1, step_major(st, ids, 1, 1), e.initial_keyframe_state(S))
    with pytest.raises(PlstvoError):
        tw.A.read_keyframes()
    assert tw.A.device_bytes <= full - sum(per_step)
    e.close()


def test_errors_leave_the_session_usable():
    e = Engine()
    S = 3
    tw = Twins(e, "plain", S)
    st = tw.frames(S, 4, 111)
    ids = np.int32([0, 1, 2])
    tw.init(st, ids)
    fr = step_major(st, ids, 1, 1)
    good = e.initial_keyframe_state(S)
    lib, ctx = e.lib, e.ctx
    import ctypes as C
    h = T.handler_config(tw.h)
    fs, keep = T.stereo_images_as_c(fr)
    res = np.zeros((1, S), T.POSE_RESULT_DTYPE)
    kf = np.zeros((1, S), T.KEYFRAME_RESULT_DTYPE)
    k = kcfg()

    def call(kp, sp, kfp):
        return lib.plstvo_stereo_session_run_keyframes(ctx, tw.A.handle, C.byref(h), kp, S, ids.ctypes.data_as(T.c_int32_p), 1,
                                                       C.byref(fs), None, None, sp, res.ctypes.data, kfp, None, None)
    assert call(None, good.ctypes.data, kf.ctypes.data) == -1
    assert call(k.ctypes.data, None, kf.ctypes.data) == -1
    assert call(k.ctypes.data, good.ctypes.data, None) == -1
    for f in ("min_entropy_ratio", "max_kf_t_dist", "max_kf_r_dist"):
        bad = k.copy()
        bad[f] = np.nan
        assert call(bad.ctypes.data, good.ctypes.data, kf.ctypes.data) == -1, f
    for f, v in (("prev_f_iskf", 2), ("prev_f_iskf", -1), ("N_prevKF_currF", -1)):
        bad = good.copy()
        bad[f][1] = v
        before = bad.tobytes()
        assert call(k.ctypes.data, bad.ctypes.data, kf.ctypes.data) == -1, f
        assert bad.tobytes() == before
    # a run error (an id out of range) leaves the state untouched too
    st0 = good.tobytes()
    with pytest.raises(PlstvoError):
        tw.A.run_keyframes(tw.h, k, np.int32([0, 1, 7]), 1, fr, good)
    assert good.tobytes() == st0
    # +-inf is allowed, and the session and context stay usable: the run equals the twin's loop
    del keep
    want = kf_loop(tw.B, tw.h, tw.oc, kcfg(-INF, INF, INF), ids, fr, 1, good.copy())
    got = tw.A.run_keyframes(tw.h, kcfg(-INF, INF, INF), ids, 1, fr, good)
    assert got[0].tobytes() == want[0].tobytes()
    e.close()


def test_run_kf_example(tmp_path):
    from test_session_keyframes_host import build_run_kf_example
    r = subprocess.run([build_run_kf_example(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "run with key frames equals the per-frame loop" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    assert " 0 key frames" not in r.stdout
