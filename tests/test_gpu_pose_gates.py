"""The gates and the finishing step of optimizePose whose inputs the caller controls exactly, through the public API:
plstvo_track_batch and plstvo_optimize_pose, run once with K2 pinned and once with the streamed solver pinned (PLSTVO_STREAM_SOLVE
is read once per process, so each setting runs in a subprocess), against the oracle and, where oracle/_ref is built, the
reference's own optimizePose.

  * the motion-model prior gate (isGoodSolution on the prior, src/stereoFrameHandler.cpp:317-326), with DT_cov, err_norm and DT
    placed at its thresholds: both verdicts occur, each changes (or leaves) the oracle's result, and both solvers give
    the oracle's status and iteration counts exactly (the gate is the same code in both);
  * a previous frame whose heading is pi - delta with 1 km of translation and an anisotropic Tfw_cov: Tfw within the logmap bound
    of hp_pose evaluated on the returned DT (the fixed 1e-8 of test_gpu_pose.compare does not hold near pi), Tfw_cov within
    1e-12 relative;
  * a 40-frame chain through the Python handler mirror at 0.1 rad of yaw per frame across pi, against the oracle's chain."""
import os
import pickle
import subprocess
import sys

import mpmath as mp
import numpy as np
import pytest

import hp_pose as HP
import ref_numpy as R
from conftest import ROOT
from oracle import ref as ref_mod
from stvo_pl_b200 import synth, types as T
from test_gpu_pose import compare

pytestmark = pytest.mark.gpu
STREAM_ANG, STREAM_TR = 1e-7, 1e-6        # the streamed solver's bars where a pair's inlier flags equal the oracle's
E12 = 1e-12

SCRIPT = r'''
import pickle, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from stvo_pl_b200.engine import Engine
calls = pickle.load(open(sys.argv[2], "rb"))
eng = Engine(0)
out = []
for c in calls:
    if c[0] == "track":
        out.append(eng.track_batch(*c[1:]))
    else:
        res, ip, il = eng.optimize_pose(*c[1:])
        out.append(dict(results=res, inlier_pt=ip, inlier_ls=il))
eng.close()
pickle.dump(out, open(sys.argv[3], "wb"))
'''


def _pinned(tmp_path, setting, calls):
    """Runs `calls` on one Engine in a subprocess with PLSTVO_STREAM_SOLVE = setting ("0": K2, "1": streamed)."""
    env = {k: v for k, v in os.environ.items() if k not in ("PLSTVO_STREAM_SOLVE", "PLSTVO_K2_FEAT_GLOBAL")}
    env["PLSTVO_STREAM_SOLVE"] = setting
    job, res = str(tmp_path / f"job{setting}.pkl"), str(tmp_path / f"res{setting}.pkl")
    with open(job, "wb") as f:
        pickle.dump(calls, f)
    r = subprocess.run([sys.executable, "-c", SCRIPT, ROOT, job, res], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    with open(res, "rb") as f:
        return pickle.load(f)


def _check_results(gpu, ref, setting, label):
    """Status, verdict and iteration counts identical to the oracle's; pose within 1e-9 rad / 1e-8 m (K2) or the streamed bars."""
    for p in range(len(ref["results"])):
        g, r = gpu["results"][p], ref["results"][p]
        for key in ("status", "good", "iters_stage1", "iters_stage2"):
            assert g[key] == r[key], (label, setting, p, key, g[key], r[key])
        ang, tr = R.pose_error(g["DT"], r["DT"])
        assert ang < (1e-9 if setting == "0" else STREAM_ANG) and tr < (1e-8 if setting == "0" else STREAM_TR), (label, setting, p, ang, tr)


def _spd(rng, lam):
    q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    A = (q * np.asarray(lam, np.float64)) @ q.T
    return 0.5 * (A + A.T)


def _gate_priors(Ts, seed):
    """One prior per pair, placed at the prior gate's thresholds; returns (priors, the exact verdict per pair)."""
    rng = np.random.default_rng(seed)
    base = np.diag([0.25, 0.125, 0.0625, 0.3125, 0.125, 0.125])          # trace exactly 1
    small = np.eye(6) * 1e-6
    upper_nan = _spd(rng, [1e-5, 2e-5, 1e-6, 3e-6, 1e-4, 5e-6])
    upper_nan[np.triu_indices(6, 1)] = np.nan                             # only the lower triangle is read
    nan_low_bad, nan_low_good = np.diag([0.1, 0.1, 1.5, 0.1, 0.1, 0.1]), np.diag([0.1] * 6)
    nan_low_bad[4, 1] = nan_low_good[4, 1] = np.nan                        # the verdict is the diagonal's (DESIGN.md §3)
    nan_dt, inf_dt = np.eye(4), np.eye(4)
    nan_dt[0, 3], inf_dt[2, 1] = np.nan, np.inf
    lam = lambda v, cl: _spd(rng, np.r_[[v] * cl, rng.uniform(0.1, 0.9, 6 - cl)])   # a cluster of cl eigenvalues at v
    # (DT_cov, err_norm, DT override or None, exact verdict or None to take it from hp_pose)
    spec = [(lam(1 - 2.5 * E12, 1), 0.2, None, None), (lam(1 + 2.5 * E12, 1), 0.2, None, None),
            (lam(1 + 2.5 * E12, 3), 0.2, None, None), (lam(1 - 2.5 * E12, 6), 0.2, None, None),
            (lam(2.5 * E12, 2), 0.2, None, None), (lam(-2.5 * E12, 1), 0.2, None, None),
            (lam(-2.5 * E12, 4), 0.2, None, None),
            (base, 0.2, None, None), (base * (1 + 2.0 ** -52), 0.2, None, None),
            (np.diag([0.4, 0.1, 0.05, 0.02, 0.01, 0.4 * 1e-10 * (1 - 2.0 ** -40)]), 0.2, None, None),
            (small, 1.0, None, None), (small, np.nextafter(1.0, 2), None, None), (small, -0.0, None, None),
            (small, -5e-324, None, None), (small, np.nan, None, True),
            (small, 0.2, nan_dt, False), (small, 0.2, inf_dt, False),
            (upper_nan, 0.2, None, True), (nan_low_bad, 0.2, None, False), (nan_low_good, 0.2, None, True)]
    assert len(spec) == len(Ts)
    pri = T.identity_priors(len(Ts))
    want = []
    for p, (cov, err, dt, v) in enumerate(spec):
        pri["DT"][p] = Ts[p] if dt is None else dt                       # the true motion: GN from it takes fewer steps
        pri["DT_cov"][p], pri["err_norm"][p] = cov, err
        if v is None:
            v = HP.is_good(pri["DT"][p], cov, err)
            if np.all(np.isfinite(cov)):
                w = HP.eigvals(cov)
                assert min(abs(float(w[0])), abs(float(w[-1] - 1))) > HP.eig_bound(cov)   # placed outside the eigenvalue bound
        want.append(bool(v))
    return pri, want


def _gate_check(ref, ref_off, want, label):
    """Both verdicts occur, and each matters: an accepted prior starts Gauss-Newton elsewhere, so the oracle's result differs
    from its result without the motion model (in the iteration counts for most pairs, in the pose bits for all); a rejected one
    leaves the oracle's result exactly as without the motion model."""
    assert any(want) and not all(want)
    iters_changed = 0
    for p, v in enumerate(want):
        r, o = ref["results"][p], ref_off["results"][p]
        if v:
            assert r["DT_opt"].tobytes() != o["DT_opt"].tobytes(), (label, p)
            iters_changed += (r["iters_stage1"], r["iters_stage2"]) != (o["iters_stage1"], o["iters_stage2"])
        else:
            assert r.tobytes() == o.tobytes(), (label, p)
    assert 2 * iters_changed >= sum(want), (label, iters_changed, sum(want))


def test_prior_gate_through_track_batch_and_optimize_pose(tmp_path, oracle):
    n = 20
    prev, curr, Ts, cam = synth.make_batch("kitti", n, first_pair=300, n_pt=500, n_ls=120)
    pri, want = _gate_priors(Ts, 51)
    mb, Tm, cam_m = synth.make_matched_batch("kitti", n, first_pair=300)
    pri_m, want_m = _gate_priors(Tm, 52)
    cfg, cfg_off = T.kitti_config(), T.kitti_config()
    cfg.use_motion_model = 1
    ref = oracle.track_batch(cam, cfg, prev, curr, priors=pri, threads=4)
    _gate_check(ref, oracle.track_batch(cam, cfg_off, prev, curr, priors=pri, threads=4), want, "track")
    _, res_m, ip_m, il_m = oracle.optimize_pose(cam_m, cfg, mb, priors=pri_m)
    ref_m = dict(results=res_m, inlier_pt=ip_m, inlier_ls=il_m)
    _, res_off, _, _ = oracle.optimize_pose(cam_m, cfg_off, mb, priors=pri_m)
    _gate_check(ref_m, dict(results=res_off), want_m, "optimize_pose")
    if ref_mod.available():   # the reference's own optimizePose on the same lists and priors
        rf = ref_mod.Ref()
        _, rr, _, _ = rf.optimize_pose(cam_m, cfg, mb, priors=pri_m)
        for p in range(n):    # (its record carries no iteration counts)
            cov = pri_m["DT_cov"][p]
            if np.isnan(np.tril(cov)).any():
                # a known difference (DESIGN.md §3): its eigen solver turns a NaN entry into six NaN eigenvalues, which pass
                # isGoodSolution, so it takes a prior this project and the oracle judge by the covariance's diagonal
                assert np.isnan(rf.eig6_sym(cov)).all()
                continue
            assert rr["good"][p] == res_m["good"][p], p
            ang, tr = R.pose_error(rr["DT"][p], res_m["DT"][p])
            assert ang < 1e-9 and tr < 1e-8, (p, ang, tr)
    calls = [("track", cam, cfg, prev, curr, pri), ("opt", cam_m, cfg, mb, pri_m)]
    runs = {s: _pinned(tmp_path, s, calls) for s in ("0", "1")}
    for s, (g, gm) in runs.items():
        _check_results(g, ref, s, "track")
        _check_results(gm, ref_m, s, "optimize_pose")
    compare(runs["0"][0], ref, prev)           # K2: every tight bar of the pose suite
    for k in range(2):                          # the prior verdict is the same code in both solvers: same iterations
        for key in ("status", "iters_stage1", "iters_stage2"):
            np.testing.assert_array_equal(runs["0"][k]["results"][key], runs["1"][k]["results"][key])


def _check_tfw(res, pri, label):
    """Tfw within the logmap bound of the restatement on the returned DT wherever that bound makes a claim; Tfw_cov within 1e-12 relative of Tfw_cov_prev + Ad cov Ad^T.  Returns how many Tfw had a finite claim."""
    claims = 0
    for p in range(len(res)):
        r = res[p]
        assert r["good"], (label, p)
        want, b = HP.tfw(pri["Tfw"][p], r["DT"])
        if want is not None and b <= 1.0:   # else the cosine is within a few eps of -1, where whether the formula divides
                                            # by zero is a rounding of the product (test_gpu_pose_helpers checks exact half turns)
            claims += 1
            assert np.abs(r["Tfw"] - want).max() <= b, (label, p, np.abs(r["Tfw"] - want).max(), b)
        wc, bc = HP.unccomp(pri["Tfw"][p], pri["Tfw_cov"][p], r["DT_cov"])
        assert np.all(np.abs(r["Tfw_cov"] - wc) <= bc), (label, p)
        np.testing.assert_allclose(r["Tfw_cov"], wc, rtol=E12, atol=E12 * np.abs(wc).max())
    return claims


def test_half_turn_previous_frame(tmp_path, oracle):
    """Tfw_prev = (heading pi - delta, 1 km of translation) times the inverse of the oracle's DT, so that the Tfw each solver forms
    has the heading pi - delta to within the solvers' pose agreement; anisotropic Tfw_cov_prev."""
    deltas = [mp.mpf("1e-2"), mp.mpf("1e-4"), mp.mpf("1e-6"), mp.mpf("1e-8"), mp.mpf(0)]
    n = len(deltas)
    prev, curr, _, cam = synth.make_batch("kitti", n, first_pair=400, n_pt=500, n_ls=120)
    cfg = T.kitti_config()
    dt = oracle.track_batch(cam, cfg, prev, curr, threads=4)["results"]["DT"]
    rng = np.random.default_rng(61)
    pri = T.identity_priors(n)
    for p, d in enumerate(deltas):
        target = HP.rodrigues(mp.pi - d, [0.01, 1.0, -0.02], rng.uniform(-1e3, 1e3, 3))
        Di = np.eye(4)
        Di[:3, :3] = dt[p][:3, :3].T
        Di[:3, 3] = -dt[p][:3, :3].T @ dt[p][:3, 3]
        pri["Tfw"][p] = target @ Di
        pri["Tfw_cov"][p] = np.diag([4e-2, 1e-2, 1e-3, 3e-5, 1e-5, 2e-6]) + 1e-7 * np.ones((6, 6))
    ref = oracle.track_batch(cam, cfg, prev, curr, priors=pri, threads=4)
    assert _check_tfw(ref["results"], pri, "oracle") >= 2
    runs = {s: _pinned(tmp_path, s, [("track", cam, cfg, prev, curr, pri)])[0] for s in ("0", "1")}
    for s, g in runs.items():
        _check_results(g, ref, s, "half turn")
        assert _check_tfw(g["results"], pri, f"PLSTVO_STREAM_SOLVE={s}") >= 2
        for p in range(n):   # each Tfw really sits at the placed heading
            c = HP.cosine(pri["Tfw"][p] @ g["results"]["DT"][p])
            assert abs(float(mp.acos(c) - (mp.pi - deltas[p]))) < 1e-7 or c == -1.0, (s, p, c)


def test_forty_frame_chain_across_a_half_turn(engine, oracle):
    """app/imagesStVO.cpp's call sequence through the Python handler mirror, 40 frames turning 0.1 rad per frame about the
    camera's vertical axis, so the heading passes pi; against the oracle's own chain (each pair solved with the oracle's
    previous frame as prior).  At each frame Tfw is within the logmap bound of the restatement on the returned DT, and the two
    chains stay within the sum of those bounds plus the solvers' pose agreement."""
    from stvo_pl_b200.handler import StereoFrameHandler
    cfg, cam = T.kitti_config(), T.kitti_camera()
    step = synth.expmap_se3([0.0, 0.0, 0.8, 0.0, 0.1, 0.0])
    frames = [synth.make_batch("kitti", 1, first_pair=500 + k, n_pt=500, n_ls=120, motion=step)[:2] for k in range(40)]
    h = StereoFrameHandler(cam, cfg, engine)
    h.initialize(frames[0][0])
    pri = T.identity_priors(1)
    drift, headings = 0.0, []
    for k, (prev, curr) in enumerate(frames):
        h.prev_frame.features = prev
        Tfw_prev = h.prev_frame.Tfw.copy()
        h.insertStereoPair(curr, k + 1)
        h.optimizePose()
        r = oracle.track_batch(cam, cfg, prev, curr, priors=pri)["results"][0]
        c = h.curr_frame
        assert h.status == r["status"] and c.DT is not None
        ang, tr = R.pose_error(c.DT, r["DT"])
        assert ang < 1e-9 and tr < 1e-8, (k, ang, tr)
        want, b = HP.tfw(Tfw_prev, c.DT)
        assert want is not None and b < 1e-6, (k, b)
        assert np.abs(c.Tfw - want).max() <= b, (k, np.abs(c.Tfw - want).max(), b)
        drift += b + 1e-8 * (1.0 + np.abs(c.Tfw[:3, 3]).max())
        assert np.abs(c.Tfw - r["Tfw"]).max() <= drift, (k, np.abs(c.Tfw - r["Tfw"]).max(), drift)
        np.testing.assert_allclose(c.Tfw_cov, r["Tfw_cov"], rtol=1e-6, atol=1e-12)
        headings.append(float(np.arccos(HP.cosine(c.Tfw))))
        pri["Tfw"][0], pri["Tfw_cov"][0] = r["Tfw"], r["Tfw_cov"]
        pri["DT"][0], pri["DT_cov"][0], pri["err_norm"][0] = r["DT"], r["DT_cov"], r["err_norm"]
        h.updateFrame()
    i = int(np.argmax(headings))
    assert headings[i] > np.pi - 0.1 and 0 < i < 39 and headings[-1] < headings[i] - 0.5, headings   # the heading passed pi
