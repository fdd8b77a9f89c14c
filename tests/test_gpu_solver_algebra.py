"""The two 6x6 routines both pose solvers share besides the Cholesky (solve.cu): warp_qr6_solve, the column-pivoted QR that
solves and gives log|det| wherever the Cholesky refuses (ColPivHouseholderQR::solve / logAbsDeterminant,
src/stereoFrameHandler.cpp:417-418, :453-455), and warp_inv6, the partial-pivot LU inverse that gives every DT_cov (:429, :470).
They are run through plstvo_debug_algebra (QR x and log|det|, inverse, eigenvalues) and plstvo_debug_pose_helpers (the
Cholesky's verdict and its own QR x) on inputs placed at their edges, against the 60-digit restatement in hp_pose.py
(pinned to the oracle by test_hp_pose_host.py, which also shows the oracle's fp64 routines inside every bound used here),
and through plstvo_optimize_pose on point problems whose normal equations the Cholesky refuses, on K2 and on the streamed
solver.  Each family checks that it reached its edge and prints its largest error-to-bound ratio."""
import re

import mpmath as mp
import numpy as np
import pytest

import hp_pose as HP
from stvo_pl_b200 import synth, types as T
from test_gpu_pose_gates import _pinned

pytestmark = pytest.mark.gpu


def _ratio(err, bound):
    return float(err) / float(bound) if bound > 0 else (0.0 if err == 0 else np.inf)


def test_qr_full_rank_across_conditioning_and_scale(engine):
    """SPD systems with kappa 1 .. 1e14 at scales 1e-60 .. 1e60, point normal equations with rotation / translation scale
    disparity, and the hand-over band (kappa 4e12 .. 1e14) where the Cholesky must refuse and the QR solve at full rank: the
    backward bound everywhere, the forward and log|det| bounds where kappa eps <= 1e-2, the two hooks' x byte-identical (lane
    i's entry i against lane 0's six), and the Jacobi eigenvalues of the same matrices within the Weyl bound."""
    cases = HP.qr_full_cases(1)
    H = np.stack([c[0] for c in cases])
    g = np.stack([c[1] for c in cases])
    x, lad, _, eig = engine.debug_algebra(H, g)
    ph = engine.debug_pose_helpers(H=H, g=g)
    worst = {"back": 0.0, "fwd": 0.0, "lad": 0.0, "eig": 0.0}
    handover = 0
    for k, (Hk, gk, label) in enumerate(cases):
        assert x[k].tobytes() == ph["qr_x"][k].tobytes(), (label, x[k], ph["qr_x"][k])
        assert np.float64(lad[k]).tobytes() == np.float64(ph["qr_lad"][k]).tobytes(), label
        x_hp, lad_hp = HP.chol_solve(Hk, gk)
        bb, bf, bl = HP.qr_bounds(Hk, gk, x_hp)
        r = _ratio(HP.residual(Hk, gk, x[k]), bb)
        assert r <= 1.0, (label, "backward", r)
        worst["back"] = max(worst["back"], r)
        if HP.cond(Hk) * HP.EPS <= 1e-2:
            r = _ratio(np.linalg.norm(x[k] - x_hp), bf)
            assert r <= 1.0, (label, "forward", r)
            worst["fwd"] = max(worst["fwd"], r)
            r = _ratio(abs(lad[k] - float(lad_hp)), bl + HP.C_SOLVE * HP.EPS * abs(float(lad_hp)))
            assert r <= 1.0, (label, "log|det|", lad[k], float(lad_hp))
            worst["lad"] = max(worst["lad"], r)
        r = _ratio(np.abs(eig[k] - [float(v) for v in HP.eigvals(Hk)]).max(), HP.eig_bound(Hk))
        assert r <= 1.0, (label, "eigenvalues", r)
        worst["eig"] = max(worst["eig"], r)
        if label.startswith("handover"):
            assert not ph["chol_ok"][k], label        # the QR is what solves here
            handover += 1
    assert handover == 12
    print("full-rank QR and eigenvalues, largest error / bound:", worst)


def test_qr_rank_decisions_where_rounding_cannot_decide_them(engine):
    """P blockdiag(A, D) P^T (hp_pose.rank_cases): D's entries exactly 0 or at thr (1 +- 2^-40), and with a power-of-two diagonal
    A at thr itself and one ulp either side.  The truncated entries of x are exactly 0.0, the support is the restatement's and
    x on it within basic_bound of basic_solve, log|det| is -inf exactly where an R entry is 0, the rule is the strict > at thr,
    and both verdicts occur at every scale."""
    cases = HP.rank_cases(2)
    H = np.stack([c[0] for c in cases])
    g = np.stack([c[1] for c in cases])
    x, lad, _, _ = engine.debug_algebra(H, g)
    ph = engine.debug_pose_helpers(H=H, g=g)
    worst = 0.0
    verdicts = {}
    for k, (Hk, gk, label) in enumerate(cases):
        assert x[k].tobytes() == ph["qr_x"][k].tobytes(), label
        rank, S = HP.qr_rank(Hk)
        off = [j for j in range(6) if j not in S]
        assert np.all(x[k][off] == 0.0) and np.all(x[k][S] != 0.0), (label, x[k], S)
        want, b = HP.basic_solve(Hk, gk, S), HP.basic_bound(Hk, gk, S)
        if S:
            r = float(np.max(np.abs(x[k] - want)[S] / b[S]))
            assert r <= 1.0, (label, r)
            worst = max(worst, r)
        exact_zero = min(abs(d) for d in HP.qr_pivots(Hk)[1]) == 0.0
        assert (lad[k] == -np.inf) == exact_zero and (exact_zero or np.isfinite(lad[k])), (label, lad[k])
        r0, scale = int(re.search(r"r=(\d)", label).group(1)), label.split("s=")[1]
        if 0 < r0 < 6:
            verdicts.setdefault((label[:5], scale), set()).add(rank > r0)
        if label.startswith("exact"):
            assert rank == r0 + (" above " in label or " hi " in label), label
        assert not ph["chol_ok"][k] or rank == 6, label
    assert len(verdicts) == 6 and all(v == {True, False} for v in verdicts.values()), verdicts
    print("truncated QR, largest error / bound:", worst)


def test_qr_log_det_sign_where_the_cholesky_refuses(engine):
    """The robust loop stops with good = false on log|det H| < 0 (:455-459); where the Cholesky refuses, the QR's log|det|
    decides.  Hand-over matrices rescaled so that the exact log|det| sits at +-4x its bound: the Cholesky refuses every one,
    and the QR's sign is the exact sign."""
    rng = np.random.default_rng(7)
    H, targets = [], []
    for kappa in (4e12, 1e13, 1e14):
        for sgn in (1.0, -1.0):
            for _ in range(2):
                A = HP.handover_matrix(rng, kappa, 1.0)
                _, lad0 = HP.chol_solve(A, np.ones(6))
                _, bl = HP.solve_bounds(A, np.ones(6))
                t = sgn * 4.0 * bl
                H.append(A * float(mp.exp((t - lad0) / 6)))
                targets.append(t)
    H = np.stack(H)
    g = rng.normal(size=(len(H), 6))
    x, lad, _, _ = engine.debug_algebra(H, g)
    ph = engine.debug_pose_helpers(H=H, g=g)
    assert not ph["chol_ok"].any()
    signs = set()
    for k in range(len(H)):
        _, lad_hp = HP.chol_solve(H[k], g[k])
        _, bl = HP.solve_bounds(H[k], g[k])
        lad_hp = float(lad_hp)
        assert abs(lad_hp - targets[k]) <= 0.25 * abs(targets[k]) and abs(lad_hp) > 2 * bl, (k, lad_hp, targets[k], bl)
        assert np.sign(lad[k]) == np.sign(lad_hp) == np.sign(ph["qr_lad"][k]), (k, lad[k], lad_hp)
        signs.add(np.sign(lad_hp))
    assert signs == {1.0, -1.0}


def test_inverse_across_conditioning_scale_ties_and_asymmetry(engine):
    """warp_inv6 on hp_pose.inv_cases (kappa 1 .. 1e15 SPD at scales 1e-60 .. 1e60, non-symmetric, pivot columns of tied
    magnitudes, the hand-over band): the residual and forward bounds, and the eigenvalues of the symmetric ones up to kappa 1e14."""
    cases = HP.inv_cases(3)
    H = np.stack([c[0] for c in cases])
    _, _, X, eig = engine.debug_algebra(H, np.ones((len(H), 6)))
    worst = [0.0, 0.0]
    for k, (Hk, label) in enumerate(cases):
        res, rb, fwd, fb = HP.inv_errors(Hk, X[k])
        assert res <= rb and fwd <= fb, (label, res / rb, fwd / fb)
        worst = [max(worst[0], res / rb), max(worst[1], fwd / fb)]
        if np.array_equal(Hk, Hk.T):
            r = np.abs(eig[k] - [float(v) for v in HP.eigvals(Hk)]).max() / HP.eig_bound(Hk)
            if HP.cond(Hk) <= 1.5e14:
                assert r <= 1.0, (label, r)
            else:   # kappa 1e15: the Jacobi's stop rule leaves more than the Weyl bound (DESIGN.md §3), reported only
                print(f"Jacobi eigenvalues at {label}: error / Weyl bound {r:.3g}")
    print("LU inverse, largest residual / bound, forward / bound:", worst)


def test_inverse_at_an_exactly_zero_pivot(engine, oracle):
    """A zero row and column j: the LU meets an all-zero pivot column and divides 0 by 0, so the inverse is NaN everywhere, or
    (j = 5) NaN with +inf at (5, 5), the oracle's pattern exactly.  isGoodSolution on that DT_cov gives the oracle's verdict:
    an all-NaN covariance has a NaN diagonal, which both comparisons pass (the NaN rule of DESIGN.md §3), and the +inf is
    rejected."""
    rng = np.random.default_rng(4)
    H = []
    for j in range(6):
        A = HP.spd(rng, rng.uniform(0.5, 2.0, 6))
        A[j, :] = 0.0
        A[:, j] = 0.0
        H.append(A)
    H = np.stack(H)
    _, _, X, _ = engine.debug_algebra(H, np.ones((6, 6)))
    want_good = []
    for j in range(6):
        Xo = oracle.inv6(H[j])
        assert not np.all(np.isfinite(X[j])), j
        np.testing.assert_array_equal(np.isnan(X[j]), np.isnan(Xo))
        np.testing.assert_array_equal(np.isinf(X[j]), np.isinf(Xo))
        np.testing.assert_array_equal(X[j][np.isinf(X[j])], Xo[np.isinf(Xo)])
        want_good.append(oracle.is_good_solution(np.eye(4), Xo, 0.2))
    DT = np.tile(HP.rodrigues(mp.mpf("0.05"), [0.1, 1.0, 0.2], [0.1, 0.0, 0.8]), (6, 1, 1))
    out = engine.debug_pose_helpers(cov=X, DT=DT, err=np.full(6, 0.2))
    np.testing.assert_array_equal(out["good_full"], want_good)
    np.testing.assert_array_equal(out["good_fast"], want_good)
    assert want_good == [True] * 5 + [False]


# ---------------------------------------------------------------------------------------------------------------------
# through the public API: both solvers on normal equations the Cholesky refuses
# ---------------------------------------------------------------------------------------------------------------------
def _patch_problem(seed, n, width, depth, u0, v0=180.0):
    """n points in a width x (2/3 width) pixel patch at one depth, seen after a small motion with 0.05 px of noise."""
    rng = np.random.default_rng(seed)
    cam = T.kitti_camera()
    u, v = rng.uniform(u0, u0 + width, n), rng.uniform(v0, v0 + width * 2 / 3, n)
    P = synth.back_projection(cam, u, v, np.full(n, cam.b * cam.fx / depth))
    Tgt = synth.expmap_se3(np.array([0.01, 0.0, -0.3, 0.001, -0.002, 0.0005]))
    obs = synth.projection(cam, P @ Tgt[:3, :3].T + Tgt[:3, 3]) + rng.normal(0, 0.05, (n, 2))
    return P, obs


def _points_batch(problems):
    P = np.concatenate([p[0] for p in problems])
    obs = np.concatenate([p[1] for p in problems])
    off = np.r_[0, np.cumsum([len(p[0]) for p in problems])]
    n = len(P)
    return T.MatchedBatch(pt_off=off, ls_off=np.zeros(len(problems) + 1, np.int64), pt_P=P, pt_pl_obs=obs,
                          pt_sigma2=np.ones(n), ls_sP=np.zeros((0, 3)), ls_eP=np.zeros((0, 3)), ls_le_obs=np.zeros((0, 3)),
                          ls_spl=np.zeros((0, 2)), ls_epl=np.zeros((0, 2)), ls_sigma2=np.zeros(0))


# (seed, width [px], depth [m], u0 [px]): kappa(H at the prior) 4e13 .. 9e13, Cholesky pivots <= 1e-13 max diag
API_PROBLEMS = [(3, 1.4, 1.0, 300.0), (5, 1.4, 1.0, 450.0), (7, 1.4, 1.0, 300.0), (3, 1.2, 1.0, 450.0)]


def test_both_solvers_through_the_qr_on_refused_normal_equations(tmp_path, engine, oracle):
    """Points-only problems on a 1.2-1.4 px patch at 1 m: H at the prior has kappa 1e13 .. 1e14, its Cholesky pivots fall
    below 1e-13 max diag (10x inside the fast path's 1e-12 refusal; the device refuses each) and the QR keeps full rank.  So
    stage 1's Gauss-Newton steps are warp_qr6_solve<false> solves, and its DT_cov comes from warp_inv6; 1 / lambda_min(H) > 1
    fails the isGoodSolution gate, so the robust fallback runs (removeOutliers is not reached: no problem with lambda_min(H)
    < 1 passes that gate, and the inlier flags stay the input's).  Its H has log|det| between -50 and -80, so the QR's
    log|det| < 0 stops it at its first iteration with good = false and the start pose.  K2 and the streamed solver, each
    pinned in a subprocess, give the oracle's status, verdict, flags, err_norm and iteration counts (stage 1's count follows
    the QR's increments through the stop rules), and its DT_opt exactly."""
    cfg, cam = T.kitti_config(), T.kitti_camera()
    cfg.has_lines = 0
    problems = [_patch_problem(s, 60, w, d, u0) for s, w, d, u0 in API_PROBLEMS]
    m = _points_batch(problems)
    B = len(problems)
    Hs = []
    for p in range(B):
        H, g, _ = oracle.optimize_functions(cam, cfg, m, p, np.eye(4))
        assert 1e13 <= HP.kappa(H) <= 1e14, p
        assert min(HP.chol_pivots(H)) <= 1e-13 * np.diag(H).max(), p
        perm, diag, maxpivot = HP.qr_pivots(H)
        assert min(abs(d) for d in diag) >= 4 * maxpivot * (HP.EPS * 6.0), p
        assert float(HP.eigvals(H)[0]) < 1.0, p
        Hs.append(H)
    ph = engine.debug_pose_helpers(H=np.stack(Hs), g=np.zeros((B, 6)))
    assert not ph["chol_ok"].any()
    _, res_o, ip_o, il_o = oracle.optimize_pose(cam, cfg, m)
    assert (res_o["status"] == T.ST_ROBUST_FALLBACK).all() and not res_o["good"].any() and ip_o.all()
    assert (res_o["iters_stage1"] >= 2).all() and (res_o["iters_stage2"] == 1).all()
    for p in range(B):
        Hr, _, _ = oracle.optimize_functions(cam, cfg, m, p, np.eye(4), robust=True)
        _, lad = HP.chol_solve(Hr, np.ones(6))
        _, bl = HP.solve_bounds(Hr, np.ones(6))
        assert lad < -(bl + 10.0), (p, lad, bl)          # the sign the robust loop stops on, far outside the QR's bound
    for s in ("0", "1"):
        got = _pinned(tmp_path, s, [("opt", cam, cfg, m, None)])[0]
        np.testing.assert_array_equal(got["inlier_pt"], ip_o)
        for p in range(B):
            g_, o_ = got["results"][p], res_o[p]
            for key in ("status", "good", "iters_stage1", "iters_stage2"):
                assert g_[key] == o_[key], (s, p, key, g_[key], o_[key])
            assert abs(g_["err_norm"] - o_["err_norm"]) <= 1e-9 * abs(o_["err_norm"]), (s, p, g_["err_norm"], o_["err_norm"])
            np.testing.assert_array_equal(g_["DT_opt"], o_["DT_opt"])
