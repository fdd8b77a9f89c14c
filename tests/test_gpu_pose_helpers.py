"""The device helpers both pose solvers decide and finish a problem with (solve.cu: warp_chol6_solve, chol6_solve_regs,
cov_surely_inside_unit, warp_is_good_solution, inverse_se3 / expmap_se3 / logmap_se3, finalize_pose), run through the
plstvo_debug_pose_helpers hook on inputs placed at their branch points, against the 60-digit restatement in hp_pose.py
(pinned to the oracle and the reference by test_hp_pose_host.py) and the oracle.  Every case checks that its edge is hit."""
import mpmath as mp
import numpy as np
import pytest

import hp_pose as HP

pytestmark = pytest.mark.gpu
E12 = 1e-12


def _spd(rng, lam):
    q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    A = (q * np.asarray(lam, np.float64)) @ q.T
    return 0.5 * (A + A.T)


def _run(engine, **inputs):
    return engine.debug_pose_helpers(**inputs)


def _check_solves(out, H, g):
    """x and lad of the Cholesky within their bounds where it accepts; the register copy and the lad-free call byte-identical."""
    for k in range(len(H)):
        assert out["chol_ok"][k] == out["chol0_ok"][k] == out["regs_ok"][k], k
        assert out["chol_x"][k].tobytes() == out["chol0_x"][k].tobytes() == out["regs_x"][k].tobytes(), k
        if out["chol_ok"][k]:
            x, lad = HP.chol_solve(H[k], g[k])
            bx, bl = HP.solve_bounds(H[k], x)
            assert np.abs(out["chol_x"][k] - x).max() <= bx, (k, np.abs(out["chol_x"][k] - x).max(), bx)
            assert abs(out["chol_lad"][k] - float(lad)) <= bl + HP.C_SOLVE * HP.EPS * abs(float(lad)), (k, out["chol_lad"][k], lad)


def _ok_rule(H):
    """warp_chol6_solve's acceptance on a DIAGONAL H, where the pivots are the diagonal entries exactly."""
    d = np.diag(H)
    dmax = max(float(np.max(d)), 0.0) if not np.any(np.isnan(d)) else np.nan
    if not (dmax > 0.0 and dmax < 1e300):
        return False
    return bool(np.all(d > dmax * 1e-12))


def test_cholesky_random_spd_across_conditioning(engine):
    rng = np.random.default_rng(11)
    H, g = [], []
    for e in range(12):
        for _ in range(4):
            H.append(_spd(rng, np.geomspace(1.0, 10.0 ** e, 6) * 10.0 ** rng.integers(-6, 7)))
            g.append(rng.normal(size=6))
    H, g = np.stack(H), np.stack(g)
    out = _run(engine, H=H, g=g)
    assert out["chol_ok"][:40].all()          # kappa <= 1e9: the fast path is taken
    _check_solves(out, H, g)


def test_cholesky_acceptance_flips_where_the_rule_says(engine):
    rng = np.random.default_rng(12)
    H, want = [], []
    for dmax in (1.0, 3.7e5, 2.0 ** -70):
        thr = dmax * 1e-12
        for small in (thr * (1 - 2.0 ** -40), thr, thr * (1 + 2.0 ** -40)):
            for pos in range(6):
                d = rng.uniform(0.5, 1.0, 6) * dmax
                d[(pos + 1) % 6] = dmax
                d[pos] = small
                D = np.diag(d)
                p = rng.permutation(6)
                H.append(D)                         # diagonal
                H.append(D[p][:, p])                # permuted diagonal: still diagonal, the small pivot moves
    # dmax at and above 1e300, zero, negative and NaN diagonals
    H += [np.eye(6) * 1e300, np.eye(6) * np.nextafter(1e300, 0), np.eye(6) * 1.7e308, np.zeros((6, 6)),
          np.diag([1.0, 1, 1, -1e-3, 1, 1]), -np.eye(6), np.diag([1.0, 1, np.nan, 1, 1, 1]), np.diag([np.nan] + [1.0] * 5)]
    H = np.stack(H)
    want = [_ok_rule(h) for h in H]
    assert any(want) and not all(want)
    g = np.ones((len(H), 6))
    out = _run(engine, H=H, g=g)
    np.testing.assert_array_equal(out["chol_ok"], want)
    _check_solves(out, H, g)
    # the boundary is resolved to 2^-40 relative: both verdicts occur at every dmax
    assert out["chol_ok"][:-8].any() and not out["chol_ok"][:-8].all()


def test_cholesky_log_det_through_rescaling_and_its_sign(engine):
    rng = np.random.default_rng(13)
    H = []
    for scale in (1e60, 1e-60, 1e95, 1e-95):            # pivot products leave [1e-100, 1e100] several times
        d = scale * rng.uniform(1.0, 1e3, 6)
        H.append(np.diag(d))
        H.append(_spd(rng, d))
    n_big = len(H)
    targets = []
    for sgn in (1.0, -1.0):                              # log|det H| placed at +-1e-12
        for _ in range(4):
            a = float(mp.expm1(mp.mpf(sgn * E12)))
            H.append(np.diag([1.0 + a, 1, 1, 1, 1, 1]))
            H.append(_spd(rng, [1.0 + a, 2.0, 0.5, 4.0, 0.25, 1.0]))
            targets += [sgn * E12, sgn * E12]
    H = np.stack(H)
    g = rng.normal(size=(len(H), 6))
    out = _run(engine, H=H, g=g)
    assert out["chol_ok"].all()
    _check_solves(out, H, g)
    for k, t in enumerate(targets):
        k += n_big
        _, lad = HP.chol_solve(H[k], g[k])
        _, bl = HP.solve_bounds(H[k], g[k])
        assert abs(float(lad) - t) <= 0.5 * E12 and abs(float(lad)) > bl, (k, lad)   # placed, and outside the bound
        assert np.sign(out["chol_lad"][k]) == np.sign(float(lad)) == np.sign(out["qr_lad"][k]), (k, out["chol_lad"][k], lad)


def _verdicts(engine, oracle, cov, err=None, DT=None):
    n = len(cov)
    err = np.full(n, 0.2) if err is None else np.asarray(err, np.float64)
    DT = np.tile(np.eye(4), (n, 1, 1)) if DT is None else DT
    out = _run(engine, cov=cov, err=err, DT=DT)
    np.testing.assert_array_equal(out["good_fast"], out["good_full"])
    orc = [oracle.is_good_solution(DT[k], cov[k], err[k]) for k in range(n)]
    np.testing.assert_array_equal(out["good_full"], orc)
    return out


def test_is_good_solution_at_the_eigenvalue_thresholds(engine, oracle):
    rng = np.random.default_rng(21)
    cov, placed = [], []
    for cl in range(1, 7):                               # clusters of 1 to 6 equal eigenvalues at the threshold
        for side in (-1.0, 1.0):
            for at_top in ((True, False) if cl < 6 else (True,)):
                lam = rng.uniform(0.1, 0.9, 6)
                if at_top:
                    lam[:cl] = 1.0 + side * E12 * 2.5
                else:
                    lam[:cl] = side * E12 * 2.5
                A = _spd(rng, lam)
                cov.append(A)
                placed.append(at_top)
    cov = np.stack(cov)
    out = _verdicts(engine, oracle, cov)
    hit = [0, 0]
    for k, A in enumerate(cov):
        w = HP.eigvals(A)
        b = HP.eig_bound(A)
        edge = float(w[-1] - 1) if placed[k] else float(w[0])
        assert E12 <= abs(edge) <= 4 * E12 * max(1.0, np.linalg.norm(A)), (k, edge)      # placed, outside the eigenvalue bound
        assert b < E12
        want = HP.is_good(np.eye(4), A, 0.2)
        assert out["good_full"][k] == want, (k, edge, out["eig"][k])
        hit[want] += 1
        np.testing.assert_array_less(np.abs(out["eig"][k] - [float(v) for v in w]), b)   # the Jacobi stop rule's error
    assert hit[0] and hit[1]


def test_is_good_solution_shortcut_trace_err_dt_and_upper_triangle(engine, oracle):
    rng = np.random.default_rng(22)
    cov, err, DT, surely = [], [], [], []
    base = np.diag([0.25, 0.125, 0.0625, 0.3125, 0.125, 0.125])   # trace exactly 1
    for f in (1.0, 1 - 2.0 ** -53, 1 - 2.0 ** -52, 1 + 2.0 ** -52):
        cov.append(base * f)
    for f in (1 - 2.0 ** -40, 1.0, 1 + 2.0 ** -40):   # the shortcut's pivot test at 1e-10 * dmax
        d = np.array([0.4, 0.1, 0.05, 0.02, 0.01, 0.4 * 1e-10 * f])
        cov.append(np.diag(d))
    A = _spd(rng, [0.1, 0.2, 0.05, 0.01, 0.3, 0.02])
    cov.append(A)
    G = A.copy()
    iu = np.triu_indices(6, 1)
    G[iu] = rng.normal(size=len(iu[0])) * 10
    cov.append(G)                                     # garbage in the upper triangle: only the lower one is read
    G = A.copy()
    G[iu] = np.nan
    cov.append(G)
    n0 = len(cov)
    for e in (1.0, np.nextafter(1.0, 2), np.nextafter(1.0, 0), 0.0, -0.0, -5e-324, np.nan, np.inf, -np.inf):
        cov.append(A)
        err.append(e)
    n1 = len(cov)
    for i in range(16):
        for bad in (np.nan, np.inf, -np.inf):
            D = np.eye(4)
            D[i // 4, i % 4] = bad
            DT.append(D)
            cov.append(A)
    cov = np.stack(cov)
    err = np.array([0.2] * n0 + err + [0.2] * (len(cov) - n1))
    DTs = np.stack([np.eye(4)] * n1 + DT)
    out = _verdicts(engine, oracle, cov, err, DTs)
    for k in range(len(cov)):
        assert out["good_full"][k] == HP.is_good(DTs[k], cov[k], err[k]), k
    # the shortcut decides exactly where its rule says: trace < 1 (summed in index order) and every pivot > 1e-10 max(diag)
    for k in range(7):
        d = np.diag(cov[k])
        tr = 0.0
        for v in d:
            tr += v
        assert out["surely"][k] == (tr < 1.0 and bool(np.all(d > 1e-10 * d.max()))), k
    assert not out["surely"][0] and out["surely"][1] and not out["surely"][3]
    assert list(out["surely"][4:7]) == [False, False, True]
    assert out["surely"][7] and out["surely"][8] and out["surely"][9]
    np.testing.assert_array_equal(out["eig"][8], out["eig"][7])
    np.testing.assert_array_equal(out["eig"][9], out["eig"][7])
    assert list(out["good_full"][n0:n1]) == [True, False, True, True, True, False, True, False, False]
    assert not out["good_full"][n1:].any()


def test_is_good_solution_on_nan_covariances_follows_the_oracle(engine, oracle):
    """A NaN off-diagonal entry: the device and the oracle both stop the Jacobi iteration at once and read the diagonal,
    which can be finite; so the verdict is the diagonal's (DESIGN.md §3 says what Eigen would do)."""
    cov = []
    for diag in ([0.1] * 6, [0.1, 0.1, 1.5, 0.1, 0.1, 0.1], [0.1, -0.2, 0.1, 0.1, 0.1, 0.1]):
        for (i, j) in ((1, 0), (5, 4), (5, 0)):
            A = np.diag(diag)
            A[i, j] = np.nan
            cov.append(A)
    A = np.diag([0.1] * 6)
    A[2, 2] = np.nan
    cov.append(A)
    cov = np.stack(cov)
    out = _verdicts(engine, oracle, cov)
    assert list(out["good_full"]) == [True] * 3 + [False] * 3 + [False] * 3 + [True]
    assert not out["surely"].any()


def test_expmap_at_its_branch_point(engine):
    rng = np.random.default_rng(31)
    e6 = 0.000001
    mags = [np.nextafter(np.nextafter(e6, 0), 0), np.nextafter(e6, 0), e6, np.nextafter(e6, 1), np.nextafter(np.nextafter(e6, 1), 1),
            0.0, 1e-8, 1e-3, 1.0, np.pi - 1e-6, np.pi]
    xi = []
    for m in mags:
        for axis in range(3):
            for sgn in (1.0, -1.0):
                x = np.concatenate([rng.uniform(-1e3, 1e3, 3), np.zeros(3)])
                x[3 + axis] = sgn * m                    # one axis: |w| is exactly m, the branch is placed exactly
                xi.append(x)
    xi = np.stack(xi)
    out = _run(engine, xi=xi)
    for k, x in enumerate(xi):
        want = HP.tonp(HP.expmap(x))
        assert np.abs(out["exp"][k] - want).max() <= HP.exp_bound(x), (k, x, np.abs(out["exp"][k] - want).max())
        m = np.abs(x[3:]).max()
        assert np.array_equal(out["exp"][k][:3, :3], np.eye(3)) == (m < e6), (k, m)


def test_logmap_and_inverse_at_their_edges(engine, oracle):
    cases = HP.log_cases(32)
    # theta just above and below logmap's 1e-6 on the fp64 cosine grid: rotations about z with exact cos / sin entries
    c6 = float(mp.cos(mp.mpf("1e-6")))
    for c in (np.nextafter(np.nextafter(c6, 0), 0), np.nextafter(c6, 0), c6, np.nextafter(c6, 2), np.nextafter(np.nextafter(c6, 2), 2)):
        T = np.eye(4)
        s = float(mp.sqrt(1 - mp.mpf(c) ** 2))
        T[:2, :2] = [[c, -s], [s, c]]
        T[:3, 3] = [700.0, -300.0, 20.0]
        cases.append(T)
    Ts = np.stack(cases)
    out = _run(engine, T=Ts)
    n_nan = 0
    edge = {True: 0, False: 0}
    for k, T in enumerate(Ts):
        got = out["log"][k]
        HP.check_log(got, T, k)
        o = oracle.logmap_se3(T)
        np.testing.assert_array_equal(np.isnan(got), np.isnan(o))       # where cos rounds to -1: the oracle's NaN / inf pattern
        np.testing.assert_array_equal(np.isinf(got), np.isinf(o))
        n_nan += HP.cosine(T) == -1.0
        th = float(mp.acos(mp.mpf(HP.cosine(T))))
        if 0.9e-6 < th < 1.1e-6:
            edge[th > 1e-6] += 1
            assert np.any(got[3:] != 0) == (th > 1e-6), (k, th, got)   # logmap's branch, as the rule says
        Ti = out["inv"][k]
        np.testing.assert_array_equal(Ti[:3, :3], T[:3, :3].T)
        assert np.abs(Ti[:3, 3] + T[:3, :3].T @ T[:3, 3]).max() <= 8 * HP.EPS * np.abs(T[:3, 3]).sum()
    assert n_nan > 0 and edge[True] and edge[False], (n_nan, edge)


def test_pose_finalisation_with_a_half_turn_heading(engine, oracle):
    """finalize_pose on a prior frame whose heading is pi - delta (large translation, anisotropic Tfw_cov): Tfw within the logmap
    bound of the restatement on the returned DT, Tfw_cov within its componentwise bound, eigenvalues and verdict."""
    rng = np.random.default_rng(41)
    DT, cov, Tp, Tcp = [], [], [], []
    for d in HP.HALF_TURN:
        for _ in range(3):
            D = HP.rodrigues(mp.mpf(rng.uniform(0.01, 0.2)), rng.normal(size=3), rng.uniform(-1.0, 1.0, 3))
            # Tfw_prev = (heading pi - delta) DT_opt, so that Tfw = Tfw_prev DT_opt^-1 has the heading pi - delta
            Tp.append(HP.rodrigues(mp.pi - d, [0.02, 1.0, 0.03] + rng.normal(0, 0.01, 3), rng.uniform(-1e3, 1e3, 3)) @ D)
            DT.append(D)
            J = rng.normal(size=(30, 6)) * np.array([30, 30, 30, 300, 300, 300])
            cov.append(np.linalg.inv(J.T @ J))
            Tcp.append(np.diag([1e-2, 4e-2, 1e-3, 1e-5, 3e-5, 2e-6]) + 1e-7 * np.ones((6, 6)))
    DT, cov, Tp, Tcp = map(np.stack, (DT, cov, Tp, Tcp))
    err = np.full(len(DT), 0.3)
    out = _run(engine, DT=DT, cov=cov, err=err, Tfw_prev=Tp, Tfw_cov_prev=Tcp)
    assert out["fin_good"].all()
    near_pi = singular = 0
    for k in range(len(DT)):
        Ti = np.eye(4)
        Ti[:3, :3] = DT[k][:3, :3].T
        Ti[:3, 3] = -DT[k][:3, :3].T @ DT[k][:3, 3]
        x = HP.logmap(Ti)
        want_dt = HP.tonp(HP.expmap(x))
        bw, bt = HP.log_bounds(Ti)
        assert np.abs(out["fin_DT"][k] - want_dt).max() <= bw + bt + HP.exp_bound([float(v) for v in x]), k
        want, b = HP.tfw(Tp[k], out["fin_DT"][k])
        near_pi += HP.cosine(Tp[k] @ out["fin_DT"][k]) < -0.99
        if want is None or b > 1.0:   # the product's cosine is -1 or within a few eps of it: no claim on the value (the exact
            singular += want is None  # half turns below check the NaN pattern where the product is known exactly)
        else:
            assert np.abs(out["fin_Tfw"][k] - want).max() <= b, (k, np.abs(out["fin_Tfw"][k] - want).max(), b)
        wc, bc = HP.unccomp(Tp[k], Tcp[k], cov[k])
        assert np.all(np.abs(out["fin_Tfw_cov"][k] - wc) <= bc), (k, np.max(np.abs(out["fin_Tfw_cov"][k] - wc) / bc))
        np.testing.assert_allclose(out["fin_Tfw_cov"][k], wc, rtol=1e-12, atol=1e-12 * np.abs(wc).max())
        np.testing.assert_array_less(np.abs(out["fin_eig"][k] - [float(v) for v in HP.eigvals(cov[k])]), HP.eig_bound(cov[k]))
        assert out["fin_err"][k] == 0.3
    assert near_pi == len(DT) and singular > 0


def test_pose_finalisation_at_an_exact_half_turn(engine, oracle):
    """Inputs whose product is a half turn to the last bit: DT is a quarter turn about a coordinate axis and Tfw_prev a
    three-quarter turn about the same axis (entries 0 and +-1), so inverse_se3 is exact, exp(log(.)) returns the quarter turn up
    to 1.1e-16 off the axis, and the product's entries are those entries permuted: the finalisation's cosine is exactly -1 and
    the reference's formula divides by sine = 0.  Tfw must carry the oracle's NaN / inf pattern on the same
    product; Tfw_cov is unaffected."""
    Rz = np.array([[0.0, -1, 0], [1, 0, 0], [0, 0, 1]])
    Rx = np.array([[1.0, 0, 0], [0, 0, -1], [0, 1, 0]])
    DT, Tp = [], []
    for R3, t in ((Rz, [0.5, -0.25, 1.0]), (Rx, [0.0, 0.0, 0.0]), (Rz.T, [300.0, 2.0, -7.0])):
        D = np.eye(4)
        D[:3, :3], D[:3, 3] = R3, t
        P = np.eye(4)
        P[:3, :3], P[:3, 3] = R3 @ R3 @ R3, [120.0, -900.0, 35.0]    # R^3 R^T = R^2: a half turn
        DT.append(D)
        Tp.append(P)
    DT, Tp = np.stack(DT), np.stack(Tp)
    cov = np.tile(np.diag([1e-4, 2e-4, 3e-4, 1e-6, 2e-6, 3e-6]), (len(DT), 1, 1))
    Tcp = np.tile(np.diag([1e-2, 4e-2, 1e-3, 1e-5, 3e-5, 2e-6]), (len(DT), 1, 1))
    out = _run(engine, DT=DT, cov=cov, err=np.full(len(DT), 0.3), Tfw_prev=Tp, Tfw_cov_prev=Tcp)
    assert out["fin_good"].all()
    for k in range(len(DT)):
        Dinv = np.eye(4)
        Dinv[:3, :3] = DT[k][:3, :3].T
        Dinv[:3, 3] = -DT[k][:3, :3].T @ DT[k][:3, 3]
        np.testing.assert_allclose(out["fin_DT"][k][:3, :3], Dinv[:3, :3], rtol=0, atol=4 * HP.EPS)
        P = Tp[k] @ out["fin_DT"][k]
        assert HP.cosine(P) == -1.0 and HP.logmap(P) is None
        want = oracle.expmap_se3(oracle.logmap_se3(P))
        got = out["fin_Tfw"][k]
        assert not np.all(np.isfinite(got))
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_array_equal(np.isinf(got), np.isinf(want))
        wc, bc = HP.unccomp(Tp[k], Tcp[k], cov[k])
        assert np.all(np.abs(out["fin_Tfw_cov"][k] - wc) <= bc), k


def test_pose_finalisation_rejects(engine):
    """finalize_pose's rejecting branch (:382-390): an identity DT, a covariance outside (0, 1), an err outside [0, 1] and a
    non-finite DT give DT = I, DT_cov = 0, err_norm = -1, Tfw and Tfw_cov = the previous frame's, eigenvalues 0."""
    rng = np.random.default_rng(42)
    good_cov = np.diag([1e-4, 2e-4, 3e-4, 1e-6, 2e-6, 3e-6])
    D = HP.rodrigues(mp.mpf("0.05"), [0.1, 1.0, 0.2], [0.1, 0.0, 0.8])
    bad_D = D.copy()
    bad_D[1, 3] = np.nan
    cases = [(np.eye(4), good_cov, 0.3), (D, good_cov - np.diag([0, 0, 0, 0, 0, 1e-5]), 0.3),
             (D, good_cov + np.diag([0, 0, 1.0, 0, 0, 0]), 0.3), (D, good_cov, 1.5), (D, good_cov, -1e-300), (bad_D, good_cov, 0.3),
             (D, good_cov, 0.3)]
    DT, cov, err = (np.stack([c[i] for c in cases]) for i in range(3))
    Tp = np.stack([HP.rodrigues(mp.pi - mp.mpf("1e-3"), rng.normal(size=3), rng.uniform(-1e3, 1e3, 3)) for _ in cases])
    Tcp = np.stack([np.diag(rng.uniform(1e-6, 1e-1, 6)) for _ in cases])
    out = _run(engine, DT=DT, cov=cov, err=err, Tfw_prev=Tp, Tfw_cov_prev=Tcp)
    assert list(out["fin_good"]) == [False] * 6 + [True]
    for k in range(6):
        np.testing.assert_array_equal(out["fin_DT"][k], np.eye(4))
        np.testing.assert_array_equal(out["fin_Tfw"][k], Tp[k])
        np.testing.assert_array_equal(out["fin_Tfw_cov"][k], Tcp[k])
        np.testing.assert_array_equal(out["fin_eig"][k], np.zeros(6))
        assert out["fin_err"][k] == -1.0
