"""High-precision restatement of the helpers both pose solvers decide and finish a problem with: the 6x6 Cholesky solve and
log|det|, the column-pivoted QR that solves where the Cholesky refuses (ColPivHouseholderQR::solve and logAbsDeterminant,
src/stereoFrameHandler.cpp:417-418, :453-455), the inverse that gives DT_cov (Matrix6d::inverse, :429, :470), the symmetric
eigenvalues and isGoodSolution (src/stereoFrameHandler.cpp:292-305), expmap_se3 / logmap_se3 as the
reference writes them (src/auxiliar.cpp:113-173), and the pose finalisation's Tfw and Tfw_cov (:372-378, src/auxiliar.cpp:
175-197).  Everything is evaluated with mpmath at 60 digits on the exact fp64 inputs, so the only error left in a
comparison is the fp64 implementation's, and each quantity comes with the bound an fp64 evaluation is held to.

The bounds (eps = 2^-52):
  Cholesky x:        |dx| <= C_SOLVE * kappa(H) * eps * |x|          (backward-stable solve; kappa in the 2-norm)
  log|det H|:        |dlad| <= C_SOLVE * kappa(H) * eps              (tr(H^-1 dH) with |dH| <= c eps |H|)
  eigenvalues:       |dlambda| <= C_EIG * eps * |A|_F                 (Weyl; the Jacobi stop rule must stay inside it)
  logmap_se3 w:      |dw| <= C_LOG * eps * (1 + theta / (1 - cos^2))  (sine = sqrt(1 - cos^2) from the trace: near theta = 0
                                                                        and theta = pi its relative error is eps / sin^2)
  logmap_se3 t:      |dt| <= (1 + |t|) * that bound
  expmap_se3:        |dT| <= C_LOG * eps * (1 + |t| (1 + 1 / theta)) (V's (1 - cos theta) / theta cancels)
  Tfw_cov:           componentwise C_SOLVE * eps * (|Tfw_cov_prev| + |Ad| |cov| |Ad|^T)
  QR x, backward:    |H x - g| <= C_SOLVE * eps * (|H|_F |x| + |g|)      (Householder QR is backward stable: the computed x
                                                                        solves (H + dH) x = g + dg with |dH| <= c eps |H|_F,
                                                                        |dg| <= c eps |g|, whatever kappa; the residual is
                                                                        formed here at 60 digits.  Full rank only)
  QR x, forward:     |dx| <= C_SOLVE * kappa(H) * eps * |x|             (that backward error through H^-1; kappa eps << 1)
  QR log|det|:       as the Cholesky's                                  (the R diagonal of H + dH)
  QR truncated x:    |dz| <= C_SOLVE * eps * k_s * (|z| + |g| / |B| + k_s |r| / |B|),  dx_j = dz_j / |H_j|
                                                                        (rank r: x_S is the least-squares solution of
                                                                        H_S x_S ~ g on the support S, and Householder QR's
                                                                        backward error is columnwise, |dH_j| <= c eps |H_j|;
                                                                        so the problem is the column-scaled B = H_S / |H_j|,
                                                                        z = |H_j| x_j, k_s = kappa(B), r = g - H_S x_S, and
                                                                        the least-squares perturbation bound applies to it)
  LU inverse:        |H X - I|_F <= C_SOLVE * eps * |H|_F |X|_F           (each column of X solves (H + dH_j) x_j = e_j with
                                                                        |dH_j| <= c eps |L||U|, and partial pivoting keeps
                                                                        |L||U| near |H| for the growth these matrices have)
                     |X - H^-1|_F <= C_SOLVE * kappa(H) * eps * |H^-1|_F  (that residual through H^-1)
The branch points (expmap's theta < 1e-6, logmap's theta > 1e-6) are decided here on the exact theta of expmap's input and
on the fp64 cosine of logmap's; tests that place an input at a branch point place it so that fp64 decides it the same way.
"""
from __future__ import annotations

import mpmath as mp
import numpy as np

mp.mp.dps = 60
EPS = 2.0 ** -52
C_SOLVE, C_EIG, C_LOG = 64.0, 64.0, 64.0
EDGE = mp.mpf(0.000001)        # the fp64 literal both SE(3) branches compare theta with


def mpm(A) -> mp.matrix:
    A = np.asarray(A, np.float64)
    return mp.matrix([[mp.mpf(float(v)) for v in row] for row in A])


def tonp(M) -> np.ndarray:
    return np.array([[float(M[i, j]) for j in range(M.cols)] for i in range(M.rows)])


# ---------------------------------------------------------------------------------------------------------------------
# 6x6: Cholesky solve, log|det|, eigenvalues, isGoodSolution
# ---------------------------------------------------------------------------------------------------------------------
def eigvals(A) -> list:
    """Ascending eigenvalues of the symmetric matrix whose LOWER triangle is A's (what SelfAdjointEigenSolver reads)."""
    A = np.asarray(A, np.float64)
    L = np.tril(A) + np.tril(A, -1).T
    return sorted(mp.eigsy(mpm(L), eigvals_only=True))


def kappa(H) -> float:
    w = eigvals(H)
    return float(abs(w[-1]) / abs(w[0])) if w[0] != 0 else float("inf")


def chol_solve(H, g):
    """x = H^-1 g and log|det H| of the symmetric H (lower triangle read), at 60 digits."""
    Hm = mpm(np.tril(H) + np.tril(H, -1).T)
    x = mp.lu_solve(Hm, mp.matrix([mp.mpf(float(v)) for v in np.asarray(g, np.float64)]))
    lad = mp.log(abs(mp.det(Hm)))
    return np.array([float(v) for v in x]), lad


def solve_bounds(H, x):
    """(|dx| bound per entry, |dlad| bound) of an fp64 Cholesky on H."""
    k = kappa(H)
    return C_SOLVE * k * EPS * max(np.abs(x).max(), 1e-300), C_SOLVE * k * EPS


def eig_bound(A) -> float:
    A = np.asarray(A, np.float64)
    return C_EIG * EPS * float(np.linalg.norm(np.tril(A) + np.tril(A, -1).T))


def is_good(DT, cov, err) -> bool:
    """isGoodSolution on exact eigenvalues (a NaN err passes, as in the reference: both comparisons are false).  Only
    meaningful for finite cov (see DESIGN.md §3 for NaN covariances)."""
    w = eigvals(cov)
    DT = np.asarray(DT, np.float64)
    finite = bool(np.all(np.isfinite(DT)))
    return not (w[0] < 0 or w[-1] > 1 or err < 0.0 or err > 1.0 or not finite)


def verdict_margin(cov) -> float:
    """Distance of the exact eigenvalues from isGoodSolution's thresholds (lambda_min = 0, lambda_max = 1)."""
    w = eigvals(cov)
    return float(min(abs(w[0]), abs(w[-1] - 1)))


def chol_pivots(H) -> list:
    """The exact pivots of the symmetric H's Cholesky (lower triangle read), in index order, negative ones included."""
    A = mpm(np.tril(H) + np.tril(H, -1).T)
    piv = []
    for k in range(6):
        d = A[k, k]
        piv.append(float(d))
        for i in range(k + 1, 6):
            for j in range(k + 1, 6):
                A[i, j] -= A[i, k] * A[k, j] / d if d != 0 else 0
    return piv


def cond(H) -> float:
    """2-norm condition number of the (not necessarily symmetric) H: the singular values from H^T H at 60 digits."""
    M = mpm(H)
    s = sorted(mp.eigsy(M.T * M, eigvals_only=True))
    return float(mp.sqrt(s[-1] / s[0])) if s[0] > 0 else float("inf")


def qr_pivots(H):
    """The exact column-pivoted Householder QR of H (all of it read, as the solvers do): (pivot order, diagonal of R in pivot
    order, maxpivot = max |R_kk|).  The pivot is the remaining column with the largest norm below row k, the first one on
    ties, as on the device and in orc_qr6_solve."""
    A = mpm(H)
    perm = list(range(6))
    diag = []
    for k in range(6):
        norms = [mp.fsum(A[i, j] ** 2 for i in range(k, 6)) for j in range(6)]
        best = k
        for j in range(k + 1, 6):
            if norms[j] > norms[best]:
                best = j
        if best != k:
            for i in range(6):
                A[i, k], A[i, best] = A[i, best], A[i, k]
            perm[k], perm[best] = perm[best], perm[k]
        c0, nrm = A[k, k], mp.sqrt(norms[best])
        if nrm == 0:
            diag.append(mp.mpf(0))
            continue
        beta = -nrm if c0 >= 0 else nrm
        v = [mp.mpf(0)] * 6
        v[k] = c0 - beta
        for i in range(k + 1, 6):
            v[i] = A[i, k]
        vv = mp.fsum(t * t for t in v)
        for j in range(k, 6):
            s = mp.fsum(v[i] * A[i, j] for i in range(k, 6)) * 2 / vv
            for i in range(k, 6):
                A[i, j] -= s * v[i]
        diag.append(A[k, k])
    return perm, [float(d) for d in diag], float(max(abs(d) for d in diag))


def qr_rank(H):
    """(rank, support) of the truncated solve: the R diagonal above fl(maxpivot * 6 eps), the first `rank` pivots."""
    perm, diag, maxpivot = qr_pivots(H)
    thr = maxpivot * (EPS * 6.0)
    rank = sum(abs(d) > thr for d in diag)
    return rank, sorted(perm[:rank])


def basic_solve(H, g, support) -> np.ndarray:
    """The truncated solution a rank-r column-pivoted solve returns: the least-squares solution of H[:, S] x_S ~ g on the
    support S, zeros off it (60 digits, normal equations)."""
    S = list(support)
    x = np.zeros(6)
    if not S:
        return x
    Hs = mpm(np.asarray(H, np.float64)[:, S])
    gm = mp.matrix([mp.mpf(float(v)) for v in np.asarray(g, np.float64)])
    xs = mp.lu_solve(Hs.T * Hs, Hs.T * gm)
    for i, j in enumerate(S):
        x[j] = float(xs[i])
    return x


def residual(H, g, x) -> float:
    """|H x - g| formed at 60 digits on the fp64 x."""
    r = mpm(H) * mp.matrix([mp.mpf(float(v)) for v in x]) - mp.matrix([mp.mpf(float(v)) for v in g])
    return float(mp.norm(r))


def qr_bounds(H, g, x):
    """(backward bound on |H x - g|, forward bound on |dx|, bound on |dlad|) of an fp64 column-pivoted QR at full rank."""
    H, g = np.asarray(H, np.float64), np.asarray(g, np.float64)
    k = cond(H)
    nx = float(np.linalg.norm(x))
    return (C_SOLVE * EPS * (float(np.linalg.norm(H)) * nx + float(np.linalg.norm(g))), C_SOLVE * k * EPS * nx,
            C_SOLVE * k * EPS)


def basic_bound(H, g, support) -> np.ndarray:
    """Per-entry bound on the truncated solve's x (zeros off the support): see the docstring's QR truncated x."""
    H, g = np.asarray(H, np.float64), np.asarray(g, np.float64)
    S = list(support)
    out = np.zeros(6)
    if not S:
        return out
    x = basic_solve(H, g, S)
    cn = np.linalg.norm(H[:, S], axis=0)
    B = mpm(H[:, S] / cn)
    s = sorted(mp.eigsy(B.T * B, eigvals_only=True))
    nB, ks = float(mp.sqrt(s[-1])), float(mp.sqrt(s[-1] / s[0]))
    z = float(np.linalg.norm(cn * x[S]))
    r = residual(H, g, x)
    dz = C_SOLVE * EPS * ks * (z + float(np.linalg.norm(g)) / nB + ks * r / nB)
    out[S] = dz / cn
    return out


def inv(H) -> np.ndarray:
    """H^-1 at 60 digits, rounded."""
    return tonp(mp.inverse(mpm(H)))


def inv_errors(H, X):
    """(|H X - I|_F at 60 digits, its bound, |X - H^-1|_F, its bound) of an fp64 inverse X of H."""
    Hm = mpm(H)
    res = float(mp.mnorm(Hm * mpm(X) - mp.eye(6), "f"))
    Hi = mp.inverse(Hm)
    fwd = float(mp.mnorm(mpm(X) - Hi, "f"))
    nH, nX, nHi = (float(mp.mnorm(M, "f")) for M in (Hm, mpm(X), Hi))
    return res, C_SOLVE * EPS * nH * nX, fwd, C_SOLVE * cond(H) * EPS * nHi


# ---------------------------------------------------------------------------------------------------------------------
# SE(3), src/auxiliar.cpp:29-62, :113-197
# ---------------------------------------------------------------------------------------------------------------------
def _skew(w):
    return mp.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])


def expmap(x):
    """expmap_se3 of x = [t; w] (exact arithmetic, same branch rule) -> 4x4 mp.matrix."""
    x = [mp.mpf(float(v)) for v in np.asarray(x, np.float64)] if not isinstance(x[0], mp.mpf) else list(x)
    t, w = mp.matrix(x[:3]), x[3:]
    theta = mp.sqrt(w[0] ** 2 + w[1] ** 2 + w[2] ** 2)
    R = mp.eye(3)
    if not theta < EDGE:
        s = _skew(w) / theta
        R = mp.eye(3) + s * mp.sin(theta) + s * s * (1 - mp.cos(theta))
        V = mp.eye(3) + s * (1 - mp.cos(theta)) / theta + s * s * (theta - mp.sin(theta)) / theta
        t = V * t
    T = mp.eye(4)
    for i in range(3):
        for j in range(3):
            T[i, j] = R[i, j]
        T[i, 3] = t[i]
    return T


def cosine(T) -> float:
    """cos(theta) = (trace(R) - 1) / 2, clamped to [-1, 1], as fp64 evaluates it: three additions and a halving, which every
    implementation rounds the same way (nothing in it can be contracted).  Where it rounds to -1, sine = 0 below."""
    T = np.asarray(T, np.float64)
    c = (T[0, 0] + T[1, 1] + T[2, 2] - 1.0) / 2.0
    return min(max(float(c), -1.0), 1.0)


def logmap(T):
    """logmap_se3 of the fp64 T -> list of 6 mpf, or None where the formula divides by sine = 0 (theta = pi): there every
    fp64 evaluation gives NaN / inf.  The cosine is the fp64 one (see cosine()); everything after it is exact."""
    T = np.asarray(T, np.float64)
    c = mp.mpf(cosine(T))
    T = mpm(T)
    sine = min(mp.sqrt(1 - c * c), mp.mpf(1))
    theta = mp.acos(c)
    w = [mp.mpf(0)] * 3
    V = mp.eye(3)
    if theta > EDGE:
        if sine == 0:
            return None
        f = theta / (2 * sine)
        w = [f * (T[2, 1] - T[1, 2]), f * (T[0, 2] - T[2, 0]), f * (T[1, 0] - T[0, 1])]
        s = _skew(w) / theta
        V = mp.eye(3) + s * (1 - c) / theta + s * s * (theta - sine) / theta
    t = mp.inverse(V) * mp.matrix([T[0, 3], T[1, 3], T[2, 3]])
    return [t[0], t[1], t[2]] + w


def log_bounds(T):
    """(bound on |dw|, bound on |dt|) of an fp64 logmap_se3 of T."""
    T = np.asarray(T, np.float64)
    c = cosine(T)
    theta = float(np.arccos(c))
    s2 = 1.0 - c * c
    bw = C_LOG * EPS * (1.0 + (theta / s2 if s2 > 0 else np.inf))
    return bw, bw * (1.0 + float(np.abs(T[:3, 3]).max()))


def exp_bound(x) -> float:
    """Bound on each entry of an fp64 expmap_se3(x): V's (1 - cos theta) / theta loses eps / theta to cancellation."""
    x = np.asarray(x, np.float64)
    theta = float(np.linalg.norm(x[3:]))
    return C_LOG * EPS * (1.0 + float(np.abs(x[:3]).max()) * (1.0 + (1.0 / theta if theta >= 1e-6 else 0.0)))


def tfw(Tfw_prev, DT):
    """Tfw = expmap(logmap(Tfw_prev DT)) (:377) -> (4x4 float array or None, bound per entry).  The product is rounded to fp64
    before the logmap; the rounding moves the cosine by a few eps, which the logmap bound covers (d theta = d cos / sin)."""
    P = tonp(mpm(Tfw_prev) * mpm(DT))
    x = logmap(P)
    if x is None:
        return None, np.inf
    bw, bt = log_bounds(P)
    tn = max(abs(float(v)) for v in x[:3])
    return tonp(expmap(x)), bw + bt + bw * tn + exp_bound([float(v) for v in x])


def adjoint(T):
    T = mpm(T) if not isinstance(T, mp.matrix) else T
    R = T[0:3, 0:3]
    SR = _skew([T[0, 3], T[1, 3], T[2, 3]]) * R
    Ad = mp.zeros(6, 6)
    for i in range(3):
        for j in range(3):
            Ad[i, j] = R[i, j]
            Ad[i, j + 3] = SR[i, j]
            Ad[i + 3, j + 3] = R[i, j]
    return Ad


def unccomp(T1, cov1, covinc):
    """unccomp_se3 (src/auxiliar.cpp:192-197): cov1 + Ad(T1) covinc Ad(T1)^T -> (6x6 float array, componentwise bound)."""
    Ad = adjoint(T1)
    out = mpm(cov1) + Ad * mpm(covinc) * Ad.T
    absAd = np.abs(tonp(Ad))
    scale = np.abs(np.asarray(cov1, np.float64)) + absAd @ np.abs(np.asarray(covinc, np.float64)) @ absAd.T
    return tonp(out), C_SOLVE * EPS * scale


def rodrigues(theta, axis, t) -> np.ndarray:
    """The fp64 rounding of the exact rigid motion of rotation angle theta (mpf) about axis, translation t."""
    a = [mp.mpf(float(v)) for v in axis]
    n = mp.sqrt(a[0] ** 2 + a[1] ** 2 + a[2] ** 2)
    K = _skew([v / n for v in a])
    R = mp.eye(3) + K * mp.sin(theta) + K * K * (1 - mp.cos(theta))
    T = np.eye(4)
    T[:3, :3] = tonp(R)
    T[:3, 3] = np.asarray(t, np.float64)
    return T


# ---------------------------------------------------------------------------------------------------------------------
# cases shared by the host and the GPU tests
# ---------------------------------------------------------------------------------------------------------------------
HALF_TURN = [mp.mpf("1e-2"), mp.mpf("1e-4"), mp.mpf("1e-6"), mp.mpf("1e-8"), mp.mpf(0)]


def log_cases(seed):
    """fp64 rigid motions at the logmap's edges: theta in {0, 1e-8, ~1e-6, 1e-3, 1, pi - delta, pi}, random axes, translations up
    to 1e3 m."""
    rng = np.random.default_rng(seed)
    thetas = [mp.mpf(0), mp.mpf("1e-8"), mp.mpf("1e-6") * (1 - mp.mpf("1e-4")), mp.mpf("1e-6") * (1 + mp.mpf("1e-4")),
              mp.mpf("1e-3"), mp.mpf(1)] + [mp.pi - d for d in HALF_TURN]
    out = []
    for th in thetas:
        for _ in range(3):
            out.append(rodrigues(th, rng.normal(size=3), rng.uniform(-1e3, 1e3, 3)))
    return out


def check_log(got, T, what):
    """An fp64 logmap_se3(T) within log_bounds of the restatement, or not finite where the fp64 cosine is -1."""
    x = logmap(T)
    if x is None:   # the cosine rounds to -1: the formula divides by sine = 0
        assert cosine(T) == -1.0
        assert not np.all(np.isfinite(got)), (what, got)
        return
    bw, bt = log_bounds(T)
    xf = np.array([float(v) for v in x])
    assert np.abs(got[3:] - xf[3:]).max() <= bw, (what, cosine(T), got, xf, bw)
    assert np.abs(got[:3] - xf[:3]).max() <= bt, (what, cosine(T), got, xf, bt)


# ---------------------------------------------------------------------------------------------------------------------
# 6x6 systems for the QR and the inverse, shared by the host and the GPU tests
# ---------------------------------------------------------------------------------------------------------------------
KAPPAS = [1.0, 1e2, 1e4, 1e6, 1e8, 1e10, 1e12, 1e13, 1e14, 1e15]
SCALES = [1e-60, 1.0, 1e60]


def spd(rng, lam) -> np.ndarray:
    q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    A = (q * np.asarray(lam, np.float64)) @ q.T
    return 0.5 * (A + A.T)


def point_normal_equations(rng, n, half_angle, depth, rot_scale) -> np.ndarray:
    """J^T J of n points in a cone of the given half angle at one depth: the projection's Jacobian with respect to [t; w]
    (u = x / z, v = y / z after X + t + w x X), rotation columns times rot_scale.  Small cones make translation and
    rotation barely separable, as on a distant, narrow patch."""
    X = np.c_[rng.uniform(-half_angle, half_angle, (n, 2)) * depth, np.full(n, depth)]
    J = []
    for x, y, z in X:
        Jp = np.array([[1 / z, 0, -x / z ** 2], [0, 1 / z, -y / z ** 2]])
        Sx = np.array([[0, z, -y], [-z, 0, x], [y, -x, 0]])             # d(w x X)/dw = -[X]x
        J.append(np.c_[Jp, rot_scale * Jp @ Sx])
    J = np.vstack(J)
    return J.T @ J


def handover_matrix(rng, kappa, scale) -> np.ndarray:
    """SPD H of condition ~kappa whose weak direction lies near the last coordinate: the Cholesky's last pivot is then
    ~lambda_min, below its 1e-12 * max diag refusal once kappa is a few 1e12."""
    lam = np.r_[np.geomspace(1.0, 0.1, 5), 1.0 / kappa]
    q5, _ = np.linalg.qr(rng.normal(size=(5, 5)))
    Q = np.eye(6)
    Q[:5, :5] = q5
    a = 0.05
    G = np.eye(6)
    G[[4, 4, 5, 5], [4, 5, 4, 5]] = [np.cos(a), -np.sin(a), np.sin(a), np.cos(a)]
    Q = G @ Q
    A = (Q * lam) @ Q.T * scale
    return 0.5 * (A + A.T)


def qr_full_cases(seed):
    """Full-rank systems -> list of (H, g, label): SPD across KAPPAS x SCALES up to kappa 1e14, point normal equations with
    rotation / translation scale disparity, and the Cholesky's hand-over band (kappa 4e12 .. 1e14, weak direction near the
    last coordinate).  At kappa 1e15 the smallest R entry is within a few eps |H| of the rank threshold 6 eps maxpivot, so
    whether the QR keeps full rank is a rounding: such systems belong to neither this family nor rank_cases."""
    rng = np.random.default_rng(seed)
    out = []
    for k in KAPPAS[:-1]:
        for s in SCALES:
            for _ in range(2):
                lam = np.geomspace(1.0, 1.0 / k, 6)
                out.append((spd(rng, rng.permutation(lam) * s), rng.normal(size=6) * s, f"spd k={k:g} s={s:g}"))
    for half, depth, rs in ((0.3, 5.0, 1.0), (0.05, 20.0, 30.0), (0.02, 40.0, 1.0), (0.02, 40.0, 30.0), (0.01, 20.0, 10.0)):
        H = point_normal_equations(rng, 40, half, depth, rs)
        out.append((H, rng.normal(size=6) * np.abs(H).max(), f"points a={half} z={depth} r={rs}"))
    for k in (4e12, 1e13, 3e13, 1e14):
        for s in SCALES:
            out.append((handover_matrix(rng, k, s), rng.normal(size=6) * s, f"handover k={k:g} s={s:g}"))
    return out


def rank_cases(seed):
    """Rank decisions placed where rounding cannot decide them -> list of (H, g, label).  H = P blockdiag(A, D) P^T with A
    a generic SPD block of size r = 0..6 (kappa <= 1e3) and D diagonal, each entry exactly 0 or at thr (1 +- 2^-40),
    thr = fl(maxpivot * 6 eps).  Zero columns stay exactly zero through every Householder step and the D columns are
    orthogonal to A's, so the R diagonal holds |D| to a few eps and exact zeros.  Where A is diagonal with power-of-two
    entries and D has one non-zero entry, every reflection is an exact signed row swap, so that entry is placed at thr and
    one ulp either side.  Generic matrices singular in exact arithmetic are not here: their trailing R entries are
    rounding noise of order eps |H| on either side of 6 eps maxpivot, where the device, the oracle and Eigen may
    legitimately differ."""
    rng = np.random.default_rng(seed)
    out = []
    lo, hi = 1.0 - 2.0 ** -40, 1.0 + 2.0 ** -40
    for s in SCALES:
        for r in range(7):
            for pat in range(2 if 0 < r < 6 else 1):
                M = np.zeros((6, 6))
                if r:
                    M[:r, :r] = spd(rng, np.geomspace(1.0, 1e-3, r) * s)[:r, :r] if r == 6 else \
                        _spd_block(rng, np.geomspace(1.0, 1e-3, r) * s)
                maxpivot = qr_pivots(M)[2]
                thr = maxpivot * (EPS * 6.0)
                for i in range(r, 6):   # alternate the verdicts; pattern 1 shifts them so both occur at every r
                    M[i, i] = [0.0, thr * lo, thr * hi][(i + pat) % 3] * rng.choice([-1.0, 1.0]) if r else 0.0
                p = rng.permutation(6)
                out.append((M[p][:, p], rng.normal(size=6) * s, f"generic r={r} s={s:g}"))
    for s in (2.0 ** -200, 1.0, 2.0 ** 200):
        for r in (1, 3, 5):
            for f in ("at", "below", "above", "lo", "hi"):
                d = np.zeros(6)
                d[:r] = s * 2.0 ** rng.integers(-8, 9, r).astype(float) * rng.choice([-1.0, 1.0], r)
                thr = float(np.abs(d).max()) * (EPS * 6.0)
                d[r] = {"at": thr, "below": np.nextafter(thr, 0), "above": np.nextafter(thr, np.inf), "lo": thr * lo,
                        "hi": thr * hi}[f] * rng.choice([-1.0, 1.0])
                p = rng.permutation(6)
                M = np.diag(d)
                out.append((M[p][:, p], rng.normal(size=6) * s, f"exact r={r} {f} s={s:g}"))
    return out


def _spd_block(rng, lam) -> np.ndarray:
    r = len(lam)
    q, _ = np.linalg.qr(rng.normal(size=(r, r)))
    A = (q * np.asarray(lam, np.float64)) @ q.T
    return 0.5 * (A + A.T)


def inv_cases(seed):
    """Inverse inputs -> list of (H, label): SPD across KAPPAS x SCALES, non-symmetric matrices with prescribed singular
    values, pivot columns with tied magnitudes (+-equal entries: every pivot choice among them must meet the bounds), and the
    hand-over band."""
    rng = np.random.default_rng(seed)
    out = []
    for k in KAPPAS:
        for s in SCALES:
            out.append((spd(rng, rng.permutation(np.geomspace(1.0, 1.0 / k, 6)) * s), f"spd k={k:g} s={s:g}"))
    for k in (1.0, 1e3, 1e6, 1e9, 1e12):
        for s in SCALES:
            U, _ = np.linalg.qr(rng.normal(size=(6, 6)))
            V, _ = np.linalg.qr(rng.normal(size=(6, 6)))
            out.append(((U * np.geomspace(1.0, 1.0 / k, 6)) @ V.T * s, f"nonsym k={k:g} s={s:g}"))
    for s in SCALES:
        for col in range(3):
            M = rng.normal(size=(6, 6))
            M[:, col] = rng.choice([-1.0, 1.0], 6) * 2.0          # every candidate of the first pivot search ties
            M[col, :] += rng.normal(size=6) * 1e-3
            M[:, col] = rng.choice([-1.0, 1.0], 6) * 2.0
            out.append((M * s, f"tied col={col} s={s:g}"))
        T = np.array([[1.0, 1, 0, 0, 0, 0], [-1, 1, 0, 0, 0, 0], [0, 0, 1, -1, 0, 0], [0, 0, 1, 1, 0, 0],
                      [0, 0, 0, 0, 3, 3], [0, 0, 0, 0, -3, 3]])      # ties at every step
        out.append((T * s, f"tied all s={s:g}"))
    for k in (4e12, 1e13, 1e14):
        out.append((handover_matrix(rng, k, 1.0), f"handover k={k:g}"))
    return out
