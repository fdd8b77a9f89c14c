"""High-precision restatement of the helpers both pose solvers decide and finish a problem with: the 6x6 Cholesky solve and
log|det|, the symmetric eigenvalues and isGoodSolution (src/stereoFrameHandler.cpp:292-305), expmap_se3 / logmap_se3 as the
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
