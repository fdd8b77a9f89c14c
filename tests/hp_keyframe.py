"""High-precision restatement of the key-frame test (StereoFrameHandler::needNewKF and currFrameIsKF,
src/stereoFrameHandler.cpp:1136-1218), with the bound each fp64 quantity is held to, and the placed cases the host and the
GPU tests share.  Everything after the fp64 inputs is evaluated with mpmath at 60 digits (hp_pose's precision); logmap_se3
reuses hp_pose.logmap, whose cosine is the fp64 one every implementation rounds the same way.

What is restated, per step:
  entropy_first_prevKF  K + log(det DT_cov) / 2 where prev_f_iskf (det 0: -999999999.99), K = 3 (1 + log 2 pi) exactly;
  t, r                  |logmap(inverse(Tfw) T_prevKF)| of the translation and (in degrees) of the rotation;
  cov_prevKF_currF      += Ad(T_prevKF) Ad(inverse(DT)) DT_cov Ad(inverse(DT))^T Ad(T_prevKF)^T, exact on the fp64 inputs;
  entropy_curr, ratio   K + log(det cov) / 2, and entropy_curr / entropy_first_prevKF;
  the decision          ratio < min_entropy_ratio, ratio NaN or inf, DT_cov == 0 and DT == I, t > max_kf_t_dist,
                        r > max_kf_r_dist, N_prevKF_currF > 10; then the counter, and currFrameIsKF where it fires.

The bounds (eps = 2^-52, C = hp_pose.C_SOLVE = 64):
  t, r:        hp_pose.log_bounds of the product P (its w bound bw, its per-entry t bound bt): |dt| <= sqrt(3) bt and
               |dr| <= sqrt(3) bw 180 / pi, plus C eps (1 + |t_Tfw| + |t_prevKF|) for the rounding of P's translation and
               4 eps |t|, 4 eps |r| for the norm.  Where P's fp64 cosine is exactly 1 (theta = 0: V = I, w = 0) and t is
               formed without rounding (every square, sum and the root exact), the bound of t is 0 and r is exactly 0.
  cov:         componentwise C eps (|cov_prev| + |Ad_k| |Ad_i| |DT_cov| |Ad_i|^T |Ad_k|^T), |Ad| with |skew(t)| |R| in its
               corner (DESIGN.md holds Tfw_cov to the same form), summed over the steps since the key frame.
  entropy:     log det moves by tr(C^-1 dC) to first order, so |de| <= 1/2 sum_ij |C^-1|_ji (dcov_ij + C eps |C_ij|) (the
               accumulated cov error plus the LU's backward error, |dC| <= c eps |L||U|, taken as C eps |C| for the growth
               partial pivoting has on these matrices), plus 8 eps (|K| + |log det| / 2) for log and the sum.  Only while the
               first-order term is below 1/8; beyond it nothing is asserted.
  ratio:       |d(a / b)| <= (|da| + |a / b| |db|) / |b| + 2 eps |a / b|, first order while |db| < |b| / 2: it grows as 1 / b,
               so near entropy_first_prevKF = 0 the band widens and exact decisions are asserted less often.
  decision:    each criterion is decided where the exact value lies outside its band (value +- bound strictly on one side of
               the threshold); the decision is exact where one decided criterion fires, or where all are decided and none
               does.  Inside a band no implementation's decision is asserted.

Non-finite inputs, and determinants that an fp64 LU overflows or underflows, are artefacts of fp64: there the 60-digit values
say nothing about what the reference computes, and run() stops (the tests take the reference library's fp64 result as the
answer instead).  Exactly singular covariances are restated only where the singularity is structural (a zero row or
column in a product whose every term is an exact zero), since only there every fp64 LU gives exactly +-0.
"""
from __future__ import annotations

import math

import mpmath as mp
import numpy as np

import hp_pose as hp

mp.mp.dps = 60
EPS = hp.EPS
C = hp.C_SOLVE
K_ENTROPY = 3 * (1 + mp.log(2 * mp.pi))
FIRST_ZERO = -999999999.99
DEG = 180 / mp.pi


def _absad(T):
    """|Ad(T)| with the corner as |skew(t)| |R| (the bound of fp64's skew(t) R, not its value)."""
    T = np.asarray(T, np.float64)
    R, t = np.abs(T[:3, :3]), np.abs(T[:3, 3])
    S = np.array([[0, t[2], t[1]], [t[2], 0, t[0]], [t[1], t[0], 0]])
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = R
    A[:3, 3:] = S @ R
    return A


def _inverse(T):
    """inverse_se3 exactly: [R^T, -R^T t] as a 4x4 mp.matrix."""
    M = hp.mpm(T)
    out = mp.eye(4)
    for i in range(3):
        for j in range(3):
            out[i, j] = M[j, i]
        out[i, 3] = -mp.fsum(M[k, i] * M[k, 3] for k in range(3))
    return out


def _structurally_singular(cov, scale) -> bool:
    """A zero row or column whose every term is an exact zero (scale row / column 0): every fp64 LU gives det = +-0."""
    z = (scale == 0) & (cov == 0)
    return bool(z.all(axis=1).any() or z.all(axis=0).any())


def entropy(cov, dcov):
    """(entropy as mpf, or -inf / nan as float where the determinant is structurally 0 / surely negative, its bound) of an fp64
    evaluation of K + log(det cov) / 2, cov known to within dcov componentwise.  (None, inf) where undecidable: the
    first-order bound is too large, or det overflows / underflows fp64."""
    cov = np.asarray(cov, np.float64)
    if _structurally_singular(cov, dcov):
        return -math.inf, 0.0
    M = hp.mpm(cov)
    d = mp.det(M)
    if d == 0:
        return None, math.inf
    Ci = hp.tonp(mp.inverse(M))
    first = 0.5 * float(np.sum(np.abs(Ci.T) * (dcov + C * EPS * np.abs(cov))))
    if not first < 0.125:
        return None, math.inf
    if not 1e-300 < abs(d) < 1e300:
        return None, math.inf
    if d < 0:
        return math.nan, 0.0
    e = K_ENTROPY + mp.log(d) / 2
    return e, first + 8 * EPS * (float(K_ENTROPY) + abs(float(mp.log(d))) / 2)


def _side(v, b, th):
    """True / False where v (exact) +- b lies strictly above / at-or-below th; None inside the band."""
    if isinstance(v, float) and math.isnan(v):
        return False
    v = mp.mpf(v) if not isinstance(v, mp.mpf) else v
    if v - b > th:
        return True
    if v + b <= th and not (b > 0 and v + b == th):
        return False
    return None


def step(kcfg, s, Tfw, DT, DT_cov):
    """One needNewKF (+ currFrameIsKF) at 60 digits from the exact state s (dict; updated in place).  Returns a dict of the
    exact values (floats), their bounds, and `fire` (True / False, or None where a band decides), or None where an input or
    an intermediate is an fp64 artefact."""
    min_ratio, max_t, max_r = (float(v) for v in kcfg)
    Tfw, DT, DT_cov = (np.asarray(a, np.float64).reshape(n, n) for a, n in ((Tfw, 4), (DT, 4), (DT_cov, 6)))
    if not (np.isfinite(Tfw).all() and np.isfinite(DT).all() and np.isfinite(DT_cov).all()):
        return None
    out = {}
    if s["prev_f_iskf"]:                                             # :1140-1153
        e, b = entropy(DT_cov, np.zeros((6, 6)))
        if e is None:
            return None
        if isinstance(e, float) and e == -math.inf:
            s["e_first"], s["b_first"] = mp.mpf(FIRST_ZERO), 0.0
        else:
            s["e_first"], s["b_first"] = e, b
        s["prev_f_iskf"] = False
    # :1156-1159
    P = hp.tonp(_inverse(Tfw) * hp.mpm(s["T_prevKF"]))
    x = hp.logmap(P)
    if x is None:
        return None
    tn = mp.sqrt(x[0] ** 2 + x[1] ** 2 + x[2] ** 2)
    rn = mp.sqrt(x[3] ** 2 + x[4] ** 2 + x[5] ** 2) * DEG
    scale = 1.0 + float(np.abs(Tfw[:3, 3]).max()) + float(np.abs(np.asarray(s["T_prevKF"])[:3, 3]).max())
    if hp.cosine(P) == 1.0:
        # R = I and T_prevKF = I: every implementation forms P exactly; then t is exact where its squares, sums and root are
        tf = [float(v) for v in x[:3]]
        t64 = math.sqrt((tf[0] * tf[0] + tf[1] * tf[1]) + tf[2] * tf[2])
        exact = (np.array_equal(Tfw[:3, :3], np.eye(3)) and np.array_equal(s["T_prevKF"], np.eye(4))
                 and all(mp.mpf(v) ** 2 == mp.mpf(v * v) for v in tf) and mp.mpf(float(tn ** 2)) == tn ** 2
                 and mp.mpf(t64) == tn)
        bt = 0.0 if exact else C * EPS * scale + 8 * EPS * float(tn)
        br = 0.0
    else:
        bw, btl = hp.log_bounds(P)
        bt = math.sqrt(3) * btl + C * EPS * scale + 4 * EPS * float(tn)
        br = math.sqrt(3) * bw * float(DEG) + 4 * EPS * float(rn)
    # :1162-1164
    DTi = _inverse(DT)
    Ai, Ak = hp.adjoint(DTi), hp.adjoint(s["T_prevKF"])
    add = Ak * (Ai * hp.mpm(DT_cov) * Ai.T) * Ak.T
    aAi, aAk = _absad(hp.tonp(DTi)), _absad(s["T_prevKF"])
    s["b_cov"] = s["b_cov"] + C * EPS * (np.abs(hp.tonp(s["cov"])) + aAk @ aAi @ np.abs(DT_cov) @ aAi.T @ aAk.T)
    s["cov"] = s["cov"] + add
    cov64 = hp.tonp(s["cov"])
    e, be = entropy(cov64, s["b_cov"])
    if e is None or not np.isfinite(s["b_cov"]).all():
        return None
    ef, bf = s["e_first"], s["b_first"]
    if isinstance(ef, float) and math.isnan(ef):
        ratio, bq = math.nan, 0.0
    elif isinstance(e, float):                                       # -inf or NaN: exact in every implementation
        with np.errstate(all="ignore"):
            ratio, bq = float(np.float64(e) / np.float64(float(ef))), 0.0
    else:
        if not bf < abs(float(ef)) / 2:
            return None
        q = e / ef
        ratio, bq = q, (be + abs(float(q)) * bf) / abs(float(ef)) + 2 * EPS * abs(float(q))
    # :1173-1175
    if isinstance(ratio, float) and not math.isfinite(ratio):
        c_ratio = True
    else:
        below = _side(-ratio, bq, -min_ratio)                         # ratio < min  <=>  -ratio > -min
        c_ratio = below
    c_fail = (not DT_cov.any()) and bool(np.array_equal(DT, np.eye(4)))
    c_t = _side(tn, bt, max_t) if max_t != math.inf else False
    c_r = _side(rn, br, max_r) if max_r != math.inf else False
    c_n = s["N"] > 10
    crit = [c_ratio, c_fail, c_t, c_r, c_n]
    fire = True if any(c is True for c in crit) else (False if all(c is False for c in crit) else None)
    out.update(fire=fire, e_first=float(ef) if not isinstance(ef, float) else ef, b_first=bf,
               e_curr=float(e) if not isinstance(e, float) else e, b_e=be,
               ratio=float(ratio) if not isinstance(ratio, float) else ratio, b_ratio=bq,
               t=float(tn), b_t=bt, r=float(rn), b_r=br, cov=cov64, b_cov=s["b_cov"].copy())
    if fire is None:
        return out
    if not fire:
        s["N"] += 1
    out["N"] = s["N"]
    if fire:                                                         # currFrameIsKF (:1189-1218)
        reset(s)
    return out


def state(rec) -> dict:
    """The exact state of one T.KEYFRAME_STATE_DTYPE record."""
    rec = np.asarray(rec).reshape(-1)[0]
    return {"prev_f_iskf": bool(rec["prev_f_iskf"]), "N": int(rec["N_prevKF_currF"]),
            "e_first": mp.mpf(float(rec["entropy_first_prevKF"])), "b_first": 0.0,
            "T_prevKF": np.array(rec["T_prevKF"], np.float64), "cov": hp.mpm(rec["cov_prevKF_currF"]),
            "b_cov": np.zeros((6, 6))}


def reset(s):
    s.update(prev_f_iskf=True, N=0, T_prevKF=np.eye(4), cov=mp.zeros(6, 6), b_cov=np.zeros((6, 6)))


def run(kcfg, rec, steps) -> list:
    """needNewKF over the steps [(Tfw, DT, DT_cov)] from the state record rec: one dict per step (see step()), stopping after
    the first step that is an artefact (None) or whose decision a band decides (the state after it is not known)."""
    s = state(rec)
    out = []
    for Tfw, DT, DT_cov in steps:
        o = step(kcfg, s, Tfw, DT, DT_cov)
        out.append(o)
        if o is None or o["fire"] is None:
            break
    return out


# ---------------------------------------------------------------------------------------------------------------------
# placed cases shared by the host and the GPU tests
# ---------------------------------------------------------------------------------------------------------------------
INF = math.inf


def make_state(prev_f_iskf=1, N=0, e_first=0.0, T_prevKF=None, cov=None):
    from stvo_pl_b200 import types as T
    s = np.zeros(1, T.KEYFRAME_STATE_DTYPE)
    s["prev_f_iskf"], s["N_prevKF_currF"], s["entropy_first_prevKF"] = prev_f_iskf, N, e_first
    s["T_prevKF"][0] = np.eye(4) if T_prevKF is None else T_prevKF
    s["cov_prevKF_currF"][0] = np.zeros((6, 6)) if cov is None else cov
    return s


def _motion(rng, theta, t_scale):
    return hp.rodrigues(mp.mpf(theta), rng.normal(size=3), rng.normal(size=3) * t_scale)


def _place(case, which, sign):
    """The case with its `which` threshold moved to the exact value of its one step -+ 4 bounds: sign +1 places the value
    above the threshold (t, r fire; the ratio does not), -1 below."""
    k, st, steps = case["k"], case["state"], case["steps"]
    o = run(k, st, steps)[-1]
    v, b = {"t": (o["t"], o["b_t"]), "r": (o["r"], o["b_r"]), "ratio": (o["ratio"], o["b_ratio"])}[which]
    th = float(mp.mpf(v) - sign * 4 * mp.mpf(b)) if b > 0 else v
    kk = list(k)
    kk[{"ratio": 0, "t": 1, "r": 2}[which]] = th
    return dict(case, k=tuple(kk), label=f"{case['label']} {which} {'above' if sign > 0 else 'below'}")


def cases(seed=0) -> list:
    """Placed key-frame cases -> list of {label, k (min_entropy_ratio, max_kf_t_dist, max_kf_r_dist), state (one
    KEYFRAME_STATE record), steps [(Tfw, DT, DT_cov)]}."""
    rng = np.random.default_rng(seed)
    cov_good = hp.spd(rng, np.geomspace(1e-4, 1e-6, 6))
    small = _motion(rng, 0.01, 0.05)
    out = []

    def add(label, k, state, steps):
        out.append(dict(label=label, k=tuple(float(v) for v in k), state=state, steps=steps))

    # t at its threshold, exactly: R = I, translation (3, 4, 0) 2^k, so t = 5 2^k in every implementation
    for e in (-3, 0, 4):
        Tfw = np.eye(4)
        Tfw[:3, 3] = np.array([3.0, 4.0, 0.0]) * 2.0 ** e
        t = 5.0 * 2.0 ** e
        for th, lab in ((t, "at"), (np.nextafter(t, 0), "ulp below"), (np.nextafter(t, INF), "ulp above")):
            add(f"t exact 5*2^{e} th {lab}", (-INF, th, INF), make_state(), [(Tfw, small, cov_good)])
    # r exactly 0 (R = I): the strict > at 0 and at the smallest negative threshold
    Tfw = np.eye(4)
    Tfw[:3, 3] = [1.0, 0.0, 0.0]
    add("r exact 0 th 0", (-INF, INF, 0.0), make_state(), [(Tfw, small, cov_good)])
    add("r exact 0 th -tiny", (-INF, INF, -5e-324), make_state(), [(Tfw, small, cov_good)])
    # r and t placed at 4 bounds either side: small angles just above the 1e-6 branch, moderate ones, headings near pi
    for theta in (1.5e-6, 3e-6, 1e-3, 0.3, 2.0, math.pi - 1e-3, math.pi - 1e-5):
        base = dict(label=f"theta {theta:.6g}", k=(-INF, INF, INF), state=make_state(),
                    steps=[(_motion(rng, theta, 2.0), small, cov_good)])
        for sign in (1, -1):
            out.append(_place(base, "r", sign))
            if theta in (1e-3, 0.3, math.pi - 1e-3):
                out.append(_place(base, "t", sign))
    # the same with a previous key frame away from the origin (Ad(T_prevKF) in the covariance, the product in logmap)
    Tk = _motion(rng, 0.5, 3.0)
    base = dict(label="T_prevKF moved", k=(-INF, INF, INF), state=make_state(T_prevKF=Tk),
                steps=[(Tk @ _motion(rng, 0.2, 1.0), small, cov_good)])
    for sign in (1, -1):
        out.append(_place(base, "r", sign))
        out.append(_place(base, "t", sign))
    # the entropy ratio at 4 bounds either side: entropy_first_prevKF positive, negative and near 0; well- and
    # ill-conditioned accumulated covariances
    for kappa in (10.0, 1e10):
        prev = hp.spd(rng, np.geomspace(1e-3, 1e-3 / kappa, 6))
        for ef in (12.0, -30.0, 1e-3, -2e-6):
            base = dict(label=f"ratio kappa {kappa:g} e_first {ef:g}", k=(-INF, INF, INF),
                        state=make_state(0, 3, ef, cov=prev), steps=[(small, small, hp.spd(rng, np.geomspace(1e-5, 1e-7, 6)))])
            for sign in (1, -1):
                out.append(_place(base, "ratio", sign))
    # entropy_first_prevKF from a first step whose det(DT_cov) is near e^(-2K): the ratio is badly conditioned
    for eps_e in (1e-2, -1e-2, 1e-6):
        c = float(mp.exp((-2 * K_ENTROPY + 2 * eps_e) / 6))
        Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
        D = c * (Q @ Q.T)
        base = dict(label=f"ratio first near 0 ({eps_e:g})", k=(-INF, INF, INF), state=make_state(), steps=[(small, small, D)])
        for sign in (1, -1):
            out.append(_place(base, "ratio", sign))
    # a covariance that accumulates over several calls from an ill-conditioned DT_cov: the ratio falls step by step
    # (entropy_first_prevKF < 0), so a threshold placed at the last step leaves the earlier ones quiet
    steps = [(_motion(rng, 0.01 * (i + 1), 0.1 * (i + 1)), _motion(rng, 0.01, 0.05), hp.spd(rng, np.geomspace(1e-4, 1e-14, 6)))
             for i in range(5)]
    acc = dict(label="accumulated kappa 1e10", k=(-INF, INF, INF), state=make_state(), steps=steps)
    last = run(acc["k"], acc["state"], steps)[-1]
    for sign in (1, -1):
        th = float(mp.mpf(last["ratio"]) + sign * 4 * mp.mpf(last["b_ratio"]))
        out.append(dict(acc, k=(th, INF, INF), label=f"accumulated kappa 1e10 ratio {'below' if sign > 0 else 'above'}"))
    # the counter: N = 10 stays quiet and leaves 11, N = 11 fires; 11 quiet steps then a 12th that fires
    q = (-INF, INF, INF)
    add("counter N=10", q, make_state(0, 10, -30.0, cov=cov_good), [(small, small, cov_good)])
    add("counter N=11", q, make_state(0, 11, -30.0, cov=cov_good), [(small, small, cov_good)])
    add("counter chain", q, make_state(), [(_motion(rng, 0.002 * i, 0.01 * i), small, cov_good) for i in range(1, 13)])
    # first step and degenerate covariances
    Z = cov_good.copy()
    Z[2, :] = Z[:, 2] = 0.0
    add("first det 0 (zero row/col)", (0.85, 5.0, 15.0), make_state(), [(small, np.eye(4), Z)])
    add("first det < 0", (0.85, 5.0, 15.0), make_state(), [(small, small, np.diag([1e-4] * 5 + [-1e-4]))])
    S = np.zeros((6, 6))
    S[[0, 3, 5], [0, 2, 5]] = -0.0
    add("first +-0 entries, DT = I", (0.85, 5.0, 15.0), make_state(), [(small, np.eye(4), S)])
    add("failed solve: DT_cov 0, DT = I", (-INF, INF, INF), make_state(0, 2, -30.0, cov=cov_good),
        [(small, np.eye(4), np.zeros((6, 6)))])
    for lab, (i, j), v in (("diag", (0, 0), np.nextafter(1.0, 0)), ("translation", (0, 3), np.nextafter(0.0, 1))):
        D = np.eye(4)
        D[i, j] = v
        add(f"DT_cov 0, DT one ulp off I ({lab})", (-INF, INF, INF), make_state(0, 2, -30.0, cov=cov_good),
            [(small, D, np.zeros((6, 6)))])
    nan_cov = np.full((6, 6), np.nan)
    inf55 = nan_cov.copy()
    inf55[5, 5] = INF
    pivot_inf = np.diag([0.0, INF, 1e-4, 1e-4, 1e-4, 1e-4])
    for lab, D in (("all-NaN DT_cov", nan_cov), ("NaN DT_cov, +inf at (5,5)", inf55), ("zero pivot then inf", pivot_inf)):
        add(f"first {lab}", (0.85, 5.0, 15.0), make_state(), [(small, small, D)])
        add(f"later {lab}", (0.85, 5.0, 15.0), make_state(0, 2, -30.0, cov=cov_good), [(small, small, D)])
    # non-finite Tfw: the patterns optimizePose leaves within ~1.5e-8 rad of a half turn (NaN / inf in R and t), under
    # ordinary thresholds and under a negative max_kf_r_dist (which the reference's r = 0 passes)
    half = np.eye(4)
    half[:3, :] = np.nan
    rot_nan = np.eye(4)
    rot_nan[:3, :3] = np.nan
    rot_nan[:3, 3] = [1.0, 2.0, 3.0]
    infs = np.eye(4)
    infs[0, 0], infs[1, 1] = INF, -INF
    for lab, Tfw in (("NaN R and t", half), ("NaN R", rot_nan), ("+inf -inf on the diagonal", infs)):
        for k in ((0.85, 5.0, 15.0), (-INF, INF, -1.0)):
            add(f"Tfw {lab} max_r {k[2]:g}", k, make_state(0, 2, -30.0, cov=cov_good), [(Tfw, small, cov_good)])
    return out
