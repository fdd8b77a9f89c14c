"""The streamed evaluator's records and per-feature arithmetic (stvo_pl_b200/csrc/gn_stream.cuh), restated in NumPy.

pack_*      the fp32 records as gs_pack_point / gs_pack_line form them (pose-independent parts in fp64, then rounded)
pose32      the pose as the kernel holds it: (R - I | t), rounded to fp32 AFTER the subtraction (gs_pose_entry)
eval_*      optimizeFunctions on those fp32 inputs, every operation in fp64: what gs_point / gs_line would give with exact
            arithmetic.  Besides H (21 upper-triangle entries), g and e, each returns the magnitudes the kernel adds per feature,
            which scale its rounding: the residual's terms (|du0| + |du| for a point, |ds0| + |l . du| for a line), the residual
            norm n, the robust weight's pieces and |J|.  Both sides of the two homogTh switches are returned where asked for.
residual_*  the point residual u(DT) - u_obs in three arithmetics (fp64 truth, the delta form in fp32, the naive fp32 form),
            for the host test of the record format itself.
"""
import numpy as np

f32 = np.float32
EPS32 = 2.0 ** -24          # unit roundoff of fp32


def pose32(DT):
    r = np.asarray(DT, np.float64).reshape(-1, 4, 4)[:, :3, :4].reshape(-1, 12).copy()
    r[:, [0, 5, 10]] -= 1.0
    return r.astype(f32)


def cam32(cam, homog_th):
    fx, fy, h = f32(cam.fx), f32(cam.fy), f32(homog_th)
    return dict(fx=fx, fy=fy, h=h, inv_h=f32(1.0) / h, fx_h=fx / h)


def pack_points(cam, P, obs, s2):
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    xn, yn = x / z, y / z
    A = np.stack([xn, yn, z, np.sqrt(s2)], 1).astype(f32)
    Bv = np.stack([cam.fx * xn + cam.cx - obs[:, 0], cam.fy * yn + cam.cy - obs[:, 1]], 1).astype(f32)
    return A, Bv


def overlap_coeffs(spl, epl):
    """overlap_coeffs (gn_stream.cuh), vectorised; ob = +-inf, oc = -sv for a zero-height segment in the vertical branch."""
    su, sv, eu, ev = spl[:, 0], spl[:, 1], epl[:, 0], epl[:, 1]
    lx, ly = eu - su, ev - sv
    a, b, c = sv - ev, eu - su, su * ev - eu * sv
    with np.errstate(all="ignore"):
        lxy = 1.0 / (a * a + b * b)
        vert, horiz = np.abs(su - eu) < 1.0, np.abs(sv - ev) < 1.0
        ob_v = 1.0 / ly
        oa = np.where(vert, 0.0, np.where(horiz, 1.0 / lx, (b * b * lxy) / lx))
        ob = np.where(vert, ob_v, np.where(horiz, 0.0, (-(a * b) * lxy) / lx))
        oc = np.where(vert, np.where(np.isinf(ob_v), -sv, -sv / ly), np.where(horiz, -su / lx, (-(a * c) * lxy - su) / lx))
    return oa, ob, oc


def pack_lines(cam, sP, eP, le, spl, epl, s2):
    sxn, syn, exn, eyn = sP[:, 0] / sP[:, 2], sP[:, 1] / sP[:, 2], eP[:, 0] / eP[:, 2], eP[:, 1] / eP[:, 2]
    spu, spv = cam.fx * sxn + cam.cx, cam.fy * syn + cam.cy
    epu, epv = cam.fx * exn + cam.cx, cam.fy * eyn + cam.cy
    oa, ob, oc = overlap_coeffs(spl, epl)
    inf = np.isinf(ob)
    with np.errstate(all="ignore"):
        ls0 = np.where(inf, spv + oc, oa * spu + ob * spv + oc)
        le0 = np.where(inf, epv + oc, oa * epu + ob * epv + oc)
    A = np.stack([sxn, syn, sP[:, 2], np.sqrt(s2)], 1).astype(f32)
    Bv = np.stack([exn, eyn, eP[:, 2]], 1).astype(f32)
    C = np.stack([le[:, 0], le[:, 1], le[:, 0] * spu + le[:, 1] * spv + le[:, 2], le[:, 0] * epu + le[:, 1] * epv + le[:, 2]],
                 1).astype(f32)
    D = np.stack([oa, ob, ls0, le0], 1).astype(f32)
    return A, Bv, C, D


def _project(r, c, xn, yn, z):
    """gs_project in fp64 on fp32 inputs; also the scale of the terms the kernel adds to form du, dv"""
    r, xn, yn, z = (np.asarray(v, np.float64) for v in (r, xn, yn, z))
    x, y = xn * z, yn * z
    dd, mag = [], []
    for k in range(3):
        terms = (r[:, 4 * k] * x, r[:, 4 * k + 1] * y, r[:, 4 * k + 2] * z, r[:, 4 * k + 3])
        dd.append(terms[0] + terms[1] + terms[2] + terms[3])
        mag.append(sum(np.abs(q) for q in terms))
    X, Y, Z = x + dd[0], y + dd[1], z + dd[2]
    fx, fy = float(c["fx"]), float(c["fy"])
    du = fx * (dd[0] - xn * dd[2]) / Z
    dv = fy * (dd[1] - yn * dd[2]) / Z
    su = fx * (mag[0] + np.abs(xn) * mag[2]) / np.abs(Z)
    sv = fy * (mag[1] + np.abs(yn) * mag[2]) / np.abs(Z)
    return X, Y, Z, du, dv, su, sv


def _jac(X, Y, Z, dxs, dys):
    t, zz = X * dxs + Y * dys, Z * Z
    return np.stack([dxs * Z, dys * Z, -t, -(Y * t + zz * dys), X * t + zz * dxs, Z * (X * dys - Y * dxs)], 1)


def _fg(c, Z, side):
    """fx / max(homogTh, Z^2); side = None: the fp64 decision, True / False: forced"""
    big = (Z * Z > float(c["h"])) if side is None else np.full(Z.shape, side)
    return np.where(big, float(c["fx"]) / (Z * Z), float(c["fx_h"])), np.abs(Z * Z - float(c["h"]))


def _inv(c, n, side):
    big = (n > float(c["h"])) if side is None else np.full(n.shape, side)
    with np.errstate(divide="ignore"):
        return np.where(big, 1.0 / n, float(c["inv_h"])), np.abs(n - float(c["h"]))


def _acc(J, r, w):
    iu = np.triu_indices(6)
    H = (J[:, :, None] * J[:, None, :] * w[:, None, None])[:, iu[0], iu[1]]
    return H, J * (w * r)[:, None], r * r * w


def eval_points(c, r, A, Bv, fg_side=None, inv_side=None):
    X, Y, Z, du, dv, su, sv = _project(r, c, A[:, 0], A[:, 1], A[:, 2])
    dx, dy = Bv[:, 0].astype(np.float64) + du, Bv[:, 1].astype(np.float64) + dv
    n = np.hypot(dx, dy)
    inv, n_gap = _inv(c, n, inv_side)
    fg, z_gap = _fg(c, Z, fg_side)
    J = _jac(X, Y, Z, fg * inv * dx, fg * inv * dy)
    pss = A[:, 3].astype(np.float64)
    rr = n * pss
    wc = 1.0 / (1.0 + rr * rr)
    H, g, e = _acc(J, rr, wc)
    res = np.maximum(np.abs(Bv[:, 0]) + su, np.abs(Bv[:, 1]) + sv)          # px: the residual's terms
    one, zero = np.ones_like(X), np.zeros_like(X)
    G = np.hypot(np.linalg.norm(_jac(X, Y, Z, one, zero), axis=1), np.linalg.norm(_jac(X, Y, Z, zero, one), axis=1))
    return dict(H=H, g=g, e=e, n=n, r=rr, pss=pss, wc=wc, ov=np.ones_like(n), lam=np.zeros_like(n), res=res,
                J=np.linalg.norm(J, axis=1), Jd=2.0 * fg * inv * G, n_gap=n_gap, z_gap=[z_gap], Z=[Z])


def _lambda(oa, ob, lam0, du, dv):
    with np.errstate(all="ignore"):
        return np.where(np.isinf(ob), ob * (dv + lam0), oa * du + ob * dv + lam0), np.abs(oa * du) + np.abs(ob * dv) + np.abs(lam0)


def _overlap(ls, le):
    lo, hi = np.where(le < ls, le, ls), np.where(ls < le, le, ls)
    ov = np.where(hi > 1.0, 1.0, hi) - np.where(lo < 0.0, 0.0, lo)
    return np.where((hi < 0.0) | (lo > 1.0), 0.0, ov)


def eval_lines(c, r, A, Bv, C, D, fg_side=(None, None), inv_side=None):
    sX, sY, sZ, sdu, sdv, ssu, ssv = _project(r, c, A[:, 0], A[:, 1], A[:, 2])
    eX, eY, eZ, edu, edv, esu, esv = _project(r, c, Bv[:, 0], Bv[:, 1], Bv[:, 2])
    l0, l1, ds0, de0 = (C[:, k].astype(np.float64) for k in range(4))
    ds, de = l0 * sdu + l1 * sdv + ds0, l0 * edu + l1 * edv + de0
    n = np.hypot(ds, de)
    iden, n_gap = _inv(c, n, inv_side)
    fgs, zs_gap = _fg(c, sZ, fg_side[0])
    fge, ze_gap = _fg(c, eZ, fg_side[1])
    ks, ke = fgs * ds * iden, fge * de * iden
    J = _jac(sX, sY, sZ, ks * l0, ks * l1) + _jac(eX, eY, eZ, ke * l0, ke * l1)
    pss = A[:, 3].astype(np.float64)
    rr = n * pss
    wc = 1.0 / (1.0 + rr * rr)
    oa, ob, ls0, le0 = (D[:, k].astype(np.float64) for k in range(4))
    lam_s, ms = _lambda(oa, ob, ls0, sdu, sdv)
    lam_e, me = _lambda(oa, ob, le0, edu, edv)
    ov = _overlap(lam_s, lam_e)
    H, g, e = _acc(J, rr, wc * ov)
    res = np.maximum(np.abs(ds0) + np.abs(l0) * ssu + np.abs(l1) * ssv, np.abs(de0) + np.abs(l0) * esu + np.abs(l1) * esv)
    Gs, Ge = np.linalg.norm(_jac(sX, sY, sZ, l0, l1), axis=1), np.linalg.norm(_jac(eX, eY, eZ, l0, l1), axis=1)
    return dict(H=H, g=g, e=e, n=n, r=rr, pss=pss, wc=wc, ov=ov, lam=np.maximum(ms, me), res=res,
                J=np.linalg.norm(J, axis=1), Jd=2.0 * iden * (fgs * Gs + fge * Ge), n_gap=n_gap, z_gap=[zs_gap, ze_gap],
                Z=[sZ, eZ])


def tolerances(m, K):
    """Per-feature bounds on |H - H64|, |g - g64|, |e - e64| for a kernel whose every fp32 operation rounds within K units of
    the magnitudes it adds (EPS32 each): the residual's terms (m['res']) make an absolute error of the residual; the Jacobian
    moves with it by at most m['Jd'] per px (it is the residual's direction times fg / n and the endpoint Jacobians, whose two
    terms may cancel in a line's), and its own terms are at most m['Jd'] n; the robust weight moves with the residual and the
    overlap with the lambda terms (m['lam']); everything else is relative."""
    eps, J, n, r, pss, wc, ov = K * EPS32, m["J"], m["n"], m["r"], m["pss"], m["wc"], m["ov"]
    dres = eps * m["res"]                                              # px
    dJ = m["Jd"] * (eps * n + dres)                                    # absolute error of J
    dr = pss * dres
    dw = ov * (eps * wc + 2.0 * r * wc * wc * dr) + wc * np.minimum(2.0 * eps * m["lam"], 1.0)   # absolute error of w
    w = wc * ov
    tH = 2.0 * w * J * dJ + J * J * dw + w * dJ * dJ
    tg = w * r * dJ + J * r * dw + J * w * dr
    te = r * r * dw + 2.0 * r * w * dr + eps * r * r * w
    return tH, tg, te


# ---- the point residual in three arithmetics (host test of the record format) ----
def residual_truth(cam, P, obs, DT):
    X = P @ DT[:3, :3].T + DT[:3, 3]
    return np.stack([cam.fx * X[:, 0] / X[:, 2] + cam.cx - obs[:, 0], cam.fy * X[:, 1] / X[:, 2] + cam.cy - obs[:, 1]], 1)


def residual_delta32(cam, P, obs, DT):
    """gs_project + gs_point's residual, every operation rounded to fp32 (separate multiply and add, no FMA)"""
    A, Bv = pack_points(cam, P, obs, np.ones(len(P)))
    r = pose32(DT[None])[0]
    xn, yn, z = A[:, 0], A[:, 1], A[:, 2]
    x, y = xn * z, yn * z
    dd = [r[4 * k] * x + r[4 * k + 1] * y + r[4 * k + 2] * z + r[4 * k + 3] for k in range(3)]
    Z = z + dd[2]
    iz = f32(1.0) / Z
    du = f32(cam.fx) * (dd[0] - xn * dd[2]) * iz
    dv = f32(cam.fy) * (dd[1] - yn * dd[2]) * iz
    return np.stack([Bv[:, 0] + du, Bv[:, 1] + dv], 1).astype(np.float64)


def residual_naive32(cam, P, obs, DT):
    """the same residual formed the direct way in fp32: project through (R | t) and subtract the observation"""
    P32, R32, t32 = P.astype(f32), DT[:3, :3].astype(f32), DT[:3, 3].astype(f32)
    X = [R32[k, 0] * P32[:, 0] + R32[k, 1] * P32[:, 1] + R32[k, 2] * P32[:, 2] + t32[k] for k in range(3)]
    u = f32(cam.fx) * X[0] / X[2] + f32(cam.cx) - obs[:, 0].astype(f32)
    v = f32(cam.fy) * X[1] / X[2] + f32(cam.cy) - obs[:, 1].astype(f32)
    return np.stack([u, v], 1).astype(np.float64)
