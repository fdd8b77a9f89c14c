"""Seeded synthetic frame pairs for the PL-StVO hot path (SURVEY.md section 8(d)).

There are no images and no datasets on the box: the hot path consumes pre-extracted features only
(two N x 32 uint8 descriptor matrices per feature type and per-feature 3-D / 2-D records), so the
generator produces exactly those, shaped like the reference's configurations:

  kitti : 1241 x 376, fx = fy = 718.856 ...   (config/dataset_params/kitti00-02.yaml:2-13)
  euroc : 752 x 480                           (config/dataset_params/euroc_params.yaml:8-11)
  hd    : 1920 x 1080 (assumed roofline camera)

Seeds follow SURVEY 8(d): seed = 20260924 + 1000 * config + pair_index.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Tuple

import numpy as np

from .types import FrameBatch, PlCamera, kitti_camera, euroc_camera, hd_camera

BASE_SEED = 20260924


# ---- SE(3), numpy restatement for the generator (src/auxiliar.cpp:124-141) ---------------------------
def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], dtype=np.float64)


def expmap_se3(x):
    t, w = np.asarray(x[:3], np.float64), np.asarray(x[3:], np.float64)
    theta = np.linalg.norm(w)
    T = np.eye(4)
    if theta < 1e-6:
        T[:3, 3] = t
        return T
    s = skew(w) / theta
    R = np.eye(3) + s * np.sin(theta) + s @ s * (1.0 - np.cos(theta))
    V = np.eye(3) + s * (1.0 - np.cos(theta)) / theta + s @ s * (theta - np.sin(theta)) / theta
    T[:3, :3] = R
    T[:3, 3] = V @ t
    return T


def back_projection(cam: PlCamera, u, v, disp):
    """src/pinholeStereoCamera.cpp:221-229."""
    bd = cam.b / disp
    return np.stack([bd * (u - cam.cx), bd * (v - cam.cy), bd * cam.fx], axis=-1)


def projection(cam: PlCamera, P):
    """src/pinholeStereoCamera.cpp:231-237."""
    return np.stack([cam.cx + cam.fx * P[..., 0] / P[..., 2], cam.cy + cam.fy * P[..., 1] / P[..., 2]], axis=-1)


@dataclass
class Shape:
    """One of the BASELINE.json configurations."""
    name: str
    config_id: int
    camera: str
    n_pt: int
    n_ls: int
    depth: Tuple[float, float]
    t_mean: Tuple[float, float, float]
    t_std: Tuple[float, float, float]
    w_std: float
    pt_levels: int          # ORB pyramid levels (sigma2 = 1.2^(-2 level)); 1 = KITTI (level 0 only)


SHAPES = {
    # C2 / C4: synthetic KITTI-shape 1241x376, 2000 ORB pts + 500 LBD lines (config_kitti.yaml: orb_nlevels 1)
    "kitti": Shape("kitti", 2, "kitti", 2000, 500, (4.0, 80.0), (0, 0, -1.0), (0.02, 0.02, 0.1), 0.003, 1),
    # C1: points-only plumbing (reference CPU-runnable case)
    "kitti_points": Shape("kitti_points", 1, "kitti", 2000, 0, (4.0, 80.0), (0, 0, -1.0), (0.02, 0.02, 0.1), 0.003, 1),
    # C3: EuRoC-shape 752x480, 1000 pts + 300 lines (config_euroc.yaml: orb_nlevels 4)
    "euroc": Shape("euroc", 3, "euroc", 1000, 300, (0.8, 12.0), (0, 0, 0), (0.03, 0.03, 0.03), 0.01, 4),
    # C5: high-density 1920x1080, 8000 pts + 2000 lines
    "hd": Shape("hd", 5, "hd", 8000, 2000, (1.0, 40.0), (0, 0, -0.3), (0.02, 0.02, 0.05), 0.003, 1),
}


def camera_for(name: str) -> PlCamera:
    return {"kitti": kitti_camera, "euroc": euroc_camera, "hd": hd_camera}[name]()


def _descriptors(rng, n, tie_stress):
    if tie_stress:  # each byte from {0x00, 0xFF}: massive distance ties
        return (rng.integers(0, 2, size=(n, 32), dtype=np.uint8) * 255).astype(np.uint8)
    return rng.integers(0, 256, size=(n, 32), dtype=np.uint8)


def _flip_bits(rng, desc, p, tie_stress):
    if tie_stress:  # flip whole bytes with probability p
        m = rng.random(desc.shape) < p
        return np.where(m, desc ^ np.uint8(255), desc).astype(np.uint8)
    thr = int(round(p * 256))
    mask = np.zeros(desc.shape, np.uint8)
    for b in range(8):
        mask |= ((rng.integers(0, 256, size=desc.shape, dtype=np.uint8) < thr).astype(np.uint8) << b).astype(np.uint8)
    return desc ^ mask


def _line_eq(s, e):
    """le = (s x e) / sqrt(a^2 + b^2) with homogeneous endpoints (src/stereoFrame.cpp:356-358)."""
    sh = np.concatenate([s, np.ones((len(s), 1))], axis=1)
    eh = np.concatenate([e, np.ones((len(e), 1))], axis=1)
    l = np.cross(sh, eh)
    return l / np.sqrt(l[:, 0:1] ** 2 + l[:, 1:2] ** 2)


def make_pair(shape: Shape, pair_index: int, *, n_pt=None, n_ls=None, overlap=0.7, bitflip=0.10,
              noise_px=0.5, outlier_frac=0.10, tie_stress=False, seed_offset=0, motion=None):
    """One (prev, curr) frame pair + ground-truth motion.  Returns (prev, curr, T_gt) with prev / curr dicts
    of per-frame arrays.  `overlap` = fraction of curr rows that are noisy copies of a distinct prev row.  `motion` (optional,
    4x4): the ground-truth motion to use instead of the drawn one (the rest of the pair is drawn as without it)."""
    cam = camera_for(shape.camera)
    n_pt = shape.n_pt if n_pt is None else n_pt
    n_ls = shape.n_ls if n_ls is None else n_ls
    rng = np.random.default_rng(BASE_SEED + 1000 * shape.config_id + pair_index + seed_offset)
    W, H = cam.width, cam.height
    xi = np.concatenate([rng.normal(shape.t_mean, shape.t_std), rng.normal(0.0, shape.w_std, 3)])
    T_gt = expmap_se3(xi) if motion is None else np.asarray(motion, np.float64)  # prev-camera -> curr-camera (P' = R P + t, :567)

    def depths(n):
        lo, hi = shape.depth
        return np.exp(rng.uniform(np.log(lo), np.log(hi), n))

    def sigma2_levels(n):
        if shape.pt_levels <= 1:
            return np.ones(n), np.zeros(n, np.int32)
        lev = rng.integers(0, shape.pt_levels, n).astype(np.int32)
        s = 1.2 ** lev.astype(np.float64)  # PointFeature ctor (src/stereoFeatures.cpp:41-47)
        return 1.0 / (s * s), lev

    def fresh_points(n):
        u, v, z = rng.uniform(0, W, n), rng.uniform(0, H, n), depths(n)
        d = np.maximum(cam.b * cam.fx / z, 1.0)  # min_disp (src/config.cpp:59)
        s2, _ = sigma2_levels(n)
        return dict(pl=np.stack([u, v], 1), P=back_projection(cam, u, v, d), sigma2=s2)

    def fresh_lines(n):
        u, v, z = rng.uniform(0, W, n), rng.uniform(0, H, n), depths(n)
        length, ang = rng.uniform(30, 150, n), rng.uniform(0.2, np.pi - 0.2, n)
        s = np.stack([u, v], 1)
        e = s + np.stack([length * np.cos(ang), length * np.sin(ang)], 1)
        ze = z * rng.uniform(0.85, 1.15, n)
        ds, de = np.maximum(cam.b * cam.fx / z, 1.0), np.maximum(cam.b * cam.fx / ze, 1.0)
        return dict(spl=s, epl=e, sP=back_projection(cam, s[:, 0], s[:, 1], ds),
                    eP=back_projection(cam, e[:, 0], e[:, 1], de), le=_line_eq(s, e),
                    sigma2=np.ones(n), level=np.zeros(n, np.int32))

    def tf(P):
        return P @ T_gt[:3, :3].T + T_gt[:3, 3]

    # ---- points ----
    prev_pt = fresh_points(n_pt)
    prev_pt["desc"] = _descriptors(rng, n_pt, tie_stress)
    curr_pt = fresh_points(n_pt)
    curr_pt["desc"] = _descriptors(rng, n_pt, tie_stress)
    k = int(round(overlap * n_pt))
    src = rng.permutation(n_pt)[:k]           # prev rows that reappear
    dst = rng.permutation(n_pt)[:k]           # curr rows they land on (random order)
    obs = projection(cam, tf(prev_pt["P"][src])) + rng.normal(0, noise_px, (k, 2))
    out = rng.random(k) < outlier_frac
    obs[out] = np.stack([rng.uniform(0, W, out.sum()), rng.uniform(0, H, out.sum())], 1)
    curr_pt["pl"][dst] = obs
    curr_pt["desc"][dst] = _flip_bits(rng, prev_pt["desc"][src], bitflip, tie_stress)

    # ---- lines ----
    prev_ls = fresh_lines(n_ls)
    prev_ls["desc"] = _descriptors(rng, n_ls, tie_stress)
    curr_ls = fresh_lines(n_ls)
    curr_ls["desc"] = _descriptors(rng, n_ls, tie_stress)
    k = int(round(overlap * n_ls))
    src = rng.permutation(n_ls)[:k]
    dst = rng.permutation(n_ls)[:k]
    if k:
        s_obs = projection(cam, tf(prev_ls["sP"][src])) + rng.normal(0, noise_px, (k, 2))
        e_obs = projection(cam, tf(prev_ls["eP"][src])) + rng.normal(0, noise_px, (k, 2))
        out = rng.random(k) < outlier_frac
        no = int(out.sum())
        s_obs[out] = np.stack([rng.uniform(0, W, no), rng.uniform(0, H, no)], 1)
        e_obs[out] = s_obs[out] + np.stack([rng.uniform(30, 150, no), rng.uniform(30, 150, no)], 1)
        curr_ls["spl"][dst], curr_ls["epl"][dst] = s_obs, e_obs
        curr_ls["le"][dst] = _line_eq(s_obs, e_obs)
        curr_ls["desc"][dst] = _flip_bits(rng, prev_ls["desc"][src], bitflip, tie_stress)
    return dict(pt=prev_pt, ls=prev_ls), dict(pt=curr_pt, ls=curr_ls), T_gt


def _stack(frames) -> FrameBatch:
    pt_off = np.concatenate([[0], np.cumsum([len(f["pt"]["desc"]) for f in frames])])
    ls_off = np.concatenate([[0], np.cumsum([len(f["ls"]["desc"]) for f in frames])])
    cp = lambda key, w: np.concatenate([f["pt"][key].reshape(-1, w) if w > 1 else f["pt"][key] for f in frames])
    cl = lambda key, w: np.concatenate([f["ls"][key].reshape(-1, w) if w > 1 else f["ls"][key] for f in frames])
    return FrameBatch(pt_off=pt_off, ls_off=ls_off, pdesc=cp("desc", 32), ldesc=cl("desc", 32),
                      pt_P=cp("P", 3), pt_pl=cp("pl", 2), pt_sigma2=cp("sigma2", 1),
                      ls_sP=cl("sP", 3), ls_eP=cl("eP", 3), ls_le=cl("le", 3), ls_spl=cl("spl", 2),
                      ls_epl=cl("epl", 2), ls_sigma2=cl("sigma2", 1), ls_level=cl("level", 1))


def make_batch(shape_name: str, B: int, *, first_pair: int = 0, **kw):
    """B independent (prev, curr) pairs of one configuration.  Returns (prev, curr, T_gt[B,4,4], camera)."""
    shape = SHAPES[shape_name]
    prevs, currs, Ts = [], [], []
    for i in range(B):
        p, c, T = make_pair(shape, first_pair + i, **kw)
        prevs.append(p); currs.append(c); Ts.append(T)
    return _stack(prevs), _stack(currs), np.stack(Ts) if Ts else np.zeros((0, 4, 4)), camera_for(shape.camera)


def make_matched_batch(shape_name: str, B: int, *, first_pair: int = 0, noise_px=0.5, outlier_frac=0.10):
    """Explicit matched_pt / matched_ls lists for B problems of one configuration, without descriptors (the C5
    roofline run streams GN evaluations and never matches).  Vectorised: cheap even for 1024 x (8000 + 2000).
    Returns (MatchedBatch, T_gt[B,4,4], camera)."""
    from .types import MatchedBatch
    shape = SHAPES[shape_name]
    cam = camera_for(shape.camera)
    rng = np.random.default_rng(BASE_SEED + 1000 * shape.config_id + 500000 + first_pair)
    W, H, n, m = cam.width, cam.height, shape.n_pt, shape.n_ls
    Ts = np.stack([expmap_se3(np.concatenate([rng.normal(shape.t_mean, shape.t_std), rng.normal(0.0, shape.w_std, 3)]))
                   for _ in range(B)])
    lo, hi = shape.depth

    def lift(u, v, z):
        return back_projection(cam, u, v, np.maximum(cam.b * cam.fx / z, 1.0))

    def tf(P, b_idx):
        R, t = Ts[b_idx, :3, :3], Ts[b_idx, :3, 3]
        return np.einsum("nij,nj->ni", R, P) + t

    # points
    N = B * n
    bi = np.repeat(np.arange(B), n)
    u, v = rng.uniform(0, W, N), rng.uniform(0, H, N)
    P = lift(u, v, np.exp(rng.uniform(np.log(lo), np.log(hi), N)))
    obs = projection(cam, tf(P, bi)) + rng.normal(0, noise_px, (N, 2))
    out = rng.random(N) < outlier_frac
    obs[out] = np.stack([rng.uniform(0, W, out.sum()), rng.uniform(0, H, out.sum())], 1)
    # lines
    M = B * m
    li = np.repeat(np.arange(B), m)
    su, sv = rng.uniform(0, W, M), rng.uniform(0, H, M)
    z = np.exp(rng.uniform(np.log(lo), np.log(hi), M))
    length, ang = rng.uniform(30, 150, M), rng.uniform(0.2, np.pi - 0.2, M)
    spl = np.stack([su, sv], 1)
    epl = spl + np.stack([length * np.cos(ang), length * np.sin(ang)], 1)
    sP, eP = lift(su, sv, z), lift(epl[:, 0], epl[:, 1], z * rng.uniform(0.85, 1.15, M))
    s_obs = projection(cam, tf(sP, li)) + rng.normal(0, noise_px, (M, 2))
    e_obs = projection(cam, tf(eP, li)) + rng.normal(0, noise_px, (M, 2))
    mb = MatchedBatch(pt_off=np.arange(B + 1) * n, ls_off=np.arange(B + 1) * m, pt_P=P, pt_pl_obs=obs,
                      pt_sigma2=np.ones(N), ls_sP=sP, ls_eP=eP, ls_le_obs=_line_eq(s_obs, e_obs), ls_spl=spl,
                      ls_epl=epl, ls_sigma2=np.ones(M))
    return mb, Ts, cam
