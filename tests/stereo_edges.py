"""Edge frames for the stereo step (matchGrid, getLineCoords and the lifting of matchStereoPoints / matchStereoLines).

The ordinary generators (stvo_pl_b200/stereo_synth.py) keep every key point inside [0, W - 1e-3], never on a cell boundary,
never a zero-length segment and never a direction dot product near line_sim_th.  The frames here go exactly there:

  points   key points at float(k W / 64) and its float neighbours (cell boundaries), at x = W and y = H (a query in cell 64
           still searches cells 54..63; a train there is out of the grid), in (-1, 0) (truncation, not floor, puts it in cell
           0), far outside the image; rows that differ by exactly max_dist_epip and disparities of exactly min_disp; distance
           0, tied best distances, single candidates; one frame whose windows overflow the 128-candidate fast path.
  lines    both query endpoints in one cell (NaN direction, which passes the filter), zero-length right segments (NaN
           t_dir), segments horizontal or vertical in grid units, steep segments with swapped endpoints, segments crossing or
           outside the grid border and spanning more than 64 cells; on the grid level also integer endpoints where
           Bresenham's error hits exactly 0.
  straddle train directions whose |dot| with the query direction falls on one side of line_sim_th when evaluated as the
           reference writes it (two roundings per product, one per sum) and on the other side when one product is fused
           into an FMA.  Each straddling train is its query's only candidate, so the query's m12 itself flips.
  golden   the KITTI golden stereo frames: tests/golden/orb_kitti.npz key points, tests/golden/lbd.npz kitti_stereo lines.

Every builder returns the frame and what it was built to hit, so the tests can assert the edges are really there.
Test infrastructure only."""
from __future__ import annotations

import math
import os
from fractions import Fraction

import numpy as np

from stvo_pl_b200 import types as T

W, H = 1241, 376                               # the KITTI camera's image (types.kitti_camera)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
f32 = np.float32


# ---------------------------------------------------------------------------------------------------- exact dot products
def dot_roundings(vx, vy, tx, ty):
    """|dot| of (vx, vy) and (tx, ty) as doubles: (unfused, fused with the first product exact, fused with the second exact).
    Unfused is the reference's a.first * b.first + a.second * b.second (include/matching.h:39-41) under -ffp-contract=off."""
    a, b = Fraction(vx) * Fraction(tx), Fraction(vy) * Fraction(ty)
    ra, rb = Fraction(float(a)), Fraction(float(b))
    return abs(float(ra + rb)), abs(float(a + rb)), abs(float(ra + b))


def side(th, x):
    """The filter's verdict (src/matching.cpp:221): True = kept (not |dot| < th)."""
    return not (x < th)


def straddles(vx, vy, tx, ty, th):
    """True when the unfused |dot| and the fused one fall on opposite sides of th.  "Fused" is fma(vx, tx, vy * ty), the
    form nvcc emits for vx * tx + vy * ty (PTX: mul.f64 of the second product, then fma.rn.f64).  When the reference keeps
    the candidate, the other fused form must flip too, so the case does not hang on nvcc's choice.  When it drops it, that
    cannot be asked: the unfused sum lies at least one ulp of the smaller product below th, further than that product's
    own rounding error reaches, so only the form with the larger product exact can cross."""
    u, fa, fb = dot_roundings(vx, vy, tx, ty)
    if side(th, u):
        return not side(th, fa) and not side(th, fb)
    return side(th, fa)


def cell_direction(a, b):
    """normalize((a, b)) of integer cell differences, as matchGrid forms the query direction (:207-211)."""
    vx, vy = float(a), float(b)
    mag = math.sqrt(vx * vx + vy * vy)
    return vx / mag, vy / mag


def find_straddle(a, b, th, ref_keeps, sign=1.0, span=60):
    """A unit-ish train direction t whose |dot| with the cell direction (a, b) straddles th: the reference keeps the
    candidate and an FMA drops it (ref_keeps) or the other way round.  sign = -1 makes the dot negative."""
    vx, vy = cell_direction(a, b)
    phi, d = math.atan2(vy, vx), math.acos(th)
    def steps(x0):   # x0 and its float neighbours, nearest first
        yield x0
        lo = hi = x0
        for _ in range(span):
            lo, hi = math.nextafter(lo, -math.inf), math.nextafter(hi, math.inf)
            yield lo
            yield hi
    for theta in (phi + d, phi - d):
        for tx in steps(math.cos(theta)):
            for ty in steps(math.sin(theta)):
                t = (sign * tx, sign * ty)
                if straddles(vx, vy, t[0], t[1], th) and side(th, dot_roundings(vx, vy, *t)[0]) == ref_keeps:
                    return t
    raise RuntimeError(f"no straddle found for {(a, b, th, ref_keeps, sign)}")


# ------------------------------------------------------------------------------------------------------------ points
def _desc(rng, n):
    return rng.integers(0, 256, (n, 32), dtype=np.uint8)


def _flip(rng, d, bits):
    d = d.copy()
    for r in range(len(d)):
        for b in rng.choice(256, bits, replace=False):
            d[r, b // 8] ^= np.uint8(1 << (b % 8))
    return d


def boundary_xs(W=W):
    """float(k W / 64) for every cell boundary k = 0..64 and its two float neighbours."""
    xs = []
    for k in range(65):
        x = f32(k * W / 64.0)
        xs += [np.nextafter(x, f32(-np.inf)), x, np.nextafter(x, f32(np.inf))]
    return np.array(xs, np.float32)


def boundary_ys(H=H):
    ys = []
    for k in range(49):
        y = f32(k * H / 48.0)
        ys += [np.nextafter(y, f32(-np.inf)), y, np.nextafter(y, f32(np.inf))]
    return np.array(ys, np.float32)


def on_boundary(v, size, cells):
    """Values whose grid coordinate v * (cells / size) is an integer or within one float step of one."""
    g = v.astype(np.float64) * (cells / float(size))
    return np.abs(g - np.round(g)) <= np.abs(np.spacing(v.astype(np.float32))).astype(np.float64) * cells / size * 1.5


def points_boundaries(seed=0):
    """Key points on cell boundaries and outside the image; the right image holds each left point's match shifted by whole
    cells (so it lands on a boundary again), by exactly 1 px (disparity = min_disp), and with the row moved by exactly 1 px
    (= max_dist_epip) or by one float step more."""
    rng = np.random.default_rng(seed)
    xs, ys = boundary_xs(), boundary_ys()
    lx = np.concatenate([xs, rng.choice(xs, 60), [W, W, f32(-0.25), f32(-0.999), f32(-5000.0), f32(3 * W), f32(600.0), f32(600.0)]])
    ly = np.concatenate([rng.uniform(0, H, len(xs)).astype(np.float32), rng.choice(ys, 60),
                         [f32(100.5), f32(H), f32(50.0), f32(-0.5), f32(60.0), f32(70.0), f32(-3000.0), f32(10 * H)]])
    kp_l = np.stack([lx, ly], 1).astype(np.float32)
    n = len(kp_l)
    d1 = _desc(rng, n)
    k_cell = rng.integers(0, 4, n)
    cell_w = f32(W / 64.0)
    rx = np.empty(n, np.float32)
    ry = kp_l[:, 1].copy()
    kind = rng.integers(0, 4, n)
    for i in range(n):
        if kind[i] == 0:                                   # whole cells to the left: a boundary again
            rx[i] = f32(max(int(round(lx[i] / cell_w)) - k_cell[i], 0) * W / 64.0) if abs(lx[i]) < 2 * W else lx[i]
        elif kind[i] == 1:                                 # disparity exactly 1 px
            rx[i] = lx[i] - f32(1.0)
        elif kind[i] == 2:                                 # row exactly 1 px off
            rx[i] = lx[i] - f32(3.0)
            ry[i] = ly[i] + f32(1.0)
        else:                                              # row one float step beyond 1 px off
            rx[i] = lx[i] - f32(3.0)
            ry[i] = np.nextafter(ly[i] + f32(1.0), f32(np.inf))
    kp_r = np.stack([rx, ry], 1).astype(np.float32)
    d2 = _flip(rng, d1, 2)
    d2[::7] = d1[::7]                                      # distance 0
    perm = rng.permutation(n)
    kp_r, d2 = kp_r[perm], d2[perm]
    oct_l = rng.integers(0, 8, n).astype(np.int32)
    hits = dict(boundary_x=int(on_boundary(lx, W, 64).sum()), boundary_y=int(on_boundary(ly, H, 48).sum()),
                at_w=int((lx == f32(W)).sum()), at_h=int((ly == f32(H)).sum()),
                negative_fraction=int(((lx > -1) & (lx < 0)).sum()),
                far_outside=int(((lx < -1000) | (lx > 2 * W) | (ly < -1000) | (ly > 2 * H)).sum()),
                disp_eq_min=int(((lx - rx) == f32(1.0)).sum()), epip_eq_max=int((np.abs(ly - ry) == f32(1.0)).sum()))
    return (kp_l, oct_l, d1, kp_r, d2), hits


def points_distances(seed=1):
    """Small windows with hand-set distances: 0, tied best distances (no match at ratio <= 1), single candidates
    (best_d2 = INT_MAX), a later query at an equal distance (the bestLRMatches gate)."""
    rng = np.random.default_rng(seed)
    kp_l, kp_r, d1, d2 = [], [], [], []
    cw, ch = W / 64.0, H / 48.0
    for r in range(40):
        row = f32((r % 48 + 0.5) * ch)
        base = _desc(rng, 1)[0]
        x0 = f32((20 + (r % 30)) * cw + 3.0)
        kind = r % 4
        if kind == 0:                                  # single candidate at distance 0
            kp_l.append((x0, row)); d1.append(base)
            kp_r.append((x0 - f32(2 * cw), row)); d2.append(base)
        elif kind == 1:                                # two candidates, tied best distance
            kp_l.append((x0, row)); d1.append(base)
            for k in (1, 2):
                kp_r.append((x0 - f32(k * cw), row)); d2.append(_flip(rng, base[None], 3)[0])
        elif kind == 2:                                # single candidate far in descriptor space
            kp_l.append((x0, row)); d1.append(base)
            kp_r.append((x0 - f32(cw), row)); d2.append(~base)
        else:                                          # two queries at the same distance from one train
            kp_l += [(x0, row), (x0 + f32(1.0), row)]; d1 += [base, base]
            kp_r.append((x0 - f32(cw), row)); d2.append(_flip(rng, base[None], 1)[0])
    kp_l, kp_r = np.array(kp_l, np.float32), np.array(kp_r, np.float32)
    d1, d2 = np.array(d1, np.uint8), np.array(d2, np.uint8)
    return (kp_l, rng.integers(0, 4, len(kp_l)).astype(np.int32), d1, kp_r, d2), dict(queries=len(kp_l))


def points_dense(seed=2):
    """Hundreds of right key points in three cells of one row: every nearby query window holds more than 128
    candidates, so the frame takes matchGrid's sequential path on the GPU."""
    rng = np.random.default_rng(seed)
    cw, ch = W / 64.0, H / 48.0
    n_r, n_l = 420, 90
    kp_r = np.stack([rng.uniform(20 * cw, 23 * cw, n_r), rng.uniform(10 * ch, 11 * ch - 1e-3, n_r)], 1).astype(np.float32)
    kp_l = np.stack([rng.uniform(23 * cw, 30 * cw, n_l), rng.uniform(10 * ch, 11 * ch - 1e-3, n_l)], 1).astype(np.float32)
    d1 = _desc(rng, n_l)
    d2 = _desc(rng, n_r)
    src = rng.permutation(n_l)[:60]
    dst = rng.permutation(n_r)[:60]
    d2[dst] = _flip(rng, d1[src], 4)
    kp_r[dst, 1] = kp_l[src, 1]
    return (kp_l, rng.integers(0, 4, n_l).astype(np.int32), d1, kp_r, d2), dict(dense=n_r)


# ------------------------------------------------------------------------------------------------------------- lines
def _segs_frame(seg_l, seg_r, rng, match=None, bits=3):
    seg_l, seg_r = np.asarray(seg_l, np.float32).reshape(-1, 4), np.asarray(seg_r, np.float32).reshape(-1, 4)
    d1, d2 = _desc(rng, len(seg_l)), _desc(rng, len(seg_r))
    for i, j in (match or []):
        d2[j] = _flip(rng, d1[i][None], bits)[0]
    ang = rng.uniform(-np.pi, np.pi, len(seg_l)).astype(np.float32)
    return (seg_l, ang, rng.integers(0, 3, len(seg_l)).astype(np.int32), d1, seg_r, d2)


def lines_degenerate(seed=3):
    """Left segments inside one cell (NaN query direction), zero-length right segments (NaN t_dir), right segments
    horizontal or vertical in grid units, steep ones with swapped endpoints, and segments crossing the grid border,
    outside it, or spanning more than 64 cells."""
    rng = np.random.default_rng(seed)
    cw, ch = W / 64.0, H / 48.0
    L, R, match = [], [], []

    def pair(l, r):
        match.append((len(L), len(R)))
        L.append(l); R.append(r)
    for k in range(12):
        cx, cy = (8 + 4 * k) * cw, (4 + 3 * k) * ch
        # both left endpoints in one cell; the right one 40 px to the left, a genuine stereo pair
        l = (cx + 2, cy + 1, cx + cw - 3, cy + ch - 1)
        pair(l, (l[0] - 40, l[1], l[2] - 40, l[3]))
        # zero-length right segment in the window of a vertical left one
        l = (cx + 5, cy - 2 * ch, cx + 5.5, cy + 2 * ch)
        pair(l, (l[0] - 30, cy, l[0] - 30, cy))
        # right segment exactly horizontal (sy == ey) and exactly vertical (sx == ex)
        l = (cx - 3 * cw, cy + 2.5, cx + 2 * cw, cy + 3.5)
        pair(l, (l[0] - 25, cy + 2.5, l[2] - 25, cy + 2.5))
        l = (cx + 7, cy - 3 * ch, cx + 7, cy + 3 * ch)
        pair(l, (l[0] - 35, l[1], l[2] - 35, l[3]))
        # steep, endpoints swapped (end above start, end left of start)
        l = (cx + 9, cy + 3 * ch, cx + 1, cy - 3 * ch)
        pair(l, (l[0] - 20, l[1], l[2] - 20, l[3]))
    # across the border, outside it, and longer than the grid is wide
    for l, r in [((-150.0, 40.0, 300.0, 120.0), (-190.0, 40.0, 260.0, 120.0)),
                 ((W - 200.0, 300.0, W + 300.0, 360.0), (W - 240.0, 300.0, W + 260.0, 360.0)),
                 ((-60.0, 200.0, W + 60.0, 230.0), (-100.0, 200.0, W + 20.0, 230.0)),
                 ((100.0, -80.0, 400.0, -10.0), (60.0, -80.0, 360.0, -10.0)),
                 ((500.0, H - 40.0, 520.0, H + 90.0), (470.0, H - 40.0, 490.0, H + 90.0)),
                 ((f32(-0.5), 10.0, f32(W), 20.0), (f32(-30.5), 10.0, f32(W - 30), 20.0))]:
        pair(l, r)
    seg_l, seg_r = np.array(L, np.float32), np.array(R, np.float32)
    perm = rng.permutation(len(seg_r))
    inv = np.argsort(perm)
    frame = _segs_frame(seg_l, seg_r[perm], rng, [(i, inv[j]) for i, j in match])
    inv_w, inv_h = 64.0 / W, 48.0 / H
    q = (seg_l.astype(np.float64) * [inv_w, inv_h, inv_w, inv_h]).astype(np.int32)
    gl = seg_r.astype(np.float64) * [inv_w, inv_h, inv_w, inv_h]
    hits = dict(nan_query=int(((q[:, 0] == q[:, 2]) & (q[:, 1] == q[:, 3])).sum()),
                zero_train=int(((seg_r[:, 0] == seg_r[:, 2]) & (seg_r[:, 1] == seg_r[:, 3])).sum()),
                horizontal_train=int(((seg_r[:, 1] == seg_r[:, 3]) & (seg_r[:, 0] != seg_r[:, 2])).sum()),
                vertical_train=int(((seg_r[:, 0] == seg_r[:, 2]) & (seg_r[:, 1] != seg_r[:, 3])).sum()),
                swapped_steep=int(((np.abs(seg_l[:, 3] - seg_l[:, 1]) > np.abs(seg_l[:, 2] - seg_l[:, 0]) * ch / cw)
                                   & (seg_l[:, 3] < seg_l[:, 1])).sum()),
                over_64_cells=int((np.abs(gl[:, 2] - gl[:, 0]) > 64).sum()),
                outside=int(((gl.reshape(-1, 2, 2) < 0) | (gl.reshape(-1, 2, 2) >= [64, 48])).any(axis=(1, 2)).sum()))
    return frame, hits


def grid_lines_raster(seed=4):
    """Grid-level line frame (integer query cells, double train segments, t_dir given): integer-valued endpoints where
    Bresenham's error reaches exactly 0, steep and swapped segments, segments outside the grid and over 64 cells long."""
    rng = np.random.default_rng(seed)
    t_line = [(10.0, 5.0, 14.0, 6.0), (30.0, 9.0, 22.0, 7.0), (40.0, 20.0, 41.0, 24.0), (41.0, 30.0, 40.0, 26.0),
              (2.0, 40.0, 10.0, 42.0), (-5.0, 12.0, 70.0, 14.0), (70.0, 15.0, -6.0, 13.5), (20.0, -3.0, 22.0, -0.5),
              (60.0, 47.0, 66.0, 49.0), (5.5, 30.0, 5.5, 38.0), (12.0, 20.0, 12.0, 20.0), (33.0, 33.0, 37.0, 33.0),
              (8.0, 2.0, 16.0, 4.0), (50.0, 10.0, 46.0, 11.0), (25.0, 25.0, 27.0, 26.0), (-2.0, -2.0, 65.9, 47.9)]
    t_line = np.array(t_line, np.float64)
    v = t_line[:, 2:] - t_line[:, :2]
    with np.errstate(all="ignore"):
        t_dir = v / np.sqrt(v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1])[:, None]
    n2 = len(t_line)
    q = []
    for k in range(n2):                                    # a query near each train, plus one with a NaN direction
        x1, y1, x2, y2 = t_line[k]
        cx = int(np.clip(max(x1, x2), 0, 63)) + 2
        cy = int(np.clip(y1, 0, 47))
        q.append((min(cx, 64), cy, min(cx + int(np.sign(x2 - x1)), 64), int(np.clip(y2, 0, 47))))
        q.append((cx, cy, cx, cy))
    q = np.array(q, np.int32)
    d2 = _desc(rng, n2)
    d1 = np.repeat(d2, 2, axis=0)
    d1 = _flip(rng, d1, 2)
    zero_err = 0
    for x1, y1, x2, y2 in t_line:                          # count segments whose error passes through exactly 0
        steep = abs(y2 - y1) > abs(x2 - x1)
        if steep:
            x1, y1, x2, y2 = y1, x1, y2, x2
        if x1 > x2:
            x1, x2, y1, y2 = x2, x1, y2, y1
        dx, dy, err = x2 - x1, abs(y2 - y1), (x2 - x1) / 2.0
        for _ in range(int(x1), int(x2) + 1):
            err -= dy
            zero_err += err == 0
            if err < 0:
                err += dx
    return (q, d1, t_line, t_dir, d2), dict(zero_error=int(zero_err), nan_query=int(n2))


def grid_lines_straddle(th=0.75, seed=5):
    """Grid-level straddle frame at line_sim_th = th: each query's only candidate is a train whose t_dir straddles th,
    in both directions (reference keeps / FMA drops and the reverse) and with positive and negative dots.  Returns the
    frame and, per query, whether the reference keeps its candidate."""
    rng = np.random.default_rng(seed)
    dirs = [(2, 1), (1, 1), (1, 2), (3, -1), (-2, 3), (5, 2), (1, 3), (4, 1), (3, 2), (-1, 4)]
    q, t_line, t_dir, keeps = [], [], [], []
    k = 0
    for ref_keeps in (True, False):
        for sign in (1.0, -1.0):
            found = 0
            for a, b in dirs:                              # not every direction has a straddle within reach: take 3 that do
                try:
                    t = find_straddle(a, b, th, ref_keeps, sign, span=40)
                except RuntimeError:
                    continue
                row = 2 + 2 * (k % 22)
                col = 12 + 25 * (k // 22)
                q.append((col, row, col + a, row + b))
                t_dir.append(t)
                t_line.append((col - 3.5, row + 0.5, col - 3.2, row + 0.6))   # one cell, in the query's start window only
                keeps.append(ref_keeps)
                k += 1
                found += 1
                if found == 3:
                    break
            assert found == 3, (ref_keeps, sign)
    q, t_line, t_dir = np.array(q, np.int32), np.array(t_line, np.float64), np.array(t_dir, np.float64)
    d1 = _desc(rng, len(q))
    d2 = _flip(rng, d1, 5)
    return (q, d1, t_line, t_dir, d2), np.array(keeps)


def fused_line_straddles(n=4, seed=6, W=W, H=H, want=None):
    """Raw stereo line frames for matchStereoLines / the tracker, one per straddle: a genuine stereo pair (the right
    segment is the left one 60 px to the left) whose train direction, formed from the float endpoints as the caller forms
    it (:331-333), has an unfused |dot| u with the query's cell direction that an FMA rounds to the other side of a
    threshold.  Returns [(frame, line_sim_th, ref_keeps)]: th = u when the fused value is below u (the reference keeps the
    candidate, an FMA drops it), th = the fused value when it is above (the reference drops it, an FMA keeps it); "fused"
    as in straddles()."""
    rng = np.random.default_rng(seed)
    cw, ch = W / 64.0, H / 48.0
    inv = np.array([64.0 / W, 48.0 / H])
    out, kinds = [], []
    want = want or [True, False] * (n // 2)
    tries = 0
    while len(out) < len(want):
        tries += 1
        assert tries < 200000, "no fused straddle found"
        cx, cy = int(rng.integers(14, 60)), int(rng.integers(3, 36))   # rows 3..38: lines_dense_clutter keeps to 42..47
        # a nearly vertical left segment crossing one cell boundary in x: cell direction (1, 1) or (1, 2), actual ~80-88 deg
        dyc = int(rng.integers(1, 3))
        sx, ex = (cx + 1 - rng.uniform(0.02, 0.12)) * cw, (cx + 1 + rng.uniform(0.02, 0.12)) * cw
        sy, ey = (cy + rng.uniform(0.05, 0.9)) * ch, (cy + dyc + rng.uniform(0.05, 0.9)) * ch
        seg_l = np.array([sx, sy, ex, ey], np.float32)
        seg_r = seg_l - np.float32([60, 0, 60, 0])
        ql = (seg_l.astype(np.float64) * np.tile(inv, 2)).astype(np.int32)
        vx, vy = cell_direction(ql[2] - ql[0], ql[3] - ql[1])
        tvx = float(np.float64(f32(seg_r[2] - seg_r[0])) * inv[0])
        tvy = float(np.float64(f32(seg_r[3] - seg_r[1])) * inv[1])
        mag = math.sqrt(tvx * tvx + tvy * tvy)             # Python floats: two roundings, as normalize (matching.h:43-48)
        tx, ty = tvx / mag, tvy / mag
        u, fa, fb = dot_roundings(vx, vy, tx, ty)
        if not (0.6 < u < 0.95):
            continue
        ref_keeps = want[len(out)]
        if ref_keeps and fa < u and fb < u:
            th = u
        elif not ref_keeps and fa > u:
            th = fa
        else:
            continue
        assert straddles(vx, vy, tx, ty, th) and side(th, u) == ref_keeps
        frame = _segs_frame(seg_l[None], seg_r[None], rng, [(0, 0)], bits=2)
        out.append((frame, th, ref_keeps))
    return out


def lines_dense_clutter(n_l=40, n_r=700, seed=7, W=W, H=H):
    """Long, nearly horizontal segments crowded into grid rows 42..47: the windows of the queries there hold far more than
    128 candidates, so a frame carrying this clutter takes matchGrid's sequential path.  Rows 0..41 stay free."""
    rng = np.random.default_rng(seed)
    y0, y1 = 42 * H / 48.0 + 0.5, H - 0.5

    def segs(n):
        sx, sy = rng.uniform(0, W * 0.5, n), rng.uniform(y0, y1, n)
        return np.stack([sx, sy, sx + rng.uniform(200, W * 0.5, n), np.clip(sy + rng.uniform(-4, 4, n), y0, y1)], 1)
    seg_l, seg_r = segs(n_l), segs(n_r)
    seg_r[:n_l] = seg_l - [25.0, 0.0, 25.0, 0.0]
    return _segs_frame(seg_l, seg_r, rng, [(i, i) for i in range(n_l)])


def merge_line_frames(a, b):
    """One raw line frame holding a's lines first, then b's."""
    return tuple(np.concatenate([x, y]) for x, y in zip(a, b))


def window_candidates_lines(q_line, t_line, w, rows=T.GRID_ROWS, cols=T.GRID_COLS):
    """Largest candidate set of any query (lines: the union over both endpoint windows)."""
    from ref_matchgrid import line_cells
    grid = {}
    for idx, (x1, y1, x2, y2) in enumerate(t_line):
        for c in line_cells(float(x1), float(y1), float(x2), float(y2)):
            if 0 <= c[0] < cols and 0 <= c[1] < rows:
                grid.setdefault(c, set()).add(idx)
    best = 0
    for sx, sy, ex, ey in q_line:
        cand = set()
        for x, y in ((sx, sy), (ex, ey)):
            for x_ in range(max(0, x - w.left), min(cols, x + w.right + 1)):
                for y_ in range(max(0, y - w.up), min(rows, y + w.down + 1)):
                    cand |= grid.get((x_, y_), set())
        best = max(best, len(cand))
    return best


# ------------------------------------------------------------------------------------------------------------ golden
def golden_point_frames():
    """The two KITTI golden stereo frames' key points (cv2's ORB, tests/golden/orb_kitti.npz): [(kp_l, oct_l, d_l, kp_r, d_r)]."""
    z = np.load(os.path.join(GOLDEN, "orb_kitti.npz"))
    off, xy, octv, desc = z["det_off"], z["det_xy"], z["det_oct"], z["det_desc"]
    out = []
    for f in range(2):
        l, r = 2 * f, 2 * f + 1
        out.append((xy[off[l]:off[l + 1]], octv[off[l]:off[l + 1]].astype(np.int32), desc[off[l]:off[l + 1]],
                    xy[off[r]:off[r + 1]], desc[off[r]:off[r + 1]]))
    return out


def golden_line_frames():
    """The two KITTI golden stereo frames' key lines and the reference's LBD descriptors (tests/golden/lbd.npz kitti_stereo):
    [(seg_l, angle_l, oct_l, d_l, seg_r, d_r)]."""
    z = np.load(os.path.join(GOLDEN, "lbd.npz"))
    off, seg, desc = z["kitti_stereo/kl_off"], z["kitti_stereo/seg"], z["kitti_stereo/desc"]
    ang = z["kitti_stereo/angle_bits"].view(np.float32)
    out = []
    for f in range(2):
        l, r = 2 * f, 2 * f + 1
        out.append((seg[off[l]:off[l + 1]], ang[off[l]:off[l + 1]], np.zeros(off[l + 1] - off[l], np.int32),
                    desc[off[l]:off[l + 1]], seg[off[r]:off[r + 1]], desc[off[r]:off[r + 1]]))
    return out


# ------------------------------------------------------------------------------------------------------------ helpers
def window_candidates_points(q_cell, t_cell, w, rows=T.GRID_ROWS, cols=T.GRID_COLS):
    """Largest candidate set of any query window (points)."""
    counts = {}
    for x, y in t_cell:
        if 0 <= x < cols and 0 <= y < rows:
            counts[(int(x), int(y))] = counts.get((int(x), int(y)), 0) + 1
    best = 0
    for x, y in q_cell:
        s = sum(counts.get((x_, y_), 0) for x_ in range(max(0, x - w.left), min(cols, x + w.right + 1))
                for y_ in range(max(0, y - w.up), min(rows, y + w.down + 1)))
        best = max(best, s)
    return best


def all_point_frames():
    """(name, frame, hits) of every point edge frame."""
    return [("boundaries",) + points_boundaries(), ("distances",) + points_distances(), ("dense",) + points_dense()]
