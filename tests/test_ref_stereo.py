"""The stereo step held to the reference's own text on the CPU.

oracle/make_ref_stereo.py compiles the reference's matchGrid, GridStructure, LineIterator, matchStereoPoints /
matchStereoLines and their helpers into oracle/_ref/libplstvo_ref_stereo.so.  Here that library, the C oracle
(oracle/plstvo_oracle.c) and the Python restatements (ref_matchgrid.py, ref_lift.py) must agree bit for bit on the ordinary
generators, on the edge frames of stereo_edges.py and on the KITTI golden frames.  The edge frames are checked to hit
their edges, and every crafted direction straddle is checked in exact rational arithmetic."""
import numpy as np
import pytest

import ref_lift as RL
import ref_matchgrid as RG
import stereo_edges as E
from oracle import make_ref_stereo, stereo_ref as SR
from stvo_pl_b200 import stereo_synth as SS, types as T

need_ref = pytest.mark.skipif(not SR.available(), reason="oracle/_ref/libplstvo_ref_stereo.so not built (needs the reference checkout)")
W_STEREO = T.PlGridWindow(left=10, right=0, up=0, down=0)
W_WIDE = T.PlGridWindow(left=3, right=2, up=1, down=2)
KEYS_PT = ("pl", "disp", "P", "sigma2", "level", "desc")
KEYS_LS = ("spl", "epl", "sdisp", "edisp", "sP", "eP", "le", "angle", "sigma2", "level", "desc")
CAM = T.kitti_camera()


def _same(a, b, key):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (key, a.shape, b.shape)
    if a.dtype.kind == "f" and a.size:
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), key
    else:
        assert np.array_equal(a, b), key


def point_frames():
    """(name, raw frame) of every point frame: ordinary, edge and golden."""
    out = [(f"synth{s}", SS.make_stereo_frame_points(n, n - 30, seed=s)) for s, n in ((1, 400), (2, 60))]
    out += [(name, fr) for name, fr, _ in E.all_point_frames()]
    out += [(f"golden{i}", fr) for i, fr in enumerate(E.golden_point_frames())]
    return out


def line_frames():
    out = [(f"synth{s}", SS.make_stereo_frame_lines(n, n + 7, seed=s)) for s, n in ((3, 200), (4, 40))]
    out.append(("degenerate", E.lines_degenerate()[0]))
    out += [(f"golden{i}", fr) for i, fr in enumerate(E.golden_line_frames())]
    return out


CONFIGS = [(W_STEREO, 0.9, True), (W_STEREO, 0.75, False), (W_WIDE, 1.0, True), (W_WIDE, 0.6, False)]


# ---------------------------------------------------------------------------------------------- the recipe and the edges
@pytest.mark.skipif(not make_ref_stereo.available(), reason="needs the reference checkout")
def test_ranges_check():
    groups = make_ref_stereo.extract()
    assert set(groups) == {"stereo", "stereo_cam"}
    assert groups["stereo"].count("(verbatim)") == len(make_ref_stereo.RANGES) - 1


def test_edge_frames_hit_their_edges():
    (fr, hits), = [E.points_boundaries()]
    assert hits["boundary_x"] >= 195 and hits["boundary_y"] >= 60
    assert hits["at_w"] >= 2 and hits["at_h"] >= 1 and hits["negative_fraction"] >= 2 and hits["far_outside"] >= 4
    assert hits["disp_eq_min"] >= 20 and hits["epip_eq_max"] >= 20
    q_cell, t_cell = SS.stereo_cells_points(fr[0], fr[3], E.W, E.H)
    assert (q_cell[:, 0] == 64).sum() >= 2                     # a query in cell 64
    assert ((fr[0][:, 0] > -1) & (fr[0][:, 0] < 0) & (q_cell[:, 0] == 0)).sum() >= 2   # (-1, 0) truncates into cell 0
    # both sides of every boundary: float(k W / 64) lands in cell k, the float below it in cell k - 1
    xs = E.boundary_xs().astype(np.float64).reshape(65, 3)
    cells = (xs * (64.0 / E.W)).astype(np.int32)
    np.testing.assert_array_equal(cells[:, 1], np.arange(65))
    np.testing.assert_array_equal(cells[1:, 0], np.arange(64))
    dense = E.points_dense()[0]
    qd, td = SS.stereo_cells_points(dense[0], dense[3], E.W, E.H)
    assert E.window_candidates_points(qd, td, W_STEREO) > 128
    _, h = E.lines_degenerate()
    assert all(h[k] >= 1 for k in h) and h["nan_query"] >= 10 and h["zero_train"] >= 10, h
    _, h = E.grid_lines_raster()
    assert h["zero_error"] >= 5 and h["nan_query"] >= 10
    g = E.golden_line_frames()
    segs = np.concatenate([np.concatenate([f[0], f[4]]) for f in g])
    assert segs[:, [0, 2]].min() == 0.0 and segs[:, [0, 2]].max() > E.W - 1     # LSD lines reach both image borders


def test_straddles_are_exact():
    """Each crafted direction really straddles its threshold: Fraction arithmetic puts the unfused |dot| and the FMA's on
    opposite sides; both directions and negative dots occur."""
    (q, d1, t_line, t_dir, d2), keeps = E.grid_lines_straddle()
    neg = 0
    for i in range(len(q)):
        vx, vy = E.cell_direction(q[i, 2] - q[i, 0], q[i, 3] - q[i, 1])
        assert E.straddles(vx, vy, t_dir[i, 0], t_dir[i, 1], 0.75)
        u, fa, fb = E.dot_roundings(vx, vy, t_dir[i, 0], t_dir[i, 1])
        assert E.side(0.75, u) == keeps[i] and E.side(0.75, fa) != keeps[i]
        neg += (vx * t_dir[i, 0] + vy * t_dir[i, 1]) < 0
    assert keeps.sum() >= 6 and (~keeps).sum() >= 6 and neg >= 6
    # the issue that motivated these cases: (2, 1) against t = (0.3750164040949561, 0.9270181749349299) at 0.75
    u, fa, fb = E.dot_roundings(*E.cell_direction(2, 1), 0.3750164040949561, 0.9270181749349299)
    assert u == 0.75 and fa < 0.75 and fb < 0.75
    fused = E.fused_line_straddles()
    assert {k for _, _, k in fused} == {True, False}
    for (seg_l, _, _, _, seg_r, _), th, keep in fused:
        q_line, _, t_dir = SS.stereo_cells_lines(seg_l, seg_r, E.W, E.H)
        vx, vy = E.cell_direction(q_line[0, 2] - q_line[0, 0], q_line[0, 3] - q_line[0, 1])
        assert E.straddles(vx, vy, t_dir[0, 0], t_dir[0, 1], th)
        assert E.side(th, E.dot_roundings(vx, vy, t_dir[0, 0], t_dir[0, 1])[0]) == keep


# ------------------------------------------------------------------------------------------- reference == oracle == Python
@need_ref
def test_line_cells(oracle):
    segs = list(E.grid_lines_raster()[0][2]) + [tuple(r) for r in np.random.default_rng(9).uniform(-8, 72, (300, 4))]
    for x1, y1, x2, y2 in segs:
        ref = [tuple(c) for c in SR.line_cells(x1, y1, x2, y2)]
        assert ref == RG.line_cells(x1, y1, x2, y2), (x1, y1, x2, y2)
        assert ref == [tuple(c) for c in oracle.line_cells(x1, y1, x2, y2, cap=4096)], (x1, y1, x2, y2)


@need_ref
@pytest.mark.parametrize("w,ratio,best_lr", CONFIGS)
def test_match_grid_points(oracle, w, ratio, best_lr):
    frames = [SS.make_stereo_points(300, 280, seed=5, tie_stress=True)]
    frames += [SS.stereo_cells_points(f[0], f[3], E.W, E.H) for _, f in point_frames()]
    raw = [f for _, f in point_frames()]
    for k, fr in enumerate(frames):
        if k == 0:
            q, d1, t, d2 = fr
        else:
            (q, t), d1, d2 = fr, raw[k - 1][2], raw[k - 1][4]
        n_ref, ref = SR.match_grid_points(q, d1, t, d2, w, ratio, best_lr)
        n_o, m_o = oracle.match_grid_points(q, d1, t, d2, w, ratio, best_lr)
        n_p, m_p = RG.points(q, d1, t, d2, w, ratio, best_lr)
        np.testing.assert_array_equal(m_o, ref, err_msg=str(k))
        np.testing.assert_array_equal(m_p, ref, err_msg=str(k))
        assert n_ref == n_o == n_p


def grid_line_frames():
    """(frame, line_sim_th) of every grid-level line frame."""
    out = [(SS.make_stereo_lines(150, 160, seed=6), 0.75), (E.grid_lines_raster()[0], 0.75), (E.grid_lines_straddle()[0], 0.75)]
    for _, f in line_frames():
        q, tl, td = SS.stereo_cells_lines(f[0], f[4], E.W, E.H)
        out.append(((q, f[3], tl, td, f[5]), 0.75))
    for f, th, _ in E.fused_line_straddles():
        q, tl, td = SS.stereo_cells_lines(f[0], f[4], E.W, E.H)
        out.append(((q, f[3], tl, td, f[5]), th))
    return out


@need_ref
@pytest.mark.parametrize("w,ratio,best_lr", CONFIGS)
def test_match_grid_lines(oracle, w, ratio, best_lr):
    for k, ((q, d1, tl, td, d2), th) in enumerate(grid_line_frames()):
        n_ref, ref = SR.match_grid_lines(q, d1, tl, td, d2, w, ratio, th, best_lr)
        n_o, m_o = oracle.match_grid_lines(q, d1, tl, td, d2, w, ratio, th, best_lr)
        n_p, m_p = RG.lines(q, d1, tl, td, d2, w, ratio, th, best_lr)
        np.testing.assert_array_equal(m_o, ref, err_msg=str(k))
        np.testing.assert_array_equal(m_p, ref, err_msg=str(k))
        assert n_ref == n_o == n_p


@need_ref
def test_straddle_queries_follow_the_reference():
    """In the reference, each straddle query matches its only candidate exactly when the unfused |dot| keeps it."""
    (q, d1, tl, td, d2), keeps = E.grid_lines_straddle()
    _, m12 = SR.match_grid_lines(q, d1, tl, td, d2, W_STEREO, 0.9, 0.75, True)
    np.testing.assert_array_equal(m12, np.where(keeps, np.arange(len(q)), -1))
    mc, sc = T.default_stereo_match_config(), T.default_stereo_config()
    for f, th, keep in E.fused_line_straddles():
        mc.line_sim_th = th
        k, rec = SR.match_stereo_lines(CAM, mc, sc, *f)
        assert k == int(keep)


def _configs():
    mc, sc = T.default_stereo_match_config(), T.default_stereo_config()
    kitti = T.default_stereo_match_config()
    kitti.min_ratio_12_p = 0.75
    sk = T.default_stereo_config()
    sk.max_dist_epip = 0.0
    return [(mc, sc), (kitti, sk)]


@need_ref
@pytest.mark.parametrize("cfg", [0, 1])
def test_match_stereo_points(oracle, cfg):
    mc, sc = _configs()[cfg]
    for name, f in point_frames():
        k_ref, ref = SR.match_stereo_points(CAM, mc, sc, *f)
        m12, k_o, rec = oracle.match_stereo_points(CAM, mc, sc, *f)
        assert k_ref == k_o, name
        for key in KEYS_PT:
            _same(rec[key], ref[key], (name, key))
        py = RL.lift_points(CAM, sc, f[0], f[1], f[2], f[3], m12)
        for key in KEYS_PT:
            _same(np.asarray(py[key], rec[key].dtype).reshape(rec[key].shape), rec[key], (name, "python", key))


@need_ref
@pytest.mark.parametrize("cfg", [0, 1])
def test_match_stereo_lines(oracle, cfg):
    mc, sc = _configs()[cfg]
    frames = [(name, f, mc.line_sim_th) for name, f in line_frames()]
    frames += [(f"straddle{i}", f, th) for i, (f, th, _) in enumerate(E.fused_line_straddles())]
    for name, f, th in frames:
        m = T.PlStereoMatchConfig.from_buffer_copy(mc)
        m.line_sim_th = th
        k_ref, ref = SR.match_stereo_lines(CAM, m, sc, *f)
        m12, k_o, rec = oracle.match_stereo_lines(CAM, m, sc, *f)
        assert k_ref == k_o, name
        for key in KEYS_LS:
            _same(rec[key], ref[key], (name, key))
        py = RL.lift_lines(CAM, sc, f[0], f[1], f[2], f[3], f[4], m12)
        for key in KEYS_LS:
            _same(np.asarray(py[key], rec[key].dtype).reshape(rec[key].shape), rec[key], (name, "python", key))


@need_ref
def test_line_segment_overlap_stereo(oracle):
    sc = T.default_stereo_config()
    vals = [0.0, 0.1, 0.05, 10.0, 10.1, 10.01, -3.0, 5.0, 5.0000001, 20.0]
    rng = np.random.default_rng(3)
    for a in vals:
        for b in vals:
            for c, d in [(a, b), (b, a), tuple(rng.uniform(-5, 25, 2)), (a + 0.005, b - 0.005)]:
                r, o = SR.line_segment_overlap_stereo(sc, a, b, c, d), oracle.line_segment_overlap_stereo(sc, a, b, c, d)
                assert np.float64(r).view(np.uint64) == np.float64(o).view(np.uint64), (a, b, c, d)


# ------------------------------------------------------------------------------------------------------- ratio above one
def _seen_ties(q, d1, t, d2, w, best_lr, rows=T.GRID_ROWS, cols=T.GRID_COLS):
    """Per query, how many candidates that pass the bestLRMatches gate share the best distance.  The gate's outcome does
    not depend on the order a query's candidates are visited in, so this is well defined."""
    grid = {}
    for idx, (x, y) in enumerate(t):
        if 0 <= x < cols and 0 <= y < rows:
            grid.setdefault((int(x), int(y)), []).append(idx)
    dist = [RG.INT_MAX] * len(d2)
    ties = []
    for i1, (x, y) in enumerate(q):
        cand = set()
        RG.grid_get(grid, rows, cols, int(x), int(y), w, cand)
        seen = []
        for i2 in cand:
            d = RG.hamming(d1[i1], d2[i2])
            if best_lr:
                if d >= dist[i2]:
                    continue
                dist[i2] = d
            seen.append(d)
        ties.append(seen.count(min(seen)) if seen else 0)
    return np.array(ties)


@need_ref
@pytest.mark.parametrize("best_lr", [False, True])
def test_ratio_above_one_differs_only_on_ties(oracle, best_lr):
    """For min_ratio_12_p > 1 a tied best distance passes the ratio test, and the reference takes the first of the tied
    candidates in its unordered_set's order, which the oracle (and the GPU) do not follow.  They differ there, and only on
    queries with a tied best distance; where they differ, both picks are at that distance."""
    n_diff = 0
    for seed in range(4):
        q, d1, t, d2 = SS.make_stereo_points(250, 240, seed=40 + seed, tie_stress=True)
        _, ref = SR.match_grid_points(q, d1, t, d2, W_WIDE, 1.5, best_lr)
        _, orc = oracle.match_grid_points(q, d1, t, d2, W_WIDE, 1.5, best_lr)
        ties = _seen_ties(q, d1, t, d2, W_WIDE, best_lr)
        diff = np.nonzero(ref != orc)[0]
        assert (ties[diff] >= 2).all()
        if not best_lr:
            for i in diff:
                assert RG.hamming(d1[i], d2[ref[i]]) == RG.hamming(d1[i], d2[orc[i]])
        n_diff += len(diff)
        # at ratio <= 1 a tie never matches, so order cannot matter
        _, ref1 = SR.match_grid_points(q, d1, t, d2, W_WIDE, 1.0, best_lr)
        _, orc1 = oracle.match_grid_points(q, d1, t, d2, W_WIDE, 1.0, best_lr)
        np.testing.assert_array_equal(ref1, orc1)
    assert n_diff > 0
