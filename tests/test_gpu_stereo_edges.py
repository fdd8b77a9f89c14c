"""The stereo step on the GPU at its edges, byte for byte against the reference's own text (oracle/_ref, built by
oracle/make_ref_stereo.py) and the C oracle.

The edge frames of stereo_edges.py (cell boundaries, points outside the image, exact lifting thresholds, NaN directions,
zero-length and border-crossing segments, tied and zero distances, direction straddles, the KITTI golden frames) go through
plstvo_match_grid_points / _lines, plstvo_match_stereo_points / _lines and plstvo_track_stereo_batch, mixed into ragged
batches between ordinary frames, on the fast path and on the sequential path a frame takes when a window holds more than
128 candidates.  A straddle is a train direction whose |dot| with the query's lies on one side of line_sim_th unfused and
on the other when nvcc fuses the dot into an FMA; it is the query's only candidate, so the query's m12 shows which one the
kernel evaluated."""
import numpy as np
import pytest

import stereo_edges as E
from oracle import stereo_ref as SR
from stvo_pl_b200 import stereo_synth as SS, types as T

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not SR.available(), reason="oracle/_ref/libplstvo_ref_stereo.so not built")]
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


def _offsets(frames, i):
    return np.concatenate([[0], np.cumsum([len(f[i]) for f in frames])]).astype(np.int32)


def _cat(frames, i, width):
    return np.concatenate([np.asarray(f[i]).reshape(-1, width) if width else np.asarray(f[i]) for f in frames])


def raw_point_frames():
    """Edge point frames between ordinary ones (ragged sizes, an empty frame and a one-point frame among them)."""
    edges = [fr for _, fr, _ in E.all_point_frames()] + E.golden_point_frames()
    out = []
    for k, fr in enumerate(edges):
        out.append(SS.make_stereo_frame_points(300 - 40 * k, 280 - 30 * k, seed=500 + k))
        out.append(fr)
    out.insert(3, SS.make_stereo_frame_points(0, 0, seed=1))
    out.insert(5, SS.make_stereo_frame_points(1, 1, seed=2))
    return out


def raw_line_frames():
    dense = E.merge_line_frames(E.lines_degenerate()[0], E.lines_dense_clutter())
    edges = [E.lines_degenerate()[0], dense] + E.golden_line_frames()
    out = []
    for k, fr in enumerate(edges):
        out.append(SS.make_stereo_frame_lines(120 - 20 * k, 130 - 15 * k, seed=600 + k))
        out.append(fr)
    return out


def test_edge_batches_cover_both_paths():
    """The dense point frame and the cluttered line frame overflow the 128-candidate fast path; the others do not."""
    frames = raw_point_frames()
    over = [E.window_candidates_points(*SS.stereo_cells_points(f[0], f[3], E.W, E.H), W_STEREO) > 128 for f in frames]
    assert 1 <= sum(over) < len(frames)
    lines = raw_line_frames()
    over = [E.window_candidates_lines(*SS.stereo_cells_lines(f[0], f[4], E.W, E.H)[:2], W_STEREO) > 128 for f in lines]
    assert 1 <= sum(over) < len(lines)


# ---------------------------------------------------------------------------------------------------------- matchGrid
@pytest.mark.parametrize("w,ratio,best_lr", [(W_STEREO, 0.9, True), (W_WIDE, 0.75, False), (W_STEREO, 1.0, True)])
def test_gpu_match_grid_points_edges(engine, oracle, w, ratio, best_lr):
    frames = raw_point_frames()
    cells = [SS.stereo_cells_points(f[0], f[3], E.W, E.H) for f in frames]
    grid = [(c[0], f[2], c[1], f[4]) for c, f in zip(cells, frames)]
    q_off, t_off = _offsets(grid, 1), _offsets(grid, 3)
    total, m12, counts = engine.match_grid_points(q_off, _cat(grid, 0, 2), _cat(grid, 1, 32), t_off, _cat(grid, 2, 2),
                                                  _cat(grid, 3, 32), w, ratio, best_lr)
    for k, g in enumerate(grid):
        n_ref, ref = SR.match_grid_points(*g, w, ratio, best_lr)
        n_o, m_o = oracle.match_grid_points(*g, w, ratio, best_lr)
        np.testing.assert_array_equal(m_o, ref, err_msg=f"oracle, frame {k}")
        np.testing.assert_array_equal(m12[q_off[k]:q_off[k + 1]], ref, err_msg=f"frame {k}")
        assert counts[k] == n_ref == n_o, k
    assert total == counts.sum()


def _straddle_grid_frames(overflow):
    """The grid-level straddle frame at 0.75, alone or with the dense clutter's cells appended (which sends the frame
    down the sequential path without adding a candidate to any straddle query)."""
    fr, keeps = E.grid_lines_straddle()
    if overflow:
        c = E.lines_dense_clutter()
        q, tl, td = SS.stereo_cells_lines(c[0], c[4], E.W, E.H)
        fr = (np.concatenate([fr[0], q]), np.concatenate([fr[1], c[3]]), np.concatenate([fr[2], tl]),
              np.concatenate([fr[3], td]), np.concatenate([fr[4], c[5]]))
        assert E.window_candidates_lines(fr[0], fr[2], W_STEREO) > 128
    return fr, keeps


@pytest.mark.parametrize("overflow", [False, True])
@pytest.mark.parametrize("best_lr", [True, False])
def test_gpu_match_grid_lines_edges(engine, oracle, overflow, best_lr):
    straddle, keeps = _straddle_grid_frames(overflow)
    frames = [SS.make_stereo_lines(150, 160, seed=700), straddle, E.grid_lines_raster()[0], SS.make_stereo_lines(3, 0, seed=701)]
    for f in raw_line_frames():
        q, tl, td = SS.stereo_cells_lines(f[0], f[4], E.W, E.H)
        frames.append((q, f[3], tl, td, f[5]))
    q_off, t_off = _offsets(frames, 1), _offsets(frames, 4)
    total, m12, counts = engine.match_grid_lines(q_off, _cat(frames, 0, 4), _cat(frames, 1, 32), t_off, _cat(frames, 2, 4),
                                                 _cat(frames, 3, 2), _cat(frames, 4, 32), W_STEREO, 0.9, 0.75, best_lr)
    # the designed straddle queries first: each one's only candidate is kept exactly when the unfused |dot| keeps it
    n_s = len(keeps)
    got = m12[q_off[1]:q_off[1] + n_s]
    want = np.where(keeps, np.arange(n_s), -1)
    assert np.array_equal(got, want), f"straddle queries: got {got.tolist()}, want {want.tolist()}"
    for k, f in enumerate(frames):
        n_ref, ref = SR.match_grid_lines(*f, W_STEREO, 0.9, 0.75, best_lr)
        n_o, m_o = oracle.match_grid_lines(*f, W_STEREO, 0.9, 0.75, best_lr)
        np.testing.assert_array_equal(m_o, ref, err_msg=f"oracle, frame {k}")
        np.testing.assert_array_equal(m12[q_off[k]:q_off[k + 1]], ref, err_msg=f"frame {k}")
        assert counts[k] == n_ref == n_o, k
    assert total == counts.sum()


# ------------------------------------------------------------------------------------------- matchStereoPoints / Lines
def _configs():
    mc, sc = T.default_stereo_match_config(), T.default_stereo_config()
    kitti = T.default_stereo_match_config()
    kitti.min_ratio_12_p = 0.75
    sk = T.default_stereo_config()
    sk.max_dist_epip = 0.0
    return [(mc, sc), (kitti, sk)]


@pytest.mark.parametrize("cfg", [0, 1])
def test_gpu_match_stereo_points_edges(engine, cfg):
    mc, sc = _configs()[cfg]
    frames = raw_point_frames()
    l_off, r_off = _offsets(frames, 0), _offsets(frames, 3)
    total, out = engine.match_stereo_points(CAM, mc, sc, l_off, _cat(frames, 0, 2), _cat(frames, 1, 0), _cat(frames, 2, 32),
                                            r_off, _cat(frames, 3, 2), _cat(frames, 4, 32))
    tot = 0
    for p, f in enumerate(frames):
        k, ref = SR.match_stereo_points(CAM, mc, sc, *f)
        assert out["counts"][p] == k, p
        a = l_off[p]
        for key in KEYS_PT:
            _same(out[key][a:a + k], ref[key], (p, key))
        tot += k
    assert total == tot


def _run_lines(engine, mc, sc, frames):
    l_off, r_off = _offsets(frames, 0), _offsets(frames, 4)
    total, out = engine.match_stereo_lines(CAM, mc, sc, l_off, _cat(frames, 0, 4), _cat(frames, 1, 0), _cat(frames, 2, 0),
                                           _cat(frames, 3, 32), r_off, _cat(frames, 4, 4), _cat(frames, 5, 32))
    tot = 0
    for p, f in enumerate(frames):
        k, ref = SR.match_stereo_lines(CAM, mc, sc, *f)
        assert out["counts"][p] == k, p
        a = l_off[p]
        for key in KEYS_LS:
            _same(out[key][a:a + k], ref[key], (p, key))
        tot += k
    assert total == tot
    return l_off, out


@pytest.mark.parametrize("cfg", [0, 1])
def test_gpu_match_stereo_lines_edges(engine, cfg):
    mc, sc = _configs()[cfg]
    _run_lines(engine, mc, sc, raw_line_frames())


@pytest.mark.parametrize("overflow", [False, True])
def test_gpu_match_stereo_lines_straddles(engine, overflow):
    """Per crafted pair, line_sim_th is set to where its unfused and fused |dot| part: the pair's left line is matched
    (and lifted) exactly when the reference keeps it, on the fast path and, with the dense clutter appended to the
    frame, on the sequential path."""
    mc, sc = T.default_stereo_match_config(), T.default_stereo_config()
    for i, (fr, th, keep) in enumerate(E.fused_line_straddles()):
        if overflow:
            fr = E.merge_line_frames(fr, E.lines_dense_clutter())
        mc.line_sim_th = th
        frames = [SS.make_stereo_frame_lines(90, 95, seed=800 + i), fr, SS.make_stereo_frame_lines(40, 30, seed=900 + i)]
        l_off, out = _run_lines(engine, mc, sc, frames)
        got = int(out["m12"][l_off[1]])
        assert got == (0 if keep else -1), f"straddle {i} (th {th!r}, reference keeps: {keep}): m12 = {got}"


# ------------------------------------------------------------------------------------------------------ the tracker
def test_gpu_track_stereo_batch_edges(engine):
    """plstvo_track_stereo_batch on pairs built from the edge frames: n_stereo equals the reference's survivor counts of
    every frame, the straddle frames included (line_sim_th set to the first straddle's threshold, so that pair's line
    count shows which side the kernel took)."""
    mc, sc, cfg = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    straddles = E.fused_line_straddles()
    fr_s, th, keep = straddles[0]
    mc.line_sim_th = th
    pts = raw_point_frames()
    lns = raw_line_frames() + [fr_s, E.merge_line_frames(fr_s, E.lines_dense_clutter())]
    B = max(len(pts), len(lns)) // 2 + 1

    def frame(k, which):
        p, l = pts[(2 * k + which) % len(pts)], lns[(2 * k + which) % len(lns)]
        return p, l

    def features(which):
        fs = [frame(k, which) for k in range(B)]
        P, L = [f[0] for f in fs], [f[1] for f in fs]
        return dict(pl_off=_offsets(P, 0), pr_off=_offsets(P, 3), kp_l=_cat(P, 0, 2), kp_r=_cat(P, 3, 2), poct_l=_cat(P, 1, 0),
                    pdesc_l=_cat(P, 2, 32), pdesc_r=_cat(P, 4, 32), ll_off=_offsets(L, 0), lr_off=_offsets(L, 4),
                    seg_l=_cat(L, 0, 4), seg_r=_cat(L, 4, 4), angle_l=_cat(L, 1, 0), loct_l=_cat(L, 2, 0), ldesc_l=_cat(L, 3, 32),
                    ldesc_r=_cat(L, 5, 32)), fs
    prev, fp = features(0)
    curr, fc = features(1)
    res, n_stereo = engine.track_stereo_batch(CAM, cfg, mc, sc, prev, curr)
    want = np.zeros((B, 4), np.int32)
    for k in range(B):
        for j, (p, l) in enumerate((fp[k], fc[k])):
            want[k, 2 * j] = SR.match_stereo_points(CAM, mc, sc, *p)[0]
            want[k, 2 * j + 1] = SR.match_stereo_lines(CAM, mc, sc, *l)[0]
    np.testing.assert_array_equal(n_stereo, want)
    # the straddle frame's single line is counted exactly when the reference keeps it
    at = [(k, 2 * j + 1) for k in range(B) for j in (0, 1) if (fp, fc)[j][k][1] is fr_s]
    assert at, "the straddle frame is in the batch"
    assert all(n_stereo[k, c] == int(keep) for k, c in at), (at, keep)
