"""Parity of the CUDA matcher (K1 + finalize, through the C-ABI) with the oracle and the committed
cv2.BFMatcher golden vectors: match indices must be BIT-EXACT."""
import glob
import os

import numpy as np
import pytest

import ref_match
from conftest import GOLDEN
from stvo_pl_b200 import synth, types as T

pytestmark = pytest.mark.gpu
CASES = sorted(glob.glob(os.path.join(GOLDEN, "match_*.npz")))


@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[6:-4] for p in CASES])
def test_match_vs_cv2_golden(engine, path):
    g = np.load(path)
    d1, d2, nnr = g["d1"], g["d2"], float(g["nnr"])
    if len(d2) >= 2:
        n, m12 = engine.match_nnr(d1, d2, nnr)
        np.testing.assert_array_equal(m12, g["m12_nnr"])
        assert n == int((m12 >= 0).sum())
    n, m = engine.match(d1, d2, nnr, True)
    np.testing.assert_array_equal(m, g["m12_mutual"])
    assert n == int((m >= 0).sum())


@pytest.mark.parametrize("n1,n2,mode", [
    (2000, 2000, "random"), (2000, 2000, "synth"), (500, 500, "synth"), (1000, 300, "ties"),
    (257, 1025, "ties"), (1, 2, "random"), (2, 1, "random"), (255, 256, "random"), (256, 513, "dup"),
    (3000, 700, "random"), (33, 31, "ties")])
def test_match_vs_oracle(engine, oracle, n1, n2, mode):
    rng = np.random.default_rng(n1 * 7919 + n2)
    if mode == "random":
        d1, d2 = rng.integers(0, 256, (n1, 32), dtype=np.uint8), rng.integers(0, 256, (n2, 32), dtype=np.uint8)
    elif mode == "ties":
        d1 = (rng.integers(0, 2, (n1, 32), dtype=np.uint8) * 255).astype(np.uint8)
        d2 = (rng.integers(0, 2, (n2, 32), dtype=np.uint8) * 255).astype(np.uint8)
    elif mode == "dup":
        d1, d2 = np.zeros((n1, 32), np.uint8), np.zeros((n2, 32), np.uint8)
        d1[:, 0], d2[:, 0] = rng.integers(0, 3, n1), rng.integers(0, 3, n2)
    else:
        prev, curr, _, _ = synth.make_batch("kitti", 1, n_pt=max(n1, n2), n_ls=0)
        d1, d2 = prev.pdesc[:n1], curr.pdesc[:n2]
    for nnr in (0.75, 0.9, 1.0, 1.5):   # nnr > 1 accepts ties d1 == d2: the lowest index must win
        for best_lr in (True, False):
            n_ref, ref = oracle.match(d1, d2, nnr, best_lr)
            n, m = engine.match(d1, d2, nnr, best_lr)
            np.testing.assert_array_equal(m, ref)
            assert n == n_ref


@pytest.mark.gpu
@pytest.mark.parametrize("n1,n2", [(300, 65535), (65535, 300), (20000, 20000)])
def test_match_at_the_feature_limit(engine, oracle, n1, n2):
    """Matching-only calls take any frame up to PLSTVO_MAX_FEATURES = 65535 rows per side (the per-pair solver's shared-memory
    limits do not apply to them; the mutual filter's scratch holds 16-bit indices so that 65535 rows fit one CTA)."""
    rng = np.random.default_rng(n1 + 3 * n2)
    d1, d2 = rng.integers(0, 256, (n1, 32), dtype=np.uint8), rng.integers(0, 256, (n2, 32), dtype=np.uint8)
    k = min(n1, n2, 5000)
    pick1, pick2 = rng.permutation(n1)[:k], rng.permutation(n2)[:k]
    d2[pick2] = d1[pick1] ^ (rng.random((k, 32)) < 0.03).astype(np.uint8)     # true correspondences somewhere in the frames
    n_ref, ref = oracle.match(d1, d2, 0.75, True, threads=True) if n1 * n2 > 10**8 else oracle.match(d1, d2, 0.75, True)
    n, m = engine.match(d1, d2, 0.75, True)
    np.testing.assert_array_equal(m, ref)
    assert n == n_ref and n > k // 2


def test_match_batch_ragged(engine, oracle):
    """Several problems of different sizes in one launch, including empty sides."""
    rng = np.random.default_rng(5)
    sizes = [(300, 280), (0, 50), (40, 0), (1, 1), (513, 700), (64, 2), (1500, 1500)]
    d1 = rng.integers(0, 256, (sum(s[0] for s in sizes), 32), dtype=np.uint8)
    d2 = rng.integers(0, 256, (sum(s[1] for s in sizes), 32), dtype=np.uint8)
    # plant true matches in the last problem
    d2[-1500:] = d1[-1500:][rng.permutation(1500)] ^ (rng.random((1500, 32)) < 0.05).astype(np.uint8)
    off1 = np.concatenate([[0], np.cumsum([s[0] for s in sizes])]).astype(np.int32)
    off2 = np.concatenate([[0], np.cumsum([s[1] for s in sizes])]).astype(np.int32)
    total, m12, counts = engine.match_batch(d1, off1, d2, off2, 0.75, True)
    for p, (a, b) in enumerate(sizes):
        n_ref, ref = oracle.match(d1[off1[p]:off1[p + 1]], d2[off2[p]:off2[p + 1]], 0.75, True)
        np.testing.assert_array_equal(m12[off1[p]:off1[p + 1]], ref)
        assert counts[p] == n_ref
    assert total == counts.sum() and counts[-1] > 1000


def _tie_rows(rng, n, patterns, flip):
    """n rows drawn from a few byte patterns; flip: each with 1 or 2 bits flipped, so that its best is tied among the
    pattern's copies at a distance above 0, where a ratio test with nnr > 1 accepts it"""
    rows = patterns[rng.integers(0, len(patterns), n)]
    return ref_match.flip_bits(rng, rows, 2) if flip else rows


def test_match_batch_accepted_ties(engine, oracle):
    """nnr 1.5, queries near a few byte patterns and trains copies of them: most rows and columns have tied bests that pass
    the ratio test, so the resolve step's lowest-index scan feeds the mutual filter's index form."""
    rng = np.random.default_rng(23)
    pats = (rng.integers(0, 2, (6, 32), dtype=np.uint8) * 255).astype(np.uint8)
    sizes = [(300, 280), (1, 7), (257, 513), (640, 129), (2, 2)]
    d1 = _tie_rows(rng, sum(s[0] for s in sizes), pats, True)
    d2 = _tie_rows(rng, sum(s[1] for s in sizes), pats, False)
    off1 = np.concatenate([[0], np.cumsum([s[0] for s in sizes])]).astype(np.int32)
    off2 = np.concatenate([[0], np.cumsum([s[1] for s in sizes])]).astype(np.int32)
    for best_lr in (True, False):
        total, m12, counts = engine.match_batch(d1, off1, d2, off2, 1.5, best_lr)
        for p in range(len(sizes)):
            n_ref, ref = oracle.match(d1[off1[p]:off1[p + 1]], d2[off2[p]:off2[p + 1]], 1.5, best_lr)
            np.testing.assert_array_equal(m12[off1[p]:off1[p + 1]], ref)
            assert counts[p] == n_ref
        assert total == counts.sum() and total > 0


def test_track_batch_accepted_ties(engine, oracle):
    """The same accepted ties through the per-pair solver's own finalize (K2): match indices equal the oracle's."""
    rng = np.random.default_rng(31)
    prev, curr, _, cam = synth.make_batch("kitti", 2, n_pt=600, n_ls=150)
    pats = (rng.integers(0, 2, (6, 32), dtype=np.uint8) * 255).astype(np.uint8)
    for f in (prev, curr):
        f.pdesc = np.ascontiguousarray(_tie_rows(rng, len(f.pdesc), pats, f is prev))
        f.ldesc = np.ascontiguousarray(_tie_rows(rng, len(f.ldesc), pats, f is prev))
    cfg = T.kitti_config()
    cfg.min_ratio_12_p = cfg.min_ratio_12_l = 1.5
    gpu = engine.track_batch(cam, cfg, prev, curr)
    ref = oracle.track_batch(cam, cfg, prev, curr)
    np.testing.assert_array_equal(gpu["m12_pt"], ref["m12_pt"])
    np.testing.assert_array_equal(gpu["m12_ls"], ref["m12_ls"])
    assert (gpu["m12_pt"] >= 0).sum() > 0


def test_selected_matcher_form(engine):
    """The tensor-core matcher is the one that runs: asserted on the plan a resident batch reports (its form and its work items,
    one per 256-train block) and on the shapes of the matcher's intermediate words."""
    prev, curr, _, cam = synth.make_batch("kitti", 2, n_pt=600, n_ls=150)
    cfg = T.kitti_config()
    db = engine.upload(cam, cfg, prev, curr)
    try:
        st = db.stage_times(iters=1)
    finally:
        db.free()
    assert st["tensor_core_form"] is True
    n2 = np.concatenate([np.diff(curr.pt_off), np.diff(curr.ls_off)])
    assert st["n_items"] == int(((n2 + 255) // 256).sum())   # work items: 256-train blocks
    rowp, colp, rowkey, colkey = engine.debug_tc_partials(prev.pdesc[:5], [0, 5], curr.pdesc[:3], [0, 3], 0.9)
    assert len(rowp) == 5 and len(colp) == 3 and rowkey.shape == (5, 2) and colkey.shape == (3, 2)


def test_match_full_size_properties(engine):
    """BASELINE full size (C5: 8000 x 8000): size-independent properties — mutual matches are a partial
    permutation, planted correspondences are recovered, matching d against itself is the identity."""
    rng = np.random.default_rng(11)
    n = 8000
    d1 = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    perm = rng.permutation(n)
    d2 = d1[perm].copy()
    flip = rng.random((n, 32)) < 0.02
    d2 ^= (flip * rng.integers(1, 256, (n, 32))).astype(np.uint8)
    cnt, m = engine.match(d1, d2, 0.75, True)
    inv = np.empty(n, np.int64)
    inv[perm] = np.arange(n)
    assert cnt == int((m >= 0).sum()) and cnt > 0.99 * n
    sel = m >= 0
    np.testing.assert_array_equal(m[sel], inv[sel])           # recovered the planted permutation
    assert len(np.unique(m[sel])) == sel.sum()                # one-to-one
    cnt, m = engine.match(d1, d1, 0.75, True)
    np.testing.assert_array_equal(m, np.arange(n))            # distance 0 < 0.75 * d2
    # symmetry: match(d2, d1) is the inverse map on the mutual set
    cnt2, m21 = engine.match(d2, d1, 0.75, True)
    cnt1, m12 = engine.match(d1, d2, 0.75, True)
    assert cnt1 == cnt2
    s = m12 >= 0
    np.testing.assert_array_equal(m21[m12[s]], np.nonzero(s)[0])


def test_f2f_tracking_vs_oracle(engine, oracle):
    cfg = T.kitti_config()
    prev, curr, _, _ = synth.make_batch("kitti", 3, n_pt=700, n_ls=200)
    rc, ref_pt, ref_ls, ref_n = oracle.f2f_tracking(cfg, prev, curr)
    m12_pt, m12_ls, n = engine.f2f_tracking(cfg, prev, curr)
    np.testing.assert_array_equal(m12_pt, ref_pt)
    np.testing.assert_array_equal(m12_ls, ref_ls)
    np.testing.assert_array_equal(n, ref_n)
    cfg.has_lines = 0
    m12_pt, m12_ls, n = engine.f2f_tracking(cfg, prev, curr)
    np.testing.assert_array_equal(m12_pt, ref_pt)
    assert (m12_ls == -1).all() and (n[:, 1] == 0).all()


def test_errors(engine):
    from stvo_pl_b200.engine import PlstvoError
    d = np.zeros((4, 32), np.uint8)
    with pytest.raises(PlstvoError):
        engine._ck(engine.lib.plstvo_match(engine.ctx, d.ctypes.data_as(T.c_uint8_p), 4, d.ctypes.data_as(T.c_uint8_p),
                                           4, 64, 0.9, 1, np.zeros(4, np.int32).ctypes.data_as(T.c_int32_p)))
    big = np.zeros((70000, 32), np.uint8)
    with pytest.raises(PlstvoError) as ei:
        engine.match(big, d, 0.9)
    assert ei.value.code == -2


def test_one_context_shared_by_threads(engine):
    """The reference calls the matcher from up to four std::async tasks of one handler (src/stereoFrameHandler.cpp:113-119,
    src/matching.cpp:68-74): a context shared by threads must serialise its entry points.  Four threads hammer one context with
    different problems (ctypes releases the GIL); every result equals the single-threaded one."""
    from concurrent.futures import ThreadPoolExecutor
    rng = np.random.default_rng(5)
    probs = [(rng.integers(0, 256, (n1, 32), dtype=np.uint8), rng.integers(0, 256, (n2, 32), dtype=np.uint8))
             for n1, n2 in [(900, 800), (300, 1200), (1500, 1500), (64, 77), (2000, 500), (700, 700)]]
    ref = [engine.match(d1, d2, 0.9, True)[1].copy() for d1, d2 in probs]
    prev, curr, _, cam = synth.make_batch("kitti", 2, n_pt=600, n_ls=150)
    cfg = T.kitti_config()
    ref_pose = engine.track_batch(cam, cfg, prev, curr)["results"].tobytes()

    def job(i):
        k = i % (len(probs) + 1)
        if k == len(probs):
            return ("pose", engine.track_batch(cam, cfg, prev, curr)["results"].tobytes())
        return (k, engine.match(probs[k][0], probs[k][1], 0.9, True)[1].copy())
    with ThreadPoolExecutor(4) as ex:
        outs = list(ex.map(job, range(56)))
    for key, val in outs:
        if key == "pose":
            assert val == ref_pose
        else:
            np.testing.assert_array_equal(val, ref[key])
