"""Exact check of the tensor-core matcher's intermediate words (match_tc.cu) against the NumPy reference (tests/ref_match.py).

The final match indices hide three kinds of error in tc_hamming_kernel: a wrong candidate tag only costs speed, because
tc_resolve_kernel falls back to a scan of all trains; a zero or stale operand row or column that leaks into a top-2 reads as
distance 128, which never beats the nearest neighbour of random descriptors; a wrong second distance only shows when it
flips a ratio test.  So this test reads every row and column word and every resolved key through plstvo_debug_tc_partials
and requires them to equal the reference, and every unique-best tag to name the argmin.

The grid below runs as one batch call of about 600 work items (more than four per SM), so every CTA of the persistent kernel
wraps its work-item ring and carries its query-stage phase and train-buffer parity across items of mixed lengths."""
import numpy as np
import pytest

import ref_match as R

pytestmark = pytest.mark.gpu

# query tiles are 128 rows (two warpgroups of 64); 640 and 1025 rows are more tiles than the 4 query stages
N1 = (1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 640, 1025)
# train blocks are 256 (two halves of 128): one half only, one train in a half, a lone half after a full block
N2 = (1, 2, 127, 128, 129, 255, 256, 257, 383, 384, 385, 640, 1025)


def _mismatch(name, got, want, where):
    bad = np.nonzero(np.asarray(got) != np.asarray(want))
    if not len(bad[0]):
        return []
    first = tuple(int(a[0]) for a in bad)
    return [f"{where}: {len(bad[0])} {name} differ, first at {first}: got {got[first]:#x}, want {want[first]:#x}"]


def check_problem(where, d1, d2, nnr, rowp, colp, rowkey, colkey):
    """Failure messages (empty: all equal) and how many unique-best row / column tags were checked."""
    n1, n2 = len(d1), len(d2)
    D = R.hamming_matrix(d1, d2)
    errs = []
    best, second, unique, arg = R.row_words(D)
    rw = rowp.reshape(best.shape)
    errs += _mismatch("row words", rw & 0x3FFFF, R.pack_word(best, second), where)
    hits = R.row_tag_hits(rw >> 18, arg)
    if (unique & ~hits).any():
        b, x = (int(a[0]) for a in np.nonzero(unique & ~hits))
        errs.append(f"{where}: {int((unique & ~hits).sum())} row tags miss the unique best, first block {b} query {x}: "
                    f"tag {int(rw[b, x] >> 18):#x}, argmin {int(arg[b, x])}")
    cb, cs, cu, carg = R.col_words(D)
    errs += _mismatch("column words", colp & 0x3FFFF, R.pack_word(cb, cs), where)
    ctag, want_tag = (colp >> 18).astype(np.int64), (carg % 128) // 16
    if (cu & (ctag != want_tag)).any():
        y = int(np.nonzero(cu & (ctag != want_tag))[0][0])
        errs.append(f"{where}: column tags miss the unique best, first train {y}: tag {ctag[y]}, argmin row {int(carg[y])}")
    rk, ck = R.resolved_keys(D, nnr)
    errs += _mismatch("row keys", rowkey, rk, where)
    errs += _mismatch("column keys", colkey, ck, where)
    return errs, int(unique.sum()), int(cu.sum())


def run_and_check(engine, problems, nnr):
    """problems: [(label, d1, d2)] as one batch call"""
    d1 = np.concatenate([p[1] for p in problems])
    d2 = np.concatenate([p[2] for p in problems])
    off1 = np.concatenate([[0], np.cumsum([len(p[1]) for p in problems])]).astype(np.int32)
    off2 = np.concatenate([[0], np.cumsum([len(p[2]) for p in problems])]).astype(np.int32)
    rowp, colp, rowkey, colkey = engine.debug_tc_partials(d1, off1, d2, off2, nnr)
    errs, n_row_tags, n_col_tags, r0 = [], 0, 0, 0
    for p, (label, a, b) in enumerate(problems):
        nrow = (len(b) + 255) // 256 * len(a)
        e, nr, nc = check_problem(f"{label} {len(a)}x{len(b)} nnr {nnr}", a, b, nnr, rowp[r0:r0 + nrow],
                                  colp[off2[p]:off2[p + 1]], rowkey[off1[p]:off1[p + 1]], colkey[off2[p]:off2[p + 1]])
        errs += e
        n_row_tags += nr
        n_col_tags += nc
        r0 += nrow
    assert r0 == len(rowp)
    assert not errs, "\n".join(errs[:30])
    return n_row_tags, n_col_tags


@pytest.mark.parametrize("nnr", [0.8, 1.5])
def test_partials_boundary_grid(engine, nnr):
    """Every (n1, n2) of the grid twice, each descriptor family meeting every boundary class: family = (i1 + i2) % 6 in one
    pass and (i1 + 2 i2 + 3) % 6 in the other.  nnr 1.5 accepts ties, so the lowest-index scan of the resolve step is reached;
    at 0.8 many rows fail the ratio test and carry index 0."""
    rng = np.random.default_rng(17)
    problems = []
    for pick in (lambda i1, i2: i1 + i2, lambda i1, i2: i1 + 2 * i2 + 3):
        for i1, n1 in enumerate(N1):
            for i2, n2 in enumerate(N2):
                fam = R.FAMILIES[pick(i1, i2) % len(R.FAMILIES)]
                problems.append((fam, *R.make_family(fam, n1, n2, rng)))
    items = sum((len(p[2]) + 255) // 256 for p in problems)
    assert items > 4 * engine_sm_count()
    n_row_tags, n_col_tags = run_and_check(engine, problems, nnr)
    assert n_row_tags > 10000 and n_col_tags > 5000


@pytest.mark.parametrize("n1,n2,family,nnr", [
    (65535, 300, "planted", 1.5),   # n1 > 65024: unique column bests are resolved through the column warp tag
    (300, 65535, "far", 0.9),       # 256 train blocks, the last one 255 trains; zero columns would read as 128
    (8000, 8000, "planted", 0.75)])  # the C5 frame size
def test_partials_large(engine, n1, n2, family, nnr):
    rng = np.random.default_rng(n1 + 7 * n2)
    run_and_check(engine, [(family, *R.make_family(family, n1, n2, rng))], nnr)


def engine_sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count
