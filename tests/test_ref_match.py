"""Pins the NumPy restatement of the matcher's intermediate words (tests/ref_match.py) to the C oracle, which the cv2.BFMatcher
goldens pin in turn: the reference's keys, finalized with the device's rules, must give the oracle's m12 at every ratio,
including nnr > 1, where a tie d1 == d2 passes the ratio test and the lowest index must be chosen.  No GPU needed."""
import numpy as np
import pytest

import ref_match as R

N1 = (1, 2, 65, 128, 257, 640)
N2 = (1, 2, 129, 256, 257, 640)
RATIOS = (0.75, 0.9, 1.0, 1.5)


def _check(oracle, d1, d2):
    D = R.hamming_matrix(d1, d2)
    if len(d2) >= 2:   # distances and lowest-index order against the oracle's knn2
        idx, dist = oracle.knn2(d1, d2)
        S = np.sort(D, axis=1)
        np.testing.assert_array_equal(dist[:, 0], S[:, 0])
        np.testing.assert_array_equal(dist[:, 1], S[:, 1])
        np.testing.assert_array_equal(idx[:, 0], D.argmin(axis=1))
    for nnr in RATIOS:
        rowkey, colkey = R.resolved_keys(D, nnr)
        for best_lr in (True, False):
            m12, n = R.finalize(rowkey, colkey, len(d1), nnr, best_lr)
            n_ref, ref = oracle.match(d1, d2, nnr, best_lr)
            np.testing.assert_array_equal(m12, ref, err_msg=f"nnr {nnr} best_lr {best_lr}")
            assert n == n_ref


@pytest.mark.parametrize("family", R.FAMILIES)
def test_reference_matches_oracle(oracle, family):
    rng = np.random.default_rng(sum(map(ord, family)))
    for n1 in N1:
        for n2 in N2:
            _check(oracle, *R.make_family(family, n1, n2, rng))


def test_reference_matches_oracle_beyond_unresolved_limit(oracle):
    """n1 > 65024: column keys carry real query indices and the mutual filter compares indices."""
    rng = np.random.default_rng(3)
    _check(oracle, *R.make_family("planted", R.M21_DIST + 300, 40, rng))
    _check(oracle, *R.make_family("ties", R.M21_DIST + 300, 40, rng))


def test_row_words_by_brute_force():
    """Block top-2 words and tag decoding against a per-element loop on a small ragged case."""
    rng = np.random.default_rng(9)
    d1, d2 = R.make_family("ties", 5, 600, rng)
    D = R.hamming_matrix(d1, d2)
    best, second, unique, arg = R.row_words(D)
    for b in range(3):
        blk = D[:, 256 * b:256 * b + 256]
        for x in range(5):
            v = sorted(blk[x].tolist())
            assert best[b, x] == v[0] and second[b, x] == (v[1] if len(v) > 1 else R.NONE)
            assert unique[b, x] == (len(v) == 1 or v[0] != v[1])
            assert arg[b, x] == 256 * b + int(np.argmin(blk[x]))
    # a tag names train 256 b + 32 g + 8 i + 2 l + p for some i in 0..3
    for j in range(256):
        g, i, l, p = j // 32, (j % 32) // 8, (j % 8) // 2, j % 2
        assert 32 * g + 8 * i + 2 * l + p == j
        assert R.row_tag_hits(np.array([p | g << 1 | l << 4]), np.array([256 + j]))[0]
        assert not R.row_tag_hits(np.array([(p ^ 1) | g << 1 | l << 4]), np.array([256 + j]))[0]
