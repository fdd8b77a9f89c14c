"""Plain NumPy restatement of the tensor-core matcher's intermediate words (stvo_pl_b200/csrc/match_tc.cu), used to check
them exactly (tests/test_gpu_match_partials.py) and, through the same finalize rules, against the C oracle
(tests/test_ref_match.py).  Distances come from np.bitwise_count on XOR-ed uint64 views, computed in row chunks.

Word layouts (include/plstvo.h: plstvo_debug_tc_partials):
  row word  [256-train block][n1]: best | second << 9 | tag << 18, tag = parity | chunk group << 1 | lane << 4;
  col word  [n2]:                  best | second << 9 | tag << 18, tag = consumer warp = (row % 128) // 16;
  511 = no second value (one train in the block / one query).  Resolved keys: (d1 << 16 | index, d2 << 16 | 0xFFFE).
"""
from __future__ import annotations

import numpy as np

BLOCK = 256                  # trains per row-word block (TC_CW)
NONE = 511                   # "no value" in a word's 9-bit distance fields
KEY_NONE = 0xFFFFFFFF
KEY_IDX_UNRESOLVED = 0xFFFD  # column key of a unique best whose query index the resolve step does not recover
SECOND_IDX = 0xFFFE          # index field of every second key
M21_DIST = 0xFE00            # largest n1 whose unique column bests stay unresolved (match_finalize.cuh)
_PAD = 1023                  # padding distance of a partial block, above every real one


def hamming_matrix(d1, d2, budget=1 << 23):
    """[n1, n2] uint16 Hamming distances of 32-byte rows."""
    a = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32).view(np.uint64)
    b = np.ascontiguousarray(d2, np.uint8).reshape(-1, 32).view(np.uint64)
    D = np.empty((len(a), len(b)), np.uint16)
    step = max(1, budget // max(1, len(b)))
    for r in range(0, len(a), step):
        x = a[r:r + step, None, :] ^ b[None, :, :]
        D[r:r + step] = np.bitwise_count(x).sum(axis=2, dtype=np.uint16)
    return D


def _top2(X, axis):
    """(best, second) along axis, duplicates counted; second = NONE when the axis has one entry."""
    if X.shape[axis] < 2:
        best = X.min(axis=axis).astype(np.int64)
        return best, np.full_like(best, NONE)
    P = np.partition(X, 1, axis=axis)
    return np.take(P, 0, axis=axis).astype(np.int64), np.take(P, 1, axis=axis).astype(np.int64)


def row_words(D):
    """Per 256-train block b and query x: best, second (NONE past a one-train block), unique-best flag and the block-global
    argmin.  Arrays [nblk, n1]."""
    n1, n2 = D.shape
    nblk = (n2 + BLOCK - 1) // BLOCK
    P = np.full((n1, nblk * BLOCK), _PAD, np.uint16)
    P[:, :n2] = D
    P = P.reshape(n1, nblk, BLOCK)
    best, second = _top2(P, 2)
    second = np.where(second >= _PAD, NONE, second)
    arg = P.argmin(axis=2) + BLOCK * np.arange(nblk)[None, :]
    return best.T, second.T, best.T != second.T, arg.T


def col_words(D):
    """Per train: best and second over all queries (NONE when n1 = 1), unique-best flag, lowest argmin."""
    best, second = _top2(D, 0)
    return best, second, best != second, D.argmin(axis=0)


def pack_word(best, second):
    return (np.asarray(best, np.uint32) | (np.asarray(second, np.uint32) << 9))


def row_tag_hits(tags, arg):
    """True where a row tag names the block's unique argmin among the four trains tc_resolve_kernel re-checks:
    256 b + 32 group + 8 i + 2 lane + parity, i = 0..3."""
    j = np.asarray(arg, np.int64) % BLOCK
    tags = np.asarray(tags, np.int64)
    return (j // 32 == (tags >> 1) & 7) & ((j % 8) // 2 == (tags >> 4) & 3) & (j % 2 == tags & 1)


def ratio_pass(d1, d2, nnr):
    """The reference's float ratio test: dist1 < dist2 * nnr, all float32 (src/matching.cpp:54)."""
    return np.asarray(d1, np.float32) < np.asarray(d2, np.float32) * np.float32(nnr)


def _keys(D, axis, nnr, unresolved):
    """Resolved keys along one direction (axis = 1: rows over trains, axis = 0: columns over queries)."""
    other = D.shape[axis]
    d1, d2 = _top2(D, axis)
    idx = D.argmin(axis=axis).astype(np.int64)       # lowest index at the best distance, ties included
    if other < 2:
        return np.stack([(d1 << 16).astype(np.uint32), np.full(len(d1), KEY_NONE, np.uint32)], axis=1)
    ok = ratio_pass(d1, d2, nnr)
    if unresolved:
        idx = np.where(d1 != d2, KEY_IDX_UNRESOLVED, idx)
    idx = np.where(ok, idx, 0)
    return np.stack([((d1 << 16) | idx).astype(np.uint32), ((d2 << 16) | SECOND_IDX).astype(np.uint32)], axis=1)


def resolved_keys(D, nnr):
    """(rowkey [n1, 2], colkey [n2, 2]) as tc_resolve_kernel writes them."""
    n1 = D.shape[0]
    return _keys(D, 1, nnr, False), _keys(D, 0, nnr, n1 <= M21_DIST)


def finalize(rowkey, colkey, n1, nnr, best_lr):
    """m12 and the match count from one merged key pair per row and column (match_finalize.cuh, one-partial path): ratio
    test, then the mutual filter, where an unresolved column key matches the query whose best distance equals it."""
    rowkey, colkey = np.asarray(rowkey, np.int64), np.asarray(colkey, np.int64)

    def accept(k):
        return (k[:, 1] != KEY_NONE) & ratio_pass(k[:, 0] >> 16, k[:, 1] >> 16, nnr)
    m12 = np.where(accept(rowkey), rowkey[:, 0] & 0xFFFF, -1)
    if best_lr and len(colkey):
        dist_form = n1 <= M21_DIST
        cacc = accept(colkey)
        sel = np.nonzero(m12 >= 0)[0]
        t = m12[sel]
        ck = colkey[t, 0]
        unres = dist_form & ((ck & 0xFFFF) == KEY_IDX_UNRESOLVED)
        mutual = cacc[t] & np.where(unres, (ck >> 16) == (rowkey[sel, 0] >> 16), (ck & 0xFFFF) == sel)
        m12[sel[~mutual]] = -1
    return m12.astype(np.int32), int((m12 >= 0).sum())


# ---- descriptor families ----------------------------------------------------------------------------------------------
FAMILIES = ("random", "planted", "far", "ties", "extremes", "repeat")


def flip_bits(rng, rows, max_bits):
    """rows with 1 .. max_bits random bits flipped each"""
    out = rows.copy()
    for r in range(len(out)):
        bits = rng.choice(256, int(rng.integers(1, max_bits + 1)), replace=False)
        for b in bits:
            out[r, b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def make_family(kind, n1, n2, rng):
    """(d1 [n1, 32], d2 [n2, 32]) uint8 for one matching problem:
    random    uniform bytes;
    planted   uniform, plus correspondences at distance <= 8 (ratio tests pass, indices matter);
    far       bytes 0..19 are 0x00 in every query and 0xFF in every train: every real distance is >= 160, so a zero operand
              row or column that leaks into a top-2 shows up as 128;
    ties      rows drawn from a handful of 0x00 / 0xFF byte patterns: exact duplicates inside a block, across its two halves
              and across blocks; every other query has 1 or 2 bits flipped, so its tied best is not at distance 0;
    extremes  a query's copy (distance 0) and its complement (distance 256) in the same block; with n2 = 1 the only train is
              query 0's complement;
    repeat    trains repeated 256 apart (within a block when n2 <= 256), near queries planted on them: the best is tied
              across blocks and the lower index must win."""
    d1 = rng.integers(0, 256, (n1, 32), dtype=np.uint8)
    d2 = rng.integers(0, 256, (n2, 32), dtype=np.uint8)
    if kind == "random":
        pass
    elif kind == "planted":
        k = min(n1, n2) // 2 + 1 if min(n1, n2) else 0
        k = min(k, n1, n2)
        i, j = rng.permutation(n1)[:k], rng.permutation(n2)[:k]
        d2[j] = flip_bits(rng, d1[i], 8)
    elif kind == "far":
        d1[:, :20] = 0x00
        d2[:, :20] = 0xFF
    elif kind == "ties":
        pats = (rng.integers(0, 2, (5, 32), dtype=np.uint8) * 255).astype(np.uint8)
        d1, d2 = pats[rng.integers(0, len(pats), n1)], pats[rng.integers(0, len(pats), n2)]
        odd = np.arange(1, n1, 2)
        d1[odd] = flip_bits(rng, d1[odd], 2)   # tied bests at distance 1 or 2, which a ratio above 1 accepts
    elif kind == "extremes":
        if n2 == 1:
            d2[0] = ~d1[0]
        else:
            for i in range(min(n1, n2 // 2)):
                blk = rng.integers(0, (n2 + BLOCK - 1) // BLOCK)
                lo, hi = blk * BLOCK, min(n2, blk * BLOCK + BLOCK)
                if hi - lo < 2:
                    lo, hi = 0, min(n2, BLOCK)
                j, jc = rng.choice(np.arange(lo, hi), 2, replace=False)
                d2[j], d2[jc] = d1[i], ~d1[i]
    elif kind == "repeat":
        gap = BLOCK if n2 > BLOCK else max(1, n2 // 2)
        if n2 > gap:
            src = rng.permutation(n2 - gap)[:max(1, min(n1, n2 - gap) // 2)]
            d2[src + gap] = d2[src]
            q = rng.permutation(n1)[:len(src)]
            d1[q] = flip_bits(rng, d2[src[:len(q)]], 4)
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(d1), np.ascontiguousarray(d2)
