"""Pins the yardstick of the pose-helper tests (CPU): the high-precision restatement in hp_pose.py against the oracle's
compiled helpers (oracle/plstvo_oracle.c) and the reference's own SE(3) code and the stand-in's 6x6 algebra
(oracle/ref.py), within the conditioning bounds hp_pose.py states.  Where the reference library cannot be built, its answers
are replayed from tests/golden/ref_pose_helpers.npz (re-record where the reference is present with
PLSTVO_RECORD_REF=1 python -m pytest tests/test_hp_pose_host.py)."""
import os
import re

import mpmath as mp
import numpy as np
import pytest

import hp_pose as HP
from conftest import GOLDEN
from oracle import ref as ref_mod

REF_CALLS = os.path.join(GOLDEN, "ref_pose_helpers.npz")


@pytest.fixture(scope="module")
def ref_store():
    if os.environ.get("PLSTVO_RECORD_REF"):
        store = ref_mod.Recorded(REF_CALLS, record=ref_mod.Ref())
        yield store
        store.save()
    else:
        yield ref_mod.Recorded(REF_CALLS)


@pytest.fixture
def ref(ref_store, request):
    ref_store.begin(request.node.name)
    return ref_store


def test_logmap_restatement_vs_oracle_and_reference(oracle, ref):
    cases = HP.log_cases(1)
    hit_nan = hit_small = 0
    for T in cases:
        o, r = oracle.logmap_se3(T), ref.logmap_se3(T)
        HP.check_log(o, T, "oracle")
        HP.check_log(r, T, "reference")
        # the oracle restates the reference's formula operation for operation: same NaN / inf pattern, same branch
        np.testing.assert_array_equal(np.isnan(o), np.isnan(r))
        np.testing.assert_array_equal(np.isinf(o), np.isinf(r))
        hit_nan += HP.cosine(T) == -1.0
        hit_small += 0.0 < float(np.arccos(HP.cosine(T))) <= 1e-6
    assert hit_nan > 0 and hit_small > 0, (hit_nan, hit_small)   # both branch edges are reached


def test_expmap_restatement_vs_oracle_and_reference(oracle, ref):
    rng = np.random.default_rng(2)
    e6 = 0.000001
    for k, mag in enumerate([np.nextafter(e6, 0), e6, np.nextafter(e6, 1), 1e-8, 1e-3, 1.0, np.pi - 1e-4, 3.0]):
        for axis in range(3):
            x = np.concatenate([rng.uniform(-1e3, 1e3, 3), np.zeros(3)])
            x[3 + axis] = mag if k % 2 == 0 else -mag      # one axis: |w| is exactly mag, so the branch is placed exactly
            want = HP.tonp(HP.expmap(x))
            b = HP.exp_bound(x)
            for got in (oracle.expmap_se3(x), ref.expmap_se3(x)):
                assert np.abs(got - want).max() <= b, (mag, axis, np.abs(got - want).max(), b)
                assert np.array_equal(got[:3, :3], np.eye(3)) == (mag < e6)   # the rotation branch, as the rule says


def test_eigenvalues_and_inverse_vs_restatement(oracle, ref):
    rng = np.random.default_rng(3)
    for k in range(24):
        q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
        lam = np.geomspace(1.0, 10.0 ** (k % 12), 6) * 10.0 ** rng.integers(-8, 3)
        if k >= 12:
            lam[: 2 + k % 5] = lam[0]                      # clusters of 2 to 6 equal eigenvalues
        A = (q * lam) @ q.T
        A = 0.5 * (A + A.T)
        want = [float(v) for v in HP.eigvals(A)]
        b = HP.eig_bound(A)
        for got in (oracle.eig6_sym(A), ref.eig6_sym(A)):
            assert np.abs(np.sort(got) - want).max() <= b, (k, np.abs(np.sort(got) - want).max(), b)
        Ai = HP.tonp(mp.inverse(HP.mpm(A)))
        bi = HP.C_SOLVE * HP.kappa(A) * HP.EPS * np.abs(Ai).max()
        for got in (oracle.inv6(A), ref.inv6(A)):
            assert np.abs(got - Ai).max() <= bi, (k, np.abs(got - Ai).max(), bi)


def test_unccomp_vs_restatement(oracle, ref):
    rng = np.random.default_rng(4)
    for d in HP.HALF_TURN[:-1]:
        T1 = HP.rodrigues(mp.pi - d, rng.normal(size=3), rng.uniform(-1e3, 1e3, 3))
        c1 = np.diag(rng.uniform(1e-6, 1e-1, 6)) + 1e-7 * np.ones((6, 6))
        J = rng.normal(size=(6, 6)) * np.array([1e-3, 1e-3, 1e-3, 1e-5, 1e-5, 1e-5])
        cinc = J @ J.T
        want, b = HP.unccomp(T1, c1, cinc)
        got = ref.unccomp_se3(T1, c1, cinc)
        assert np.all(np.abs(got - want) <= b), np.max(np.abs(got - want) / b)


def _zero_pivot_cases(rng):
    """H with an exactly zero row and column j (a generic SPD block elsewhere): the partial-pivot LU meets an all-zero pivot
    column at step j."""
    out = []
    for j in range(6):
        A = HP.spd(rng, rng.uniform(0.5, 2.0, 6))
        A[j, :] = 0.0
        A[:, j] = 0.0
        out.append(A)
    return out


def test_qr_restatement_vs_oracle_full_rank(oracle):
    """Every full-rank family of the GPU test: the restatement's QR keeps rank 6 with the smallest R entry at least 4x the rank
    threshold, its x is the exact solve, and the oracle's fp64 QR meets the backward bound everywhere and the forward and
    log|det| bounds where kappa eps <= 1e-2."""
    worst = {"back": 0.0, "fwd": 0.0, "lad": 0.0}
    for H, g, label in HP.qr_full_cases(1):
        perm, diag, maxpivot = HP.qr_pivots(H)
        assert min(abs(d) for d in diag) >= 4 * maxpivot * (HP.EPS * 6.0), label
        assert HP.qr_rank(H) == (6, list(range(6))), label
        x_hp, lad_hp = HP.chol_solve(H, g)
        np.testing.assert_allclose(HP.basic_solve(H, g, range(6)), x_hp, rtol=1e-14, atol=0)
        x, lad, rank = oracle.qr6_solve(H, g)
        assert rank == 6, label
        bb, bf, bl = HP.qr_bounds(H, g, x_hp)
        worst["back"] = max(worst["back"], HP.residual(H, g, x) / bb)
        if HP.cond(H) * HP.EPS <= 1e-2:
            worst["fwd"] = max(worst["fwd"], float(np.linalg.norm(x - x_hp)) / bf)
            worst["lad"] = max(worst["lad"], abs(lad - float(lad_hp)) / (bl + HP.C_SOLVE * HP.EPS * abs(float(lad_hp))))
    print("oracle QR, largest error / bound:", worst)
    assert max(worst.values()) <= 1.0, worst


def test_qr_rank_restatement_vs_oracle(oracle):
    """The placed rank decisions: the oracle's rank and support are the restatement's, its truncated entries exactly 0.0 and
    its x on the support within basic_bound of basic_solve; both verdicts occur at every scale, and the strict > at the
    threshold itself truncates."""
    worst = 0.0
    verdicts = {}
    for H, g, label in HP.rank_cases(2):
        rank, S = HP.qr_rank(H)
        x, lad, r = oracle.qr6_solve(H, g)
        assert r == rank, (label, r, rank)
        off = [j for j in range(6) if j not in S]
        assert np.all(x[off] == 0.0) and np.all(x[S] != 0.0), (label, x, S)
        want, b = HP.basic_solve(H, g, S), HP.basic_bound(H, g, S)
        if S:
            worst = max(worst, float(np.max(np.abs(x - want)[S] / b[S])))
        assert (lad == -np.inf) == (min(abs(d) for d in HP.qr_pivots(H)[1]) == 0.0), label
        r0, scale = int(re.search(r"r=(\d)", label).group(1)), label.split("s=")[1]
        if 0 < r0 < 6:
            verdicts.setdefault((label[:5], scale), set()).add(rank > r0)   # a placed D entry kept or truncated
        if label.startswith("exact"):
            assert rank == r0 + (" above " in label or " hi " in label), label   # the strict > at thr and one ulp on
    assert all(v == {True, False} for v in verdicts.values()) and len(verdicts) == 6, verdicts
    print("oracle truncated QR, largest error / bound:", worst)
    assert worst <= 1.0


def test_inverse_restatement_vs_oracle(oracle):
    """The oracle's partial-pivot LU inverse within the residual and forward bounds on every inverse case of the GPU test
    (kappa up to 1e15, scales 1e-60 .. 1e60, non-symmetric, tied pivot magnitudes); on an exactly zero pivot it is not finite."""
    worst = [0.0, 0.0]
    for H, label in HP.inv_cases(3):
        X = oracle.inv6(H)
        res, rb, fwd, fb = HP.inv_errors(H, X)
        worst = [max(worst[0], res / rb), max(worst[1], fwd / fb)]
        np.testing.assert_allclose(HP.inv(H), HP.tonp(mp.inverse(HP.mpm(H))), rtol=0, atol=0)
    print("oracle inverse, largest residual / bound, forward / bound:", worst)
    assert max(worst) <= 1.0, worst
    for A in _zero_pivot_cases(np.random.default_rng(4)):
        assert not np.all(np.isfinite(oracle.inv6(A)))


def test_cholesky_pivots_restatement():
    """chol_pivots on a diagonal matrix is its diagonal, and on a handover_matrix its last pivot is below the Cholesky's
    refusal with a margin of 2 (what the GPU test's hand-over band relies on)."""
    d = [4.0, 1.0, 0.25, 2.0, 8.0, 0.5]
    assert HP.chol_pivots(np.diag(d)) == d
    rng = np.random.default_rng(5)
    for k in (4e12, 1e13, 3e13, 1e14):
        H = HP.handover_matrix(rng, k, 1.0)
        assert min(HP.chol_pivots(H)) < 0.5e-12 * np.diag(H).max(), k
