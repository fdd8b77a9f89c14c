"""Pins the yardstick of the pose-helper tests (CPU): the high-precision restatement in hp_pose.py against the oracle's
compiled helpers (oracle/plstvo_oracle.c) and the reference's own SE(3) code and the stand-in's 6x6 algebra
(oracle/ref.py), within the conditioning bounds hp_pose.py states.  Where the reference library cannot be built, its answers
are replayed from tests/golden/ref_pose_helpers.npz (re-record where the reference is present with
PLSTVO_RECORD_REF=1 python -m pytest tests/test_hp_pose_host.py)."""
import os

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
