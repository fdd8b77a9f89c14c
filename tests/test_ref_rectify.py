"""oracle/rectify.py, the NumPy restatement of OpenCV's undistort-rectify maps and INTER_LINEAR remap, against
tests/golden/rectify.npz (cv2 4.13) and, where cv2 is installed, against live cv2 over seeded rigs and random maps."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import rectify as R

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_rectify_golden as M  # noqa: E402

G = np.load(os.path.join(GOLDEN, "rectify.npz"))


def case_args(c):
    w, h = (int(v) for v in G[f"{c}_size"])
    return int(G[f"{c}_model"]), G[f"{c}_K"], G[f"{c}_D"], G[f"{c}_R"], G[f"{c}_P"], w, h


@pytest.mark.parametrize("case", list(G["map_cases"]))
def test_maps_and_remap_equal_golden(case):
    m1, m2 = R.init_undistort_rectify_map(*case_args(case))
    assert (M.sha(m1, m2) == G[f"{case}_map_sha"]).all()
    w, h = (int(v) for v in G[f"{case}_size"])
    out = R.remap(M.image(int(G[f"{case}_seed"]), w, h), m1, m2)
    assert (M.sha(out) == G[f"{case}_out_sha"]).all()
    if f"{case}_map1" in G:
        np.testing.assert_array_equal(m1, G[f"{case}_map1"])
        np.testing.assert_array_equal(m2, G[f"{case}_map2"])
        np.testing.assert_array_equal(out, G[f"{case}_out"])


@pytest.mark.parametrize("case", list(G["remap_cases"]))
def test_remap_equals_golden(case):
    w, h = (int(v) for v in G[f"{case}_size"])
    m1 = G[f"{case}_map1"]
    np.testing.assert_array_equal(R.remap(M.image(int(G[f"{case}_seed"]), w, h), m1, G[f"{case}_map2"]), G[f"{case}_out"])


def test_golden_covers_the_edges():
    sat = R.init_undistort_rectify_map(*case_args("pin_saturate"))[0]
    assert (sat == -32768).any()   # short saturation in the vector columns
    behind = R.init_undistort_rectify_map(*case_args("fish_behind"))
    assert (behind[0] == 0).all(-1).any()     # +-inf: INT_MIN >> 5 truncated to short
    m1 = G["remap_64x48_map1"]                 # taps beyond every edge, some far out
    assert (m1[..., 0] < 0).any() and (m1[..., 0] >= 63).any() and (m1[..., 1] < 0).any() and (m1[..., 1] >= 47).any()
    assert np.abs(m1.astype(np.int64)).max() > 10000


@pytest.mark.parametrize("bad", [dict(D=[0.1] * 12), dict(D=[0.1] * 14), dict(D=[0.1] * 3), dict(model=1, D=[0.1] * 5),
                                 dict(P=np.zeros((3, 4))), dict(w=0), dict(h=40000)])
def test_restatement_rejects(bad):
    a = dict(model=0, D=[0.1, 0.0, 0.0, 0.0], P=np.eye(3), w=8, h=8)
    a.update(bad)
    with pytest.raises(ValueError):
        R.init_undistort_rectify_map(a["model"], np.eye(3), a["D"], np.eye(3), a["P"], a["w"], a["h"])


# ---- live cv2 ----
def _sweep(seed):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(seed)
    out = []
    for k in range(12):
        strong = k % 2 == 1
        K = np.array([[380 + rng.uniform(0, 120), 0, 150 + rng.uniform(0, 40)],
                      [0, 380 + rng.uniform(0, 120), 100 + rng.uniform(0, 30)], [0, 0, 1.0]])
        Rm = cv2.Rodrigues(rng.normal(0, 0.02, 3))[0]
        P = np.hstack([K * rng.uniform(0.8, 1.1), np.zeros((3, 1))])
        P[2] = [0, 0, 1, 0]
        if k % 3 == 2:
            D = rng.normal(0, 0.02, 4) * (5 if strong else 1)
            out.append((1, K, D, Rm, P))
        else:
            nd = (4, 5, 8)[k % 3 if k % 3 < 2 else 0] if not strong else (5, 8)[k % 2]
            D = np.array([-0.28, 0.074, 2e-4, 2e-5, 0.01, 0.0, 0.0, 0.0])[:nd] if not strong else \
                np.concatenate([rng.normal(0, 0.3, 2), rng.normal(0, 0.003, 2), rng.normal(0, 0.1, 4)])[:nd]
            out.append((0, K, D, Rm, P))
    return cv2, out


def test_maps_equal_live_cv2():
    cv2, rigs = _sweep(41)
    for model, K, D, Rm, P in rigs:
        for w, h in ((331, 211), (40, 3)):
            build = cv2.fisheye.initUndistortRectifyMap if model == 1 else cv2.initUndistortRectifyMap
            m1, m2 = build(K, D, Rm, P, (w, h), cv2.CV_16SC2)
            o1, o2 = R.init_undistort_rectify_map(model, K, D, Rm, P, w, h)
            np.testing.assert_array_equal(o1, m1)
            np.testing.assert_array_equal(o2, m2)


def test_remap_equals_live_cv2():
    cv2 = pytest.importorskip("cv2")
    for k, (w, h) in enumerate(((1, 1), (2, 5), (31, 17), (160, 120))):
        rng = np.random.default_rng(900 + k)
        img = M.image(900 + k, w, h)
        mx = rng.uniform(-4, w + 3, (h, w)).astype(np.float32)
        my = rng.uniform(-4, h + 3, (h, w)).astype(np.float32)
        m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        np.testing.assert_array_equal(R.remap(img, m1, m2), cv2.remap(img, m1, m2, cv2.INTER_LINEAR))
