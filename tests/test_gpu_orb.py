"""plstvo_orb_compute_batch on the GPU: bit-identical to cv2 (through the goldens) and to the oracle (seeded cases), and
end to end: tracking fed with GPU descriptors equals tracking fed with cv2's."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import orb_images as I
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import PlstvoError

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_orb_golden as M  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def orb():
    from oracle.orb import OrbOracle
    return OrbOracle()


def _images(name):
    return M.default_images() if name == "orb_default" else M.kitti_views()


def _survivors(off, cnt):
    return np.concatenate([np.arange(off[i], off[i] + cnt[i]) for i in range(len(cnt))]).astype(np.int64)


@pytest.mark.parametrize("name", ["orb_default", "orb_kitti"])
def test_gpu_equals_golden(engine, name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    imgs = _images(name)
    assert [I.sha256(im) for im in imgs] == list(z["sha256"])
    cfg = T.default_orb_config(int(z["n_levels"]), float(z["scale"]))
    n, out = engine.orb_compute_batch(cfg, imgs, z["det_off"], z["det_xy"], z["det_oct"], None)
    np.testing.assert_array_equal(out["counts"], np.diff(z["det_off"]))
    np.testing.assert_array_equal(out["src_idx"], np.concatenate([np.arange(k) for k in np.diff(z["det_off"])]))
    np.testing.assert_array_equal(out["angle"].view(np.uint32), z["det_angle_bits"])
    np.testing.assert_array_equal(out["desc"], z["det_desc"])
    ang_in = z["given_angle_bits"].view(np.float32)
    n, out = engine.orb_compute_batch(cfg, imgs, z["given_off"], z["given_xy"], z["given_oct"], ang_in)
    np.testing.assert_array_equal(out["counts"], z["given_counts"])
    rows = _survivors(z["given_off"], out["counts"])
    assert n == len(rows)
    np.testing.assert_array_equal(out["src_idx"][rows], z["given_src_idx"])
    np.testing.assert_array_equal(out["desc"][rows], z["given_desc"])
    base = np.repeat(z["given_off"][:-1], out["counts"])
    np.testing.assert_array_equal(out["angle"][rows].view(np.uint32), z["given_angle_bits"][base + out["src_idx"][rows]])


def _check(engine, orb, images, kp_off, xy, oct_, ang, nl, s):
    cfg = T.default_orb_config(nl, s)
    for a in (ang, None):
        n, out = engine.orb_compute_batch(cfg, images, kp_off, xy, oct_, a)
        ra, rd, rs, rc = orb.compute_batch(images, kp_off, xy, oct_, a, n_levels=nl, scale=s, threads=8)
        np.testing.assert_array_equal(out["counts"], rc)
        rows = _survivors(np.asarray(kp_off), rc) if len(rc) else np.zeros(0, np.int64)
        assert n == len(rows)
        np.testing.assert_array_equal(out["src_idx"][rows], rs[rows])
        np.testing.assert_array_equal(out["angle"][rows].view(np.uint32), ra[rows].view(np.uint32))
        np.testing.assert_array_equal(out["desc"][rows], rd[rows])


def _edge_cases(W, H, nl, s, edge=19):
    """Key points exactly at the edge distance and at the last valid row / column of every level, at several angles."""
    pts, octs = [], []
    for lvl in range(nl):
        sc = np.float32(s ** lvl)
        lw, lh = I.level_size(W, H, s, lvl)
        for x in (edge, W - edge - 1):
            for y in (edge, H - edge - 1, H // 2):
                pts.append((x, y)); octs.append(lvl)
        for lx in (lw - 1, 0, lw // 2):               # last column / row of the level (kept only if inside the filter)
            for ly in (lh - 1, lh // 2):
                pts.append((lx * sc, ly * sc)); octs.append(lvl)
    xy, oct_ = np.float32(pts), np.int32(octs)
    ang = np.float32([[0, 90, 180, 270, 359.99, 45, 44.99, 45.01][i % 8] for i in range(len(xy))])
    return xy, oct_, ang


@pytest.mark.parametrize("W,H,nl,s", [(640, 480, 4, 1.2), (1241, 376, 1, 1.2), (333, 251, 4, 2.0), (301, 199, 4, 1.2),
                                      (97, 61, 2, 2.0)])
def test_gpu_equals_oracle(engine, orb, W, H, nl, s):
    imgs = np.stack([I.make_image(W, H, 40 + k) for k in range(3)])
    xy, oct_, ang = [], [], []
    for k in range(3):
        a, b, c = I.make_keypoints(W, H, 900, nl, s, 7 + k)
        e = _edge_cases(W, H, nl, s)
        xy.append(np.concatenate([e[0], a])); oct_.append(np.concatenate([e[1], b])); ang.append(np.concatenate([e[2], c]))
    xy[1] = np.concatenate([xy[1], xy[1][:50]]); oct_[1] = np.concatenate([oct_[1], oct_[1][:50]])   # duplicates
    ang[1] = np.concatenate([ang[1], ang[1][:50]])
    off = np.cumsum([0] + [len(v) for v in xy]).astype(np.int32)
    _check(engine, orb, imgs, off, np.concatenate(xy), np.concatenate(oct_), np.concatenate(ang), nl, s)


def test_gpu_image_smaller_than_patch(engine, orb):
    imgs = np.stack([I.make_image(30, 24, 1), I.make_image(30, 24, 2)])
    xy = np.float32([[15, 12], [10, 10], [20, 5]] * 2)
    n, out = engine.orb_compute_batch(T.default_orb_config(), imgs, [0, 3, 6], xy, np.zeros(6, np.int32), None)
    assert n == 0 and list(out["counts"]) == [0, 0]
    assert (out["src_idx"] == -1).all()


def test_gpu_65535_keypoints_one_image(engine, orb):
    W, H = 1241, 376
    img = I.make_image(W, H, 77)[None]
    xy, oct_, ang = I.make_keypoints(W, H, 65535, 4, 1.2, 3)
    _check(engine, orb, img, [0, 65535], xy, oct_, ang, 4, 1.2)
    xy2 = np.concatenate([xy, xy[:1]])
    with pytest.raises(PlstvoError, match="TOO_LARGE"):
        engine.orb_compute_batch(T.default_orb_config(), img, [0, 65536], xy2, np.zeros(65536, np.int32), None)


def test_gpu_64_images(engine, orb):
    W, H = 320, 240
    imgs = np.stack([I.make_image(W, H, 500 + k) for k in range(64)])
    parts = [I.make_keypoints(W, H, 300 + 7 * k, 4, 1.2, 900 + k) for k in range(64)]
    off = np.cumsum([0] + [len(p[0]) for p in parts]).astype(np.int32)
    _check(engine, orb, imgs, off, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]),
           np.concatenate([p[2] for p in parts]), 4, 1.2)


def test_gpu_invalid_config(engine):
    img = I.make_image(100, 80, 1)[None]
    xy = np.float32([[50, 40]])
    for field, v in (("patch_size", 15), ("wta_k", 3), ("n_levels", 0)):
        cfg = T.default_orb_config()
        setattr(cfg, field, v)
        with pytest.raises(PlstvoError, match="INVALID"):
            engine.orb_compute_batch(cfg, img, [0, 1], xy, [0], None)
    with pytest.raises(PlstvoError, match="INVALID"):
        engine.orb_compute_batch(T.default_orb_config(), img, [0, 1], xy, [4], None)


def test_track_stereo_with_gpu_descriptors(engine):
    """plstvo_track_stereo_batch on the KITTI-size golden frames gives identical results with GPU descriptors and with cv2's."""
    z = np.load(os.path.join(GOLDEN, "orb_kitti.npz"))
    imgs = _images("orb_kitti")
    cfg = T.default_orb_config(1, 1.2)
    n, out = engine.orb_compute_batch(cfg, imgs, z["det_off"], z["det_xy"], z["det_oct"], None)
    off = z["det_off"]

    def frames(desc):
        fr = []
        for f in range(2):
            l, r = 2 * f, 2 * f + 1
            z32, zf = np.zeros((0, 32), np.uint8), np.zeros((0, 4), np.float32)
            fr.append(dict(pl_off=[0, off[l + 1] - off[l]], pr_off=[0, off[r + 1] - off[r]], kp_l=z["det_xy"][off[l]:off[l + 1]],
                           kp_r=z["det_xy"][off[r]:off[r + 1]], poct_l=z["det_oct"][off[l]:off[l + 1]],
                           pdesc_l=desc[off[l]:off[l + 1]], pdesc_r=desc[off[r]:off[r + 1]], ll_off=[0, 0], lr_off=[0, 0],
                           seg_l=zf, seg_r=zf, angle_l=np.zeros(0, np.float32), loct_l=np.zeros(0, np.int32), ldesc_l=z32,
                           ldesc_r=z32))
        return fr

    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    tc.has_lines = 0
    cam = T.kitti_camera()
    ra, na = engine.track_stereo_batch(cam, tc, mc, sc, *frames(out["desc"]))
    rb, nb = engine.track_stereo_batch(cam, tc, mc, sc, *frames(z["det_desc"]))
    assert na[0, 0] > 100 and na[0, 2] > 100, na                    # the stereo step kept points in both frames
    np.testing.assert_array_equal(na, nb)
    assert ra.tobytes() == rb.tobytes()
