"""plstvo_lbd_compute_batch on the GPU: bit-identical to the reference's BinaryDescriptor::compute (through
tests/golden/lbd.npz and, where oracle/_ref is built, through the reference library on seeded batches), and end to end:
stereo tracking fed with GPU line descriptors equals tracking fed with the reference's."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
import orb_images as I
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError

sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_lbd_golden as M  # noqa: E402

from oracle import lbd  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(GOLDEN, "lbd.npz"))


@pytest.mark.parametrize("name", [str(c) for c in G["cases"]])
def test_gpu_equals_golden(engine, name):
    images, off, seg, ang, npix, desc = M.load_case(G, name)
    np.testing.assert_array_equal(engine.lbd_compute_batch(images, off, seg, ang, npix), desc)


def random_lines(W, H, n, seed):
    """n lines with LSD-like lengths (mostly short, a long tail up to the image size), end points up to a pixel outside the
    image, angles mostly the segment's own and sometimes arbitrary."""
    rng = np.random.default_rng(seed)
    length = np.minimum(np.float64(max(W, H)), 8.0 + rng.exponential(40.0, n) * rng.choice([1.0, 6.0], n, p=[0.85, 0.15]))
    th = rng.uniform(-np.pi, np.pi, n)
    cx, cy = rng.uniform(-1, W, n), rng.uniform(-1, H, n)
    seg = np.stack([cx - 0.5 * length * np.cos(th), cy - 0.5 * length * np.sin(th),
                    cx + 0.5 * length * np.cos(th), cy + 0.5 * length * np.sin(th)], 1)
    seg[:, 0::2] = np.clip(seg[:, 0::2], -1, W)
    seg[:, 1::2] = np.clip(seg[:, 1::2], -1, H)
    seg = seg.astype(np.float32)
    ang = np.arctan2(seg[:, 3].astype(np.float64) - seg[:, 1], seg[:, 2].astype(np.float64) - seg[:, 0])
    ang = np.where(rng.random(n) < 0.2, rng.uniform(-np.pi, np.pi, n), ang).astype(np.float32)
    npix = np.array([M.line_pixels(*s) for s in seg], np.int32)
    return seg, ang, npix


def ragged_batch(W, H, n_img, seed):
    images = np.stack([I.make_image(W, H, seed + k) for k in range(n_img)])
    counts = [0 if k in (0, n_img // 2, n_img - 1) else int(np.random.default_rng(seed + k).integers(1, 320)) for k in range(n_img)]
    parts = [random_lines(W, H, c, seed + 1000 + k) for k, c in enumerate(counts)]
    off = np.cumsum([0] + counts).astype(np.int32)
    return images, off, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), np.concatenate([p[2] for p in parts])


@pytest.mark.skipif(not lbd.available(), reason="oracle/_ref/libplstvo_ref_lbd.so not built (needs the reference checkout)")
@pytest.mark.parametrize("W,H", [(640, 480), (333, 97)])
def test_gpu_64_images_equal_reference(engine, W, H):
    images, off, seg, ang, npix = ragged_batch(W, H, 64, 300 + W)
    np.testing.assert_array_equal(engine.lbd_compute_batch(images, off, seg, ang, npix),
                                  lbd.compute_batch(images, off, seg, ang, npix))


def test_batched_equals_single_image_calls(engine):
    images, off, seg, ang, npix = ragged_batch(320, 240, 9, 40)
    full = engine.lbd_compute_batch(images, off, seg, ang, npix)
    for i in range(len(images)):
        a, b = off[i], off[i + 1]
        one = engine.lbd_compute_batch(images[i:i + 1], [0, b - a], seg[a:b], ang[a:b], npix[a:b])
        np.testing.assert_array_equal(one, full[a:b])


def test_context_reuse_big_small_big():
    big = ragged_batch(1241, 376, 6, 70)
    small = ragged_batch(37, 23, 3, 80)
    fresh = []
    for b in (big, small):
        e = Engine()
        fresh.append(e.lbd_compute_batch(*b))
        e.close()
    e = Engine()
    for b, want in ((big, fresh[0]), (small, fresh[1]), (big, fresh[0])):
        np.testing.assert_array_equal(e.lbd_compute_batch(*b), want)
    e.close()


def test_no_lines_writes_nothing(engine):
    images = np.stack([I.make_image(50, 40, 1), I.make_image(50, 40, 2)])
    seg, ang, npix = random_lines(50, 40, 5, 3)
    assert engine.lib.plstvo_lbd_compute_batch(engine.ctx, 2, 50, 40, None, np.int32([0, 0, 0]).ctypes.data_as(T.c_int32_p),
                                               None, None, None, None) == 0
    desc = engine.lbd_compute_batch(images, [0, 0, 5], seg, ang, npix)
    one = engine.lbd_compute_batch(images[1:], [0, 5], seg, ang, npix)
    np.testing.assert_array_equal(desc, one)


def test_invalid_and_too_large(engine):
    img = I.make_image(60, 40, 5)[None]
    seg, ang, npix = random_lines(60, 40, 3, 6)
    bad = [dict(npix=np.int32([0, 5, 5])), dict(npix=np.int32([5, 32768, 5])), dict(off=[0, 3], W=0),
           dict(off=[1, 3]), dict(off=[0, -1])]
    for b in bad:
        images = img if "W" not in b else np.zeros((1, 40, 0), np.uint8)
        with pytest.raises(PlstvoError, match="INVALID"):
            engine.lbd_compute_batch(images, b.get("off", [0, 3]), seg, ang, b.get("npix", npix))
    lib, ctx = engine.lib, engine.ctx
    off3 = np.int32([0, 3]).ctypes.data_as(T.c_int32_p)
    assert lib.plstvo_lbd_compute_batch(ctx, 1, 32768, 40, img.ctypes.data_as(T.c_uint8_p), off3, seg.ctypes.data_as(T.c_float_p),
                                        ang.ctypes.data_as(T.c_float_p), npix.ctypes.data_as(T.c_int32_p), None) == -1
    assert lib.plstvo_lbd_compute_batch(ctx, 1, 60, 40, None, off3, seg.ctypes.data_as(T.c_float_p),
                                        ang.ctypes.data_as(T.c_float_p), npix.ctypes.data_as(T.c_int32_p), None) == -1
    n = T_MAX = 65535
    seg2, ang2, npix2 = (np.resize(seg, (n + 1, 4)), np.resize(ang, n + 1), np.resize(npix, n + 1))
    with pytest.raises(PlstvoError, match="TOO_LARGE"):
        engine.lbd_compute_batch(img, [0, T_MAX + 1], seg2, ang2, npix2)
    d = engine.lbd_compute_batch(img, [0, T_MAX], seg2[:n], ang2[:n], npix2[:n])   # the limit itself is accepted
    np.testing.assert_array_equal(d[:3], engine.lbd_compute_batch(img, [0, 3], seg, ang, npix))


def test_more_images_than_one_grid_slice(engine):
    """65 537 images: the gradient launch covers them in slices of at most 65 535 (the grid's z limit)."""
    n = 65537
    images = np.stack([I.make_image(9, 7, 5), I.make_image(9, 7, 6)])[np.arange(n) % 2]
    seg, ang, npix = random_lines(9, 7, 6, 11)
    off = np.zeros(n + 1, np.int32)
    off[1:] = 2
    off[n - 2:] = [2, 4, 6]        # lines in the first image and in the last two (past the first slice)
    got = engine.lbd_compute_batch(images, off, seg, ang, npix)
    for i, (a, b) in ((0, (0, 2)), (n - 2, (2, 4)), (n - 1, (4, 6))):
        np.testing.assert_array_equal(got[a:b], engine.lbd_compute_batch(images[i:i + 1], [0, b - a], seg[a:b], ang[a:b], npix[a:b]))


def test_kernel_times_positive(engine):
    images, off, seg, ang, npix = ragged_batch(640, 480, 4, 90)
    engine.lbd_compute_batch(images, off, seg, ang, npix)
    ms = engine.lbd_kernel_times()
    assert ms.shape == (2,) and (ms > 0).all(), ms


def test_track_stereo_with_gpu_line_descriptors(engine):
    """plstvo_track_stereo_batch on the KITTI-size stereo frames gives byte-identical results with GPU line descriptors and
    with the reference's (the golden)."""
    images, off, seg, ang, npix, ref_desc = M.load_case(G, "kitti_stereo")
    desc = engine.lbd_compute_batch(images, off, seg, ang, npix)

    def frames(d):
        fr = []
        for f in range(2):
            l, r = 2 * f, 2 * f + 1
            z2, z32 = np.zeros((0, 2), np.float32), np.zeros((0, 32), np.uint8)
            fr.append(dict(pl_off=[0, 0], pr_off=[0, 0], kp_l=z2, kp_r=z2, poct_l=np.zeros(0, np.int32), pdesc_l=z32,
                           pdesc_r=z32, ll_off=[0, off[l + 1] - off[l]], lr_off=[0, off[r + 1] - off[r]],
                           seg_l=seg[off[l]:off[l + 1]], seg_r=seg[off[r]:off[r + 1]], angle_l=ang[off[l]:off[l + 1]],
                           loct_l=np.zeros(off[l + 1] - off[l], np.int32), ldesc_l=d[off[l]:off[l + 1]],
                           ldesc_r=d[off[r]:off[r + 1]]))
        return fr

    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    tc.has_points = 0
    cam = T.kitti_camera()
    ra, na = engine.track_stereo_batch(cam, tc, mc, sc, *frames(desc))
    rb, nb = engine.track_stereo_batch(cam, tc, mc, sc, *frames(ref_desc))
    assert na[0, 1] > 20 and na[0, 3] > 20, na                      # the stereo step kept lines in both frames
    np.testing.assert_array_equal(na, nb)
    assert ra.tobytes() == rb.tobytes()
