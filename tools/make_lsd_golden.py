"""Writes tests/golden/lsd.npz: cv2 4.13's LineSegmentDetector segments (LSD_REFINE_NONE) and the reference's key lines
(LSDDetectorC's KeyLine step and detectLineFeatures' sort-and-truncate, applied to those segments by oracle/lsd.py) for
seeded images.  The images are regenerated from their specs (cases()) and checked against the SHA-256 the file records.

    python tools/make_lsd_golden.py            # needs cv2; rewrites tests/golden/lsd.npz
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import orb_images as I  # noqa: E402
from oracle import lsd  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "lsd.npz")
SHIPPED = lsd.SHIPPED
# non-shipped values of every parameter the C-ABI accepts (scale < 1 takes the shrinking blur; scale 1 skips blur and resize)
OTHER_A = dict(scale=0.8, sigma_scale=0.8, quant=3.0, ang_th=30.0, n_bins=256, min_line_length=0.05, n_features=50)
OTHER_B = dict(scale=1.0, sigma_scale=0.6, quant=1.5, ang_th=15.0, n_bins=4096, min_line_length=0.0, n_features=0)
# blurs whose fixed-point taps take error diffusion: sigma 0.5 (taps 27, 202, 27) and 0.6 / 0.75 = 0.8 (scale 0.75 shrinks)
OTHER_C = dict(SHIPPED, sigma_scale=0.5)
OTHER_D = dict(SHIPPED, scale=0.75)


def _noise(W, H, seed):
    return np.random.default_rng(seed).integers(0, 256, (H, W), dtype=np.uint8)


def _flat(W, H, seed):
    return np.full((H, W), 128, np.uint8)


def _border(W, H, seed):
    """Strong edges along the image border: segments ending within a pixel or two of each side."""
    img = I.make_image(W, H, seed) // 4 + 60
    img[:, :2] = 230
    img[-2:, :] = 10
    img[:3, W // 3:] = 250
    return img.astype(np.uint8)


def _ties(W, H, seed):
    """Identical rectangles on a flat background: many lines of equal length, so equal responses decide the truncation."""
    img = np.full((H, W), 90, np.uint8)
    for r in range(4):
        for c in range(6):
            img[20 + 60 * r:20 + 60 * r + 24, 20 + 60 * c:20 + 60 * c + 40] = 200
    return img


def _make(W, H, seed):
    return I.make_image(W, H, seed)


def _kitti_view(W, H, k):
    """View k of the two KITTI-size stereo frames of tests/golden/orb_kitti.npz (left 0, right 1, left 2, right 3)."""
    import make_orb_golden
    return make_orb_golden.kitti_views()[k]


GEN = {"kitti_view": _kitti_view, "make": _make, "noise": _noise, "flat": _flat, "border": _border, "ties": _ties}


def seed_order_cases(n=4):
    """Small images on which the two candidate seed orders (std::sort on the bin alone, raster order within a bin) give
    different segments: the first n found in a fixed search."""
    o = lsd.LsdOracle()
    rng, found = np.random.default_rng(1), []
    for t in range(300):
        W, H = int(rng.integers(2, 40)), int(rng.integers(2, 40))
        kind = "noise" if t % 3 == 0 else "make"
        img = GEN[kind](W, H, t)
        a, b = o.segments(img, seed_order=o.STD_SORT), o.segments(img, seed_order=o.STABLE)
        if a.shape != b.shape or not np.array_equal(a, b):
            found.append((f"seed_order_{len(found)}", W, H, kind, [t], SHIPPED))
            if len(found) == n:
                break
    return found


def clip_cases(n=4):
    """Small images with a kept line whose endpoint rounds outside the image (an endpoint in [W - 0.5, W)), where
    numOfPixels is LineIterator's count after clipLine: the first n found in a fixed search.  Several also have raw
    endpoints outside the image, which checkLineExtremes clamps."""
    o = lsd.LsdOracle()
    rng, found = np.random.default_rng(2), []
    for t in range(400):
        W, H = int(rng.integers(8, 64)), int(rng.integers(8, 64))
        kind = "noise" if t % 2 else "make"
        img = GEN[kind](W, H, 500 + t)
        kl = o.detect(img)
        r = np.rint(kl["seg"].astype(np.float64))
        if ((r[:, [0, 2]] >= W).any(1) | (r[:, [1, 3]] >= H).any(1)).any():
            found.append((f"clip_{len(found)}", W, H, kind, [500 + t], SHIPPED))
            if len(found) == n:
                break
    return found


def cases():
    c = [("kitti_300", 1241, 376, "make", [1, 2], SHIPPED),
         ("kitti_100", 1241, 376, "make", [1, 2], dict(SHIPPED, n_features=100)),
         ("euroc_300", 752, 480, "make", [3, 4], SHIPPED),
         ("euroc_100", 752, 480, "make", [3, 4], dict(SHIPPED, n_features=100)),
         ("kitti_stereo", 1241, 376, "kitti_view", [0, 1, 2, 3], SHIPPED),
         ("flat", 1241, 376, "flat", [0], SHIPPED),
         ("border", 320, 200, "border", [5, 6], SHIPPED),
         ("ties", 400, 280, "ties", [0], dict(SHIPPED, n_features=10)),
         ("odd_63x17", 63, 17, "make", [7, 8, 9], SHIPPED),
         ("odd_131x77", 131, 77, "noise", [10, 11], SHIPPED),
         ("other_a", 641, 371, "make", [12, 13], OTHER_A),
         ("other_b", 641, 371, "make", [12, 13], OTHER_B),
         ("other_c", 1241, 376, "make", [1], OTHER_C),
         ("other_d", 1241, 376, "make", [1], OTHER_D)]
    for W, H in [(1, 1), (1, 8), (2, 2), (3, 5), (5, 3), (4, 4), (6, 7), (8, 8)]:
        c.append((f"tiny_{W}x{H}", W, H, "noise", [W * 10 + H, W * 10 + H + 100], SHIPPED))
    return c + seed_order_cases() + clip_cases()


def images(W, H, kind, seeds):
    return np.stack([GEN[kind](W, H, s) for s in seeds])


PARAM_KEYS = ["scale", "sigma_scale", "quant", "ang_th", "n_bins", "min_line_length", "n_features"]


def golden() -> dict:
    import cv2
    o = lsd.LsdOracle()
    out = {"cv2_version": np.array(cv2.__version__), "cases": np.array([c[0] for c in cases()])}
    for name, W, H, kind, seeds, P in cases():
        imgs = images(W, H, kind, seeds)
        det = cv2.createLineSegmentDetector(0, P["scale"], P["sigma_scale"], P["quant"], P["ang_th"], 0, 0.7, P["n_bins"])
        raw, raw_off, kl, kl_off = [], [0], {k: [] for k in ("seg", "angle", "npix", "response", "length")}, [0]
        for img in imgs:
            seg = det.detect(img)[0]
            seg = np.zeros((0, 4), np.float32) if seg is None else seg.reshape(-1, 4).astype(np.float32)
            raw.append(seg)
            raw_off.append(raw_off[-1] + len(seg))
            k = o.keylines_from_segments(W, H, seg, P["min_line_length"], P["n_features"])
            for f in kl:
                kl[f].append(k[f])
            kl_off.append(kl_off[-1] + len(k["angle"]))
        out[f"{name}/spec"] = np.array([W, H] + list(seeds), np.int64)
        out[f"{name}/kind"] = np.array(kind)
        out[f"{name}/params"] = np.array([P[k] for k in PARAM_KEYS], np.float64)
        out[f"{name}/sha256"] = np.array([I.sha256(im) for im in imgs])
        out[f"{name}/raw"] = np.concatenate(raw).reshape(-1, 4)
        out[f"{name}/raw_off"] = np.array(raw_off, np.int32)
        out[f"{name}/kl_off"] = np.array(kl_off, np.int32)
        for f in kl:
            out[f"{name}/{f}"] = np.concatenate(kl[f]) if kl[f] else np.zeros(0)
        out[f"{name}/seg"] = out[f"{name}/seg"].reshape(-1, 4)
    return out


def load_case(g, name):
    """(images, params dict, raw, raw_off, key lines dict with off) of one case of the golden file, images regenerated and
    checked against the recorded SHA-256."""
    spec = [int(v) for v in g[f"{name}/spec"]]
    imgs = images(spec[0], spec[1], str(g[f"{name}/kind"]), spec[2:])
    assert [I.sha256(im) for im in imgs] == list(g[f"{name}/sha256"]), name
    pv = g[f"{name}/params"]
    P = {k: (int(v) if k in ("n_bins", "n_features") else float(v)) for k, v in zip(PARAM_KEYS, pv)}
    kl = {f: g[f"{name}/{f}"] for f in ("seg", "angle", "npix", "response", "length")}
    kl["off"] = g[f"{name}/kl_off"]
    return imgs, P, g[f"{name}/raw"], g[f"{name}/raw_off"], kl


if __name__ == "__main__":
    np.savez_compressed(OUT, **golden())
    print("wrote", OUT)
