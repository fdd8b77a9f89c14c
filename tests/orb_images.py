"""Seeded test images and key points for the ORB description tests and the `orb` bench row.

Images use NumPy integer operations only (rectangles, discs, ramps, noise from a PCG64 generator), so the same seed gives
the same bytes on every NumPy version and machine; tests/golden/orb_*.npz records their SHA-256 to prove it."""
from __future__ import annotations

import hashlib

import numpy as np


def make_image(W: int, H: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.int64)
    img = (x * int(rng.integers(1, 5)) + y * int(rng.integers(1, 5))) % 256 // 2 + 40       # ramp
    for _ in range(max(4, W * H // 6000)):                                                  # rectangles
        x0, y0 = int(rng.integers(-20, W)), int(rng.integers(-20, H))
        w, h = int(rng.integers(4, 80)), int(rng.integers(4, 60))
        img[max(y0, 0):max(y0 + h, 0), max(x0, 0):max(x0 + w, 0)] = int(rng.integers(0, 256))
    for _ in range(max(4, W * H // 8000)):                                                  # discs
        cx, cy, r = int(rng.integers(0, W)), int(rng.integers(0, H)), int(rng.integers(3, 30))
        img[(x - cx) ** 2 + (y - cy) ** 2 <= r * r] = int(rng.integers(0, 256))
    img += rng.integers(-12, 13, size=(H, W))                                               # noise
    return np.clip(img, 0, 255).astype(np.uint8)


def sha256(img: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(img, np.uint8).tobytes()).hexdigest()


def level_size(W: int, H: int, scale: float, level: int):
    """cvRound(W * (1.f / (float)scale^level)), in float32 like ORB."""
    inv = np.float32(1.0) / np.float32(scale ** level)
    return int(np.rint(np.float32(W) * inv)), int(np.rint(np.float32(H) * inv))


def make_keypoints(W: int, H: int, n: int, n_levels: int, scale: float, seed: int, edge: int = 19):
    """n key points spread over the levels the way ORB spreads its feature budget (a geometric share 1/scale per level),
    at integer positions of their level mapped to image coordinates (level pt * scale^level, float32) like ORB's own
    detections, all inside the border filter; angles uniform in [0, 360)."""
    rng = np.random.default_rng(seed)
    share = (1.0 / scale) ** np.arange(n_levels)
    share /= share.sum()
    oct_ = np.sort(rng.choice(n_levels, size=n, p=share)).astype(np.int32)
    xy = np.zeros((n, 2), np.float32)
    for lvl in range(n_levels):
        m = oct_ == lvl
        s = np.float32(scale ** lvl)
        lw, lh = level_size(W, H, scale, lvl)
        lo = int(np.ceil(edge / float(s))) + 1
        hx, hy = max(lo + 1, min(lw, int((W - edge) / float(s))) - 1), max(lo + 1, min(lh, int((H - edge) / float(s))) - 1)
        xy[m, 0] = rng.integers(lo, hx, int(m.sum())).astype(np.float32) * s
        xy[m, 1] = rng.integers(lo, hy, int(m.sum())).astype(np.float32) * s
    angle = (rng.random(n) * 360.0).astype(np.float32)
    return xy, oct_, angle
