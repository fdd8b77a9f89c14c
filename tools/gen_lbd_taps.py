"""Recovers the fixed-point taps of cv2.GaussianBlur(img, (5, 5), 1) on 8-bit images (OpenCV's bit-exact path,
createGaussianKernelBitExact) that lbd.cu and oracle/ref_shim/lbd_standin.h use.  Needs cv2.

The 8-bit path blurs with a symmetric kernel of 8 fractional bits summing to 256: an exact integer row pass, a column
pass in 16.16, round half up.  Every symmetric kernel within 4 of 256 x the float Gaussian is tried on seeded images with
REFLECT_101 borders; exactly one must equal cv2 everywhere.

    python tools/gen_lbd_taps.py
"""
from __future__ import annotations

import numpy as np


def blur_fixed(img, k):
    H, W = img.shape
    def refl(p, n):
        if n == 1:
            return 0
        while p < 0 or p >= n:
            p = -p if p < 0 else 2 * n - 2 - p
        return p
    xs = np.array([[refl(x + i - 2, W) for i in range(5)] for x in range(W)])
    ys = np.array([[refl(y + j - 2, H) for j in range(5)] for y in range(H)])
    k = np.asarray(k, np.int64)
    row = (img.astype(np.int64)[:, xs] * k).sum(-1)            # [H, W]
    col = (row[ys] * k[None, :, None]).sum(1)                   # [H, W]
    return np.minimum((col + (1 << 15)) >> 16, 255).astype(np.uint8)


def main():
    import cv2
    g = np.exp(-(np.arange(5) - 2.0) ** 2 / 2.0)
    g = g / g.sum() * 256
    rng = np.random.default_rng(0)
    imgs = [rng.integers(0, 256, (h, w), dtype=np.uint8) for w, h in ((53, 40), (7, 5), (1, 9), (3, 2), (131, 77))]
    found = []
    for a in range(int(g[0]) - 4, int(g[0]) + 5):
        for b in range(int(g[1]) - 4, int(g[1]) + 5):
            k = [a, b, 256 - 2 * a - 2 * b, b, a]
            if all((blur_fixed(im, k) == cv2.GaussianBlur(im, (5, 5), 1)).all() for im in imgs):
                found.append(k)
    assert len(found) == 1, found
    print("taps", found[0], "cv2", cv2.__version__)


if __name__ == "__main__":
    main()
