"""NumPy restatement of what the reference does to a colour frame before its detectors: cv::cvtColor(COLOR_BGR2GRAY) on
8-bit data (LSDDetectorC::detectImpl, BinaryDescriptor::computeImpl and ORB convert with it), and rectifyImagesLR's remap of
the colour image before that conversion (Dataset::nextFrame remaps what cv::imread(..., IMREAD_UNCHANGED) gave).

cv2 4.13 converts every 8-bit BGR triple as (3735 B + 19235 G + 9798 R + 2^14) >> 15, with and without IPP.  The 14-bit
coefficients often quoted for it (1868, 9617, 4899, rounding 2^13, shift 14) disagree on 43 864 of the 2^24 triples.  Alpha,
where there is one, is not read.  cv::remap of a multi-channel image interpolates each channel as the one-channel remap does.
"""
from __future__ import annotations

import numpy as np

from oracle import rectify as R

# cv2 4.13's fixed point for 8-bit COLOR_BGR2GRAY: the coefficients sum to 2^15
B2Y, G2Y, R2Y, SHIFT = 3735, 19235, 9798, 15


def bgr_to_gray(img: np.ndarray) -> np.ndarray:
    """cv::cvtColor(img, COLOR_BGR2GRAY) of uint8[..., C] (C = 3: BGR, 4: BGRA) -> uint8[...]"""
    img = np.asarray(img, dtype=np.uint8)
    if img.shape[-1] not in (3, 4):
        raise ValueError("BGR or BGRA images: 3 or 4 channels")
    b, g, r = (img[..., c].astype(np.int64) for c in range(3))
    return ((B2Y * b + G2Y * g + R2Y * r + (1 << (SHIFT - 1))) >> SHIFT).astype(np.uint8)


def remap(img: np.ndarray, map1: np.ndarray, map2: np.ndarray) -> np.ndarray:
    """cv::remap(img, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) of uint8[H, W, C]: oracle/rectify.py's remap per channel."""
    img = np.asarray(img, dtype=np.uint8)
    return np.stack([R.remap(img[..., c], map1, map2) for c in range(img.shape[-1])], -1)


def remap_gray(img: np.ndarray, map1=None, map2=None) -> np.ndarray:
    """cvtColor(remap(img, map1, map2), COLOR_BGR2GRAY) of uint8[H, W, C]; without maps, cvtColor alone.  Only the three
    colour channels are remapped: the conversion does not read alpha."""
    img = np.asarray(img, dtype=np.uint8)
    if map1 is None:
        return bgr_to_gray(img)
    return bgr_to_gray(remap(img[..., :3], map1, map2))
