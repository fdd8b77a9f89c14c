"""What the reference's FLD line branch (use_fld_lines, src/stereoFrame.cpp:244-304) does around FastLineDetector, for the
tests: the binding of oracle/_ref/libplstvo_ref_fld.so (the branch's KeyLine step compiled from the reference's own text by
oracle/make_ref_fld.py), and a NumPy restatement of its fld_img of a colour frame, cv::cvtColor(CV_RGB2GRAY) on 8-bit data.

cv2 4.13 converts RGB to grey with the BGR2GRAY fixed point with the first and third channels swapped:
(9798 c0 + 19235 c1 + 3735 c2 + 2^14) >> 15.  A fourth channel is not read.  The library's LBD reads that image while ORB
still reads the COLOR_BGR2GRAY one (oracle/color.py).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import color as OC

LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libplstvo_ref_fld.so")
_lib = None


def rgb_to_gray(img: np.ndarray) -> np.ndarray:
    """cv::cvtColor(img, COLOR_RGB2GRAY) of uint8[..., C] (C = 3 or 4) -> uint8[...]"""
    img = np.asarray(img, dtype=np.uint8)
    if img.shape[-1] not in (3, 4):
        raise ValueError("RGB or RGBA images: 3 or 4 channels")
    r, g, b = (img[..., c].astype(np.int64) for c in range(3))
    return ((OC.B2Y * b + OC.G2Y * g + OC.R2Y * r + (1 << (OC.SHIFT - 1))) >> OC.SHIFT).astype(np.uint8)


def remap_gray_rgb(img: np.ndarray, map1=None, map2=None) -> np.ndarray:
    """cvtColor(remap(img, map1, map2), CV_RGB2GRAY) of uint8[H, W, C]; without maps, cvtColor alone."""
    img = np.asarray(img, dtype=np.uint8)
    if map1 is None:
        return rgb_to_gray(img)
    return rgb_to_gray(OC.remap(img[..., :3], map1, map2))


def available() -> bool:
    return os.path.exists(LIB)


def key_lines(width: int, height: int, n_features: int, seg) -> dict:
    """The reference's KeyLine step on FLD's segments seg float32[n, 4]: dict(seg, angle, npix, response, length) as
    plstvo_fld_key_lines returns them."""
    global _lib
    if _lib is None:
        _lib = C.CDLL(LIB)
        fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
        _lib.fld_ref_key_lines.restype = C.c_int
        _lib.fld_ref_key_lines.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, fp, fp, fp, ip, fp, fp]
    seg = np.ascontiguousarray(seg, np.float32).reshape(-1, 4)
    n = len(seg)
    out = dict(seg=np.zeros((n, 4), np.float32), angle=np.zeros(n, np.float32), npix=np.zeros(n, np.int32),
               response=np.zeros(n, np.float32), length=np.zeros(n, np.float32))
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    m = _lib.fld_ref_key_lines(width, height, n_features, n, seg.ctypes.data_as(fp), out["seg"].ctypes.data_as(fp),
                               out["angle"].ctypes.data_as(fp), out["npix"].ctypes.data_as(ip),
                               out["response"].ctypes.data_as(fp), out["length"].ctypes.data_as(fp))
    return {k: v[:m] for k, v in out.items()}
