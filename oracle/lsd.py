"""ctypes binding of the LSD restatement (oracle/lsd_oracle.cpp).

TEST INFRASTRUCTURE, like orb.py: tests/ and tools/ import it; the product package never does.  Built with g++ (so its
std::sort is libstdc++'s) and -ffp-contract=off, into the tree when build() runs, else into the per-user scratch
directory (a read-only checkout)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

from oracle.oracle import _scratch_dir

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "lsd_oracle.cpp")

# Config::lsd* of every shipped config (config/config/*.yaml), n_features 300; min_line_length relative to min(W, H)
SHIPPED = dict(scale=1.2, sigma_scale=0.6, quant=2.0, ang_th=22.5, n_bins=1024, min_line_length=0.025, n_features=300)


def _build(out: str) -> None:
    os.makedirs(os.path.dirname(out), exist_ok=True)
    tmp = f"{out}.{os.getpid()}.tmp"
    cmd = ["g++", "-O2", "-march=x86-64-v3", "-mtune=generic", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared",
           "-o", tmp, _SRC]
    subprocess.run(cmd, check=True, capture_output=True)
    os.replace(tmp, out)


def lib_path() -> str:
    lib = os.path.join(_HERE, "liblsd_oracle.so")
    if os.path.exists(lib) and os.path.getmtime(_SRC) <= os.path.getmtime(lib):
        return lib
    if not os.access(_HERE, os.W_OK):
        h = hashlib.sha1(open(_SRC, "rb").read()).hexdigest()[:16]
        lib = os.path.join(_scratch_dir(), "lsd", h, "liblsd_oracle.so")
        if os.path.exists(lib):
            return lib
    _build(lib)
    return lib


_u8, _i32, _f32 = C.POINTER(C.c_uint8), C.POINTER(C.c_int32), C.POINTER(C.c_float)


def _p(a, typ):
    return None if a is None else a.ctypes.data_as(typ)


class LsdOracle:
    STD_SORT, STABLE = 0, 1   # seed orders: std::sort on the bin alone, or raster order within a bin (cv2 4.13's)

    def __init__(self):
        self.lib = L = C.CDLL(lib_path())
        L.orc_lsd_gauss_taps.restype = C.c_int
        L.orc_lsd_gauss_taps.argtypes = [C.c_double, _i32]
        L.orc_lsd_blur.restype = None
        L.orc_lsd_blur.argtypes = [_u8, C.c_int, C.c_int, _u8, C.c_int, _i32]
        L.orc_lsd_scaled_size.restype = C.c_int
        L.orc_lsd_scaled_size.argtypes = [C.c_int, C.c_double]
        L.orc_lsd_resize.restype = None
        L.orc_lsd_resize.argtypes = [_u8, C.c_int, C.c_int, _u8, C.c_int, C.c_int, C.c_double]
        L.orc_lsd_segments.restype = C.c_int
        L.orc_lsd_segments.argtypes = [_u8, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int,
                                       C.c_int, C.c_int, _f32, _u8, _i32]
        L.orc_lsd_line_count.restype = C.c_int
        L.orc_lsd_line_count.argtypes = [C.c_int, C.c_int, _f32]
        L.orc_lsd_keylines_from_segments.restype = C.c_int
        L.orc_lsd_keylines_from_segments.argtypes = [C.c_int, C.c_int, C.c_int, _f32, C.c_double, C.c_int, _f32, _f32,
                                                     _i32, _f32, _f32]

    def blur(self, img, sigma):
        img = np.ascontiguousarray(img, np.uint8)
        taps = np.zeros(64, np.int32)
        kh = self.lib.orc_lsd_gauss_taps(sigma, _p(taps, _i32))
        out = np.zeros_like(img)
        self.lib.orc_lsd_blur(_p(img, _u8), img.shape[1], img.shape[0], _p(out, _u8), kh, _p(taps, _i32))
        return out

    def resize(self, img, scale):
        img = np.ascontiguousarray(img, np.uint8)
        h, w = img.shape
        dw, dh = self.lib.orc_lsd_scaled_size(w, scale), self.lib.orc_lsd_scaled_size(h, scale)
        out = np.zeros((dh, dw), np.uint8)
        self.lib.orc_lsd_resize(_p(img, _u8), w, h, _p(out, _u8), dw, dh, scale)
        return out

    def segments(self, img, scale=1.2, sigma_scale=0.6, quant=2.0, ang_th=22.5, n_bins=1024, seed_order=STABLE):
        """Raw LineSegmentDetector::detect output, float32 [n][4] (x1, y1, x2, y2)."""
        img = np.ascontiguousarray(img, np.uint8)
        H, W = img.shape
        cap = 4096
        while True:
            out = np.zeros((cap, 4), np.float32)
            n = self.lib.orc_lsd_segments(_p(img, _u8), W, H, scale, sigma_scale, quant, ang_th, n_bins, seed_order, cap,
                                          _p(out, _f32), None, None)
            if n <= cap:
                return out[:n]
            cap = n

    def line_count(self, W, H, seg) -> int:
        """cv::LineIterator's 8-connected count between the rounded endpoints of seg (x1, y1, x2, y2), clipped to W x H."""
        seg = np.ascontiguousarray(seg, np.float32)
        return self.lib.orc_lsd_line_count(W, H, _p(seg, _f32))

    def keylines_from_segments(self, W, H, raw, min_line_length=0.025, n_features=300):
        """The reference's KeyLine step and sort-and-truncate: dict of seg [n][4], angle, npix, response, length."""
        raw = np.ascontiguousarray(raw, np.float32).reshape(-1, 4)
        n = len(raw)
        seg, ang, npix = np.zeros((n, 4), np.float32), np.zeros(n, np.float32), np.zeros(n, np.int32)
        resp, length = np.zeros(n, np.float32), np.zeros(n, np.float32)
        k = self.lib.orc_lsd_keylines_from_segments(W, H, n, _p(raw, _f32), float(min_line_length) * min(W, H),
                                                    int(n_features), _p(seg, _f32), _p(ang, _f32), _p(npix, _i32),
                                                    _p(resp, _f32), _p(length, _f32))
        return dict(seg=seg[:k], angle=ang[:k], npix=npix[:k], response=resp[:k], length=length[:k])

    def detect(self, img, scale=1.2, sigma_scale=0.6, quant=2.0, ang_th=22.5, n_bins=1024, min_line_length=0.025,
               n_features=300):
        """detectLineFeatures' key lines for one image (the LSD branch)."""
        H, W = np.shape(img)
        raw = self.segments(img, scale, sigma_scale, quant, ang_th, n_bins)
        return self.keylines_from_segments(W, H, raw, min_line_length, n_features)
