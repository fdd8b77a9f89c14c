"""ctypes binding of the ORB description oracle (oracle/orb_oracle.c).

TEST INFRASTRUCTURE, like oracle.py: tests/, tools/ and bench.py's CPU arm import it; the product package never does.
Built with the flags oracle.py uses (x86-64-v3, -ffp-contract=off), into the tree when build() runs, else into the per-user
scratch directory (a read-only checkout)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

from oracle.oracle import _scratch_dir

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = [os.path.join(_HERE, "orb_oracle.c"), os.path.join(_HERE, "..", "stvo_pl_b200", "csrc", "orb_pattern.h")]


def _build(out: str) -> None:
    os.makedirs(os.path.dirname(out), exist_ok=True)
    tmp = f"{out}.{os.getpid()}.tmp"
    cmd = ["gcc", "-O3", "-march=x86-64-v3", "-mtune=generic", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-shared",
           "-o", tmp, _SRC[0], "-lm", "-lpthread"]
    subprocess.run(cmd, check=True, capture_output=True)
    os.replace(tmp, out)


def lib_path() -> str:
    lib = os.path.join(_HERE, "liborb_oracle.so")
    if os.path.exists(lib) and all(os.path.getmtime(s) <= os.path.getmtime(lib) for s in _SRC):
        return lib
    if not os.access(_HERE, os.W_OK):
        h = hashlib.sha1(b"".join(open(s, "rb").read() for s in _SRC)).hexdigest()[:16]
        lib = os.path.join(_scratch_dir(), "orb", h, "liborb_oracle.so")
        if os.path.exists(lib):
            return lib
    _build(lib)
    return lib


_u8, _i32, _f32 = C.POINTER(C.c_uint8), C.POINTER(C.c_int32), C.POINTER(C.c_float)


def _p(a, typ):
    return None if a is None else a.ctypes.data_as(typ)


class OrbOracle:
    def __init__(self):
        self.lib = L = C.CDLL(lib_path())
        L.orc_orb_level_size.restype = None
        L.orc_orb_level_size.argtypes = [C.c_int, C.c_int, C.c_double, C.c_int, _i32, _i32]
        L.orc_orb_resize.restype = None
        L.orc_orb_resize.argtypes = [_u8, C.c_int, C.c_int, _u8, C.c_int, C.c_int]
        L.orc_orb_blur.restype = None
        L.orc_orb_blur.argtypes = [_u8, C.c_int, C.c_int, _u8]
        L.orc_fast_atan2.restype = C.c_float
        L.orc_fast_atan2.argtypes = [C.c_float, C.c_float]
        L.orc_orb_ic_angle.restype = C.c_float
        L.orc_orb_ic_angle.argtypes = [_u8, C.c_int, C.c_int, C.c_int, C.c_int]
        L.orc_orb_pyramid.restype = C.c_size_t
        L.orc_orb_pyramid.argtypes = [_u8, C.c_int, C.c_int, C.c_int, C.c_double, _u8, _u8]
        L.orc_orb_pyramid_bytes.restype = C.c_size_t
        L.orc_orb_pyramid_bytes.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double]
        L.orc_orb_compute_batch.restype = None
        L.orc_orb_compute_batch.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, _u8, _i32, _f32, _i32,
                                            _f32, _f32, _u8, _i32, _i32, C.c_int]

    def level_size(self, W, H, scale, level):
        w, h = C.c_int32(), C.c_int32()
        self.lib.orc_orb_level_size(W, H, scale, level, C.byref(w), C.byref(h))
        return w.value, h.value

    def resize(self, img, w, h):
        img = np.ascontiguousarray(img, np.uint8)
        out = np.zeros((h, w), np.uint8)
        self.lib.orc_orb_resize(_p(img, _u8), img.shape[1], img.shape[0], _p(out, _u8), w, h)
        return out

    def blur(self, img):
        img = np.ascontiguousarray(img, np.uint8)
        out = np.zeros_like(img)
        self.lib.orc_orb_blur(_p(img, _u8), img.shape[1], img.shape[0], _p(out, _u8))
        return out

    def fast_atan2(self, y, x) -> float:
        return self.lib.orc_fast_atan2(y, x)

    def ic_angle(self, level, cx, cy) -> float:
        level = np.ascontiguousarray(level, np.uint8)
        return self.lib.orc_orb_ic_angle(_p(level, _u8), level.shape[1], level.shape[0], cx, cy)

    def pyramid(self, img, n_levels, scale):
        """[(raw, blurred)] per level."""
        img = np.ascontiguousarray(img, np.uint8)
        H, W = img.shape
        n = self.lib.orc_orb_pyramid_bytes(W, H, n_levels, scale)
        raw, blur = np.zeros(n + 1, np.uint8), np.zeros(n + 1, np.uint8)
        self.lib.orc_orb_pyramid(_p(img, _u8), W, H, n_levels, scale, _p(raw, _u8), _p(blur, _u8))
        out, off = [], 0
        for lvl in range(n_levels):
            w, h = self.level_size(W, H, scale, lvl)
            out.append((raw[off:off + w * h].reshape(h, w), blur[off:off + w * h].reshape(h, w)))
            off += w * h
        return out

    def compute_batch(self, images, kp_off, kp_xy, kp_oct, kp_angle=None, n_levels=4, scale=1.2, edge=19, threads=1):
        """images uint8[n, H, W]; returns (angle, desc, src_idx, counts) in the device layout: image i's survivors start at
        row kp_off[i]; rows past counts[i] are left zero (angle, desc) / -1 (src_idx)."""
        images = np.ascontiguousarray(images, np.uint8)
        n, H, W = images.shape
        kp_off = np.ascontiguousarray(kp_off, np.int32)
        kp_xy = np.ascontiguousarray(kp_xy, np.float32).reshape(-1, 2)
        kp_oct = np.ascontiguousarray(kp_oct, np.int32)
        kp_angle = None if kp_angle is None else np.ascontiguousarray(kp_angle, np.float32)
        N = int(kp_off[-1])
        angle, desc = np.zeros(N, np.float32), np.zeros((N, 32), np.uint8)
        src, counts = np.full(N, -1, np.int32), np.zeros(n, np.int32)
        self.lib.orc_orb_compute_batch(W, H, n_levels, scale, edge, n, _p(images, _u8), _p(kp_off, _i32), _p(kp_xy, _f32),
                                       _p(kp_oct, _i32), _p(kp_angle, _f32), _p(angle, _f32), _p(desc, _u8), _p(src, _i32),
                                       _p(counts, _i32), int(threads))
        return angle, desc, src, counts
