"""ctypes binding of oracle/_ref/libplstvo_ref_lbd.so: the reference's BinaryDescriptor::compute built from its own text
by oracle/make_ref_lbd.py.

TEST INFRASTRUCTURE: tests/ and tools/ import it; the product package never does.  The library exists only where the
recipe could run (it needs the reference checkout); available() says whether it is here."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import make_ref_lbd

LIB = make_ref_lbd.LIB
_lib = None


def available() -> bool:
    return os.path.exists(LIB)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        u8p, i16p, i32p, fp, dp = (C.POINTER(C.c_uint8), C.POINTER(C.c_int16), C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                   C.POINTER(C.c_double))
        L.lbd_ref_compute.restype = C.c_int
        L.lbd_ref_compute.argtypes = [C.c_int, C.c_int, u8p, C.c_int, fp, fp, i32p, u8p]
        L.lbd_ref_compute_batch.restype = C.c_int
        L.lbd_ref_compute_batch.argtypes = [C.c_int, C.c_int, C.c_int, u8p, i32p, fp, fp, i32p, u8p]
        L.lbd_ref_blur_sobel.restype = None
        L.lbd_ref_blur_sobel.argtypes = [C.c_int, C.c_int, u8p, u8p, i16p, i16p]
        L.lbd_ref_coefficients.restype = None
        L.lbd_ref_coefficients.argtypes = [dp, dp]
        _lib = L
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def compute(image, seg, angle, npix) -> np.ndarray:
    """Descriptors [n, 32] of one grey image's octave-0 key lines (seg [n, 4] in octave coordinates, angle, numOfPixels)."""
    image = np.ascontiguousarray(image, np.uint8)
    seg = np.ascontiguousarray(seg, np.float32).reshape(-1, 4)
    angle, npix = np.ascontiguousarray(angle, np.float32), np.ascontiguousarray(npix, np.int32)
    out = np.zeros((len(seg), 32), np.uint8)
    H, W = image.shape
    load().lbd_ref_compute(W, H, _p(image, C.c_uint8), len(seg), _p(seg, C.c_float), _p(angle, C.c_float),
                           _p(npix, C.c_int32), _p(out, C.c_uint8))
    return out


def compute_batch(images, kl_off, seg, angle, npix) -> np.ndarray:
    images = np.ascontiguousarray(images, np.uint8)
    n_img, H, W = images.shape
    kl_off = np.ascontiguousarray(kl_off, np.int32)
    seg = np.ascontiguousarray(seg, np.float32).reshape(-1, 4)
    angle, npix = np.ascontiguousarray(angle, np.float32), np.ascontiguousarray(npix, np.int32)
    out = np.zeros((len(seg), 32), np.uint8)
    load().lbd_ref_compute_batch(n_img, W, H, _p(images, C.c_uint8), _p(kl_off, C.c_int32), _p(seg, C.c_float),
                                 _p(angle, C.c_float), _p(npix, C.c_int32), _p(out, C.c_uint8))
    return out


def blur_sobel(image):
    """(blurred uint8, dx int16, dy int16) of the reference's computeSobel on the stand-in GaussianBlur / Sobel."""
    image = np.ascontiguousarray(image, np.uint8)
    H, W = image.shape
    b, dx, dy = np.zeros((H, W), np.uint8), np.zeros((H, W), np.int16), np.zeros((H, W), np.int16)
    load().lbd_ref_blur_sobel(W, H, _p(image, C.c_uint8), _p(b, C.c_uint8), _p(dx, C.c_int16), _p(dy, C.c_int16))
    return b, dx, dy


def coefficients():
    """(gaussCoefL_ [21], gaussCoefG_ [63]) of the default BinaryDescriptor, as doubles."""
    cl, cg = np.zeros(21), np.zeros(63)
    load().lbd_ref_coefficients(_p(cl, C.c_double), _p(cg, C.c_double))
    return cl, cg


def trig_binding() -> str:
    """'double' when the library calls the C double cos / sin (or sincos), 'float' for cosf / sinf (sincosf): which
    overload the reference's unqualified cos(float) took under the stand-in's name environment."""
    out = subprocess.run(["nm", "-D", "--undefined-only", LIB], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1].split("@")[0] for line in out.splitlines() if line.strip()}
    dbl, flt = names & {"cos", "sin", "sincos"}, names & {"cosf", "sinf", "sincosf"}
    if dbl and not flt:
        return "double"
    if flt and not dbl:
        return "float"
    raise RuntimeError(f"ambiguous trig binding: {sorted(dbl | flt)}")
