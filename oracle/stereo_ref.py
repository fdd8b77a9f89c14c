"""ctypes binding of oracle/_ref/libplstvo_ref_stereo.so: the reference's stereo step (matchGrid, getLineCoords,
lineSegmentOverlapStereo, matchStereoPoints / matchStereoLines) built from its own text by oracle/make_ref_stereo.py.

TEST INFRASTRUCTURE: tests/ and tools/ import it; the product package never does.  The library exists only where the
recipe could run (it needs the reference checkout); available() says whether it is here.  The calls mirror those of
oracle.oracle.Oracle with the same names, so either can be handed to the same check."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import make_ref_stereo
from stvo_pl_b200 import types as T

LIB = make_ref_stereo.LIB
_lib = None


def available() -> bool:
    return os.path.exists(LIB)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        i32p, u8p, fp, dp = C.POINTER(C.c_int32), C.POINTER(C.c_uint8), C.POINTER(C.c_float), C.POINTER(C.c_double)
        cam, mc, sc = C.POINTER(T.PlCamera), C.POINTER(T.PlStereoMatchConfig), C.POINTER(T.PlStereoConfig)
        L.stereo_ref_match_grid_points.restype = C.c_int
        L.stereo_ref_match_grid_points.argtypes = [C.c_int, C.c_int, T.PlGridWindow, C.c_int, C.c_double, C.c_int, i32p, u8p,
                                                   C.c_int, i32p, u8p, i32p]
        L.stereo_ref_match_grid_lines.restype = C.c_int
        L.stereo_ref_match_grid_lines.argtypes = [C.c_int, C.c_int, T.PlGridWindow, C.c_int, C.c_double, C.c_double, C.c_int,
                                                  i32p, u8p, C.c_int, dp, dp, u8p, i32p]
        L.stereo_ref_line_cells.restype = C.c_int
        L.stereo_ref_line_cells.argtypes = [C.c_double] * 4 + [i32p, C.c_int]
        L.stereo_ref_line_segment_overlap_stereo.restype = C.c_double
        L.stereo_ref_line_segment_overlap_stereo.argtypes = [sc] + [C.c_double] * 4
        L.stereo_ref_match_stereo_points.restype = C.c_int
        L.stereo_ref_match_stereo_points.argtypes = [cam, mc, sc, C.c_int, fp, i32p, u8p, C.c_int, fp, u8p, dp, dp, dp, dp, i32p,
                                                     u8p]
        L.stereo_ref_match_stereo_lines.restype = C.c_int
        L.stereo_ref_match_stereo_lines.argtypes = [cam, mc, sc, C.c_int, fp, fp, i32p, u8p, C.c_int, fp, u8p] + [dp] * 9 + \
                                                   [i32p, u8p]
        _lib = L
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def match_grid_points(q_cell, d1, t_cell, d2, window, ratio, best_lr=True, rows=T.GRID_ROWS, cols=T.GRID_COLS):
    q_cell = np.ascontiguousarray(q_cell, np.int32).reshape(-1, 2)
    t_cell = np.ascontiguousarray(t_cell, np.int32).reshape(-1, 2)
    d1, d2 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32), np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
    m12 = np.full(len(d1), -1, np.int32)
    n = load().stereo_ref_match_grid_points(rows, cols, window, int(best_lr), float(ratio), len(d1), _p(q_cell, C.c_int32),
                                            _p(d1, C.c_uint8), len(d2), _p(t_cell, C.c_int32), _p(d2, C.c_uint8),
                                            _p(m12, C.c_int32))
    return n, m12


def match_grid_lines(q_line, d1, t_line, t_dir, d2, window, ratio, line_sim_th, best_lr=True, rows=T.GRID_ROWS,
                     cols=T.GRID_COLS):
    q_line = np.ascontiguousarray(q_line, np.int32).reshape(-1, 4)
    t_line = np.ascontiguousarray(t_line, np.float64).reshape(-1, 4)
    t_dir = np.ascontiguousarray(t_dir, np.float64).reshape(-1, 2)
    d1, d2 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32), np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
    m12 = np.full(len(d1), -1, np.int32)
    n = load().stereo_ref_match_grid_lines(rows, cols, window, int(best_lr), float(ratio), float(line_sim_th), len(d1),
                                           _p(q_line, C.c_int32), _p(d1, C.c_uint8), len(d2), _p(t_line, C.c_double),
                                           _p(t_dir, C.c_double), _p(d2, C.c_uint8), _p(m12, C.c_int32))
    return n, m12


def line_cells(x1, y1, x2, y2, cap=4096):
    cells = np.zeros((cap, 2), np.int32)
    n = load().stereo_ref_line_cells(float(x1), float(y1), float(x2), float(y2), _p(cells, C.c_int32), cap)
    assert n <= cap, n
    return cells[:n]


def line_segment_overlap_stereo(scfg, spl_obs, epl_obs, spl_proj, epl_proj):
    return load().stereo_ref_line_segment_overlap_stereo(C.byref(scfg), float(spl_obs), float(epl_obs), float(spl_proj),
                                                          float(epl_proj))


def match_stereo_points(cam, mcfg, scfg, kp_l, octave_l, desc_l, kp_r, desc_r):
    """matchStereoPoints for one frame: (k, records) with the PointFeature fields pl, disp, P, sigma2, level and the
    rewritten pdesc_l rows as desc (the reference keeps no m12 or source index)."""
    kp_l, kp_r = np.ascontiguousarray(kp_l, np.float32).reshape(-1, 2), np.ascontiguousarray(kp_r, np.float32).reshape(-1, 2)
    octave_l = np.ascontiguousarray(octave_l, np.int32)
    desc_l, desc_r = np.ascontiguousarray(desc_l, np.uint8).reshape(-1, 32), np.ascontiguousarray(desc_r, np.uint8).reshape(-1, 32)
    n = len(kp_l)
    out = dict(pl=np.zeros((n, 2)), disp=np.zeros(n), P=np.zeros((n, 3)), sigma2=np.zeros(n), level=np.zeros(n, np.int32),
               desc=np.zeros((n, 32), np.uint8))
    k = load().stereo_ref_match_stereo_points(
        C.byref(cam), C.byref(mcfg), C.byref(scfg), n, _p(kp_l, C.c_float), _p(octave_l, C.c_int32), _p(desc_l, C.c_uint8),
        len(kp_r), _p(kp_r, C.c_float), _p(desc_r, C.c_uint8), _p(out["pl"], C.c_double), _p(out["disp"], C.c_double),
        _p(out["P"], C.c_double), _p(out["sigma2"], C.c_double), _p(out["level"], C.c_int32), _p(out["desc"], C.c_uint8))
    return k, {key: v[:k] for key, v in out.items()}


def match_stereo_lines(cam, mcfg, scfg, seg_l, angle_l, octave_l, desc_l, seg_r, desc_r):
    """matchStereoLines for one frame: (k, records) with the LineFeature fields and the rewritten ldesc_l rows as desc."""
    seg_l, seg_r = np.ascontiguousarray(seg_l, np.float32).reshape(-1, 4), np.ascontiguousarray(seg_r, np.float32).reshape(-1, 4)
    angle_l, octave_l = np.ascontiguousarray(angle_l, np.float32), np.ascontiguousarray(octave_l, np.int32)
    desc_l, desc_r = np.ascontiguousarray(desc_l, np.uint8).reshape(-1, 32), np.ascontiguousarray(desc_r, np.uint8).reshape(-1, 32)
    n = len(seg_l)
    out = dict(spl=np.zeros((n, 2)), epl=np.zeros((n, 2)), sdisp=np.zeros(n), edisp=np.zeros(n), sP=np.zeros((n, 3)),
               eP=np.zeros((n, 3)), le=np.zeros((n, 3)), angle=np.zeros(n), sigma2=np.zeros(n), level=np.zeros(n, np.int32),
               desc=np.zeros((n, 32), np.uint8))
    k = load().stereo_ref_match_stereo_lines(
        C.byref(cam), C.byref(mcfg), C.byref(scfg), n, _p(seg_l, C.c_float), _p(angle_l, C.c_float), _p(octave_l, C.c_int32),
        _p(desc_l, C.c_uint8), len(seg_r), _p(seg_r, C.c_float), _p(desc_r, C.c_uint8),
        *[_p(out[key], C.c_double) for key in ("spl", "epl", "sdisp", "edisp", "sP", "eP", "le", "angle", "sigma2")],
        _p(out["level"], C.c_int32), _p(out["desc"], C.c_uint8))
    return k, {key: v[:k] for key, v in out.items()}
