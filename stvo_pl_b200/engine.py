"""ctypes binding of the CUDA library (stvo_pl_b200/lib/libplstvo_b200.so) through its C-ABI
(include/plstvo.h).  There is no CPU fallback: a missing extension or a missing sm_90 device raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from . import types as T

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PLSTVO_LIB") or os.path.join(_HERE, "lib", "libplstvo_b200.so")   # PLSTVO_LIB: another build to load
PHASE_SLOTS = 32   # PLSTVO_PHASE_SLOTS

ERRORS = {-1: "PLSTVO_E_INVALID", -2: "PLSTVO_E_TOO_LARGE", -3: "PLSTVO_E_CUDA", -4: "PLSTVO_E_NO_DEVICE",
          -5: "PLSTVO_E_SIZE"}


class PlstvoError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"{ERRORS.get(code, code)}: {msg}")
        self.code = code


def load_library(path: str = LIB_PATH) -> C.CDLL:
    if not os.path.exists(path):
        raise RuntimeError(f"CUDA extension missing: {path}. Build it with `python -m stvo_pl_b200.build` "
                           "(there is no CPU fallback).")
    L = C.CDLL(path)
    vp, i32p, u8p, dp, fp = C.c_void_p, T.c_int32_p, T.c_uint8_p, T.c_double_p, T.c_float_p
    u32p, i16p, u16p = C.POINTER(C.c_uint32), C.POINTER(C.c_int16), C.POINTER(C.c_uint16)
    cam, cfg = C.POINTER(T.PlCamera), C.POINTER(T.PlConfig)
    fb, mb = C.POINTER(T.PlFrameBatch), C.POINTER(T.PlMatchedBatch)
    sig = {
        "plstvo_version": (C.c_int, []),
        "plstvo_create": (C.c_int, [C.c_int, C.POINTER(vp)]),
        "plstvo_destroy": (None, [vp]),
        "plstvo_last_error": (C.c_char_p, [vp]),
        "plstvo_default_config": (None, [cfg]),
        "plstvo_kitti_config": (None, [cfg]),
        "plstvo_match_nnr": (C.c_int, [vp, u8p, C.c_int, u8p, C.c_int, C.c_int, C.c_float, i32p]),
        "plstvo_match": (C.c_int, [vp, u8p, C.c_int, u8p, C.c_int, C.c_int, C.c_float, C.c_int, i32p]),
        "plstvo_match_batch": (C.c_int, [vp, C.c_int, u8p, i32p, u8p, i32p, C.c_float, C.c_int, i32p, i32p]),
        "plstvo_match_grid_points": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, T.PlGridWindow, C.c_int, C.c_double, i32p, i32p,
                                               u8p, i32p, i32p, u8p, i32p, i32p]),
        "plstvo_match_grid_lines": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, T.PlGridWindow, C.c_int, C.c_double,
                                              C.c_double, i32p, i32p, u8p, i32p, dp, dp, u8p, i32p, i32p]),
        "plstvo_default_stereo_config": (None, [C.POINTER(T.PlStereoConfig)]),
        "plstvo_stereo_lift_points": (C.c_int, [vp, cam, C.POINTER(T.PlStereoConfig), C.c_int, i32p, fp, i32p, u8p, i32p, fp,
                                                i32p, dp, dp, dp, dp, i32p, u8p, i32p, i32p]),
        "plstvo_stereo_lift_lines": (C.c_int, [vp, cam, C.POINTER(T.PlStereoConfig), C.c_int, i32p, fp, fp, i32p, u8p, i32p,
                                               fp, i32p, dp, dp, dp, dp, dp, dp, dp, dp, dp, i32p, u8p, i32p, i32p]),
        "plstvo_default_stereo_match_config": (None, [C.POINTER(T.PlStereoMatchConfig)]),
        "plstvo_match_stereo_points": (C.c_int, [vp, cam, C.POINTER(T.PlStereoMatchConfig), C.POINTER(T.PlStereoConfig), C.c_int,
                                                 i32p, fp, i32p, u8p, i32p, fp, u8p, i32p, dp, dp, dp, dp, i32p, u8p, i32p, i32p]),
        "plstvo_match_stereo_lines": (C.c_int, [vp, cam, C.POINTER(T.PlStereoMatchConfig), C.POINTER(T.PlStereoConfig), C.c_int,
                                                i32p, fp, fp, i32p, u8p, i32p, fp, u8p, i32p, dp, dp, dp, dp, dp, dp, dp, dp, dp,
                                                i32p, u8p, i32p, i32p]),
        "plstvo_track_stereo_batch": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig), C.POINTER(T.PlStereoConfig),
                                                C.POINTER(T.PlStereoFeatures), C.POINTER(T.PlStereoFeatures), vp, vp, i32p]),
        "plstvo_track_stereo_sequence": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig), C.POINTER(T.PlStereoConfig),
                                                   C.POINTER(T.PlStereoFeatures), vp, vp, i32p]),
        "plstvo_track_stereo_batch_async": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig), C.POINTER(T.PlStereoConfig),
                                                      C.POINTER(T.PlStereoFeatures), C.POINTER(T.PlStereoFeatures), vp, vp, i32p]),
        "plstvo_track_stereo_sequence_async": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig), C.POINTER(T.PlStereoConfig),
                                                         C.POINTER(T.PlStereoFeatures), vp, vp, i32p]),
        "plstvo_f2f_tracking": (C.c_int, [vp, cfg, fb, fb, i32p, i32p, i32p]),
        "plstvo_optimize_pose": (C.c_int, [vp, cam, cfg, mb, vp, vp, u8p, u8p]),
        "plstvo_track_batch": (C.c_int, [vp, cam, cfg, fb, fb, vp, vp, i32p, i32p, u8p, u8p]),
        "plstvo_track_batch_cams": (C.c_int, [vp, cam, cfg, fb, fb, vp, vp, i32p, i32p, u8p, u8p]),
        "plstvo_track_batch_async": (C.c_int, [vp, cam, cfg, fb, fb, vp, vp, i32p, i32p, u8p, u8p]),
        "plstvo_wait": (C.c_int, [vp, C.c_int]),
        "plstvo_batch_upload": (C.c_int, [vp, cam, cfg, fb, fb, vp, C.POINTER(vp)]),
        "plstvo_batch_run": (C.c_int, [vp, vp]),
        "plstvo_batch_run_timed": (C.c_int, [vp, vp, C.c_int, C.c_int, C.POINTER(C.c_float)]),
        "plstvo_batch_download": (C.c_int, [vp, vp, vp, i32p, i32p, u8p, u8p]),
        "plstvo_batch_free": (None, [vp, vp]),
        "plstvo_synchronize": (C.c_int, [vp]),
        "plstvo_host_alloc": (vp, [C.c_size_t]),
        "plstvo_host_free": (None, [vp]),
        "plstvo_launch_count": (C.c_int64, [vp]),
        "plstvo_batch_kernel_times": (C.c_int, [vp, vp, C.c_int, dp, dp, i32p, i32p]),
        "plstvo_batch_stage_times": (C.c_int, [vp, vp, C.c_int, dp, i32p]),
        "plstvo_batch_phase_cycles": (C.c_int, [vp, vp, C.POINTER(C.c_int64)]),
        "plstvo_gn_eval_stream": (C.c_int, [vp, cam, cfg, mb, dp, C.c_int, dp, dp, dp, C.POINTER(C.c_float)]),
        "plstvo_popc_rate": (C.c_int, [vp, dp]),
        "plstvo_debug_algebra": (C.c_int, [vp, C.c_int, dp, dp, dp, dp, dp, dp]),
        "plstvo_debug_pose_helpers": (C.c_int, [vp, C.c_int, dp, dp]),
        "plstvo_debug_keyframe": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, vp]),
        "plstvo_debug_select": (C.c_int, [vp, C.c_int, i32p, dp, i32p, dp, C.c_int, dp]),
        "plstvo_debug_tc_partials": (C.c_int, [vp, C.c_int, u8p, i32p, u8p, i32p, C.c_float, u32p, u32p, u32p, u32p]),
        "plstvo_debug_color_planes": (C.c_int, [vp, vp, C.POINTER(vp), C.c_int, u8p, u8p, u8p, u8p]),
        "plstvo_default_orb_config": (None, [C.POINTER(T.PlOrbConfig)]),
        "plstvo_orb_compute_batch": (C.c_int, [vp, C.POINTER(T.PlOrbConfig), C.c_int, C.c_int, C.c_int, u8p, i32p, fp, i32p, fp,
                                               fp, u8p, i32p, i32p]),
        "plstvo_orb_kernel_times": (C.c_int, [vp, fp]),
        "plstvo_default_orb_detect_config": (None, [C.POINTER(T.PlOrbDetectConfig)]),
        "plstvo_orb_detect_and_compute_batch": (C.c_int, [vp, C.POINTER(T.PlOrbDetectConfig), C.c_int, C.c_int, C.c_int, u8p,
                                                          i32p, C.c_int, i32p, fp, i32p, fp, fp, u8p]),
        "plstvo_orb_detect_kernel_times": (C.c_int, [vp, fp]),
        "plstvo_lbd_compute_batch": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, u8p, i32p, fp, fp, i32p, u8p]),
        "plstvo_lbd_kernel_times": (C.c_int, [vp, fp]),
        "plstvo_default_lsd_config": (None, [C.POINTER(T.PlLsdConfig)]),
        "plstvo_lsd_detect_batch": (C.c_int, [vp, C.POINTER(T.PlLsdConfig), C.c_int, C.c_int, C.c_int, u8p, C.c_int, i32p, fp, fp,
                                              i32p, fp, fp]),
        "plstvo_lsd_kernel_times": (C.c_int, [vp, fp]),
        "plstvo_fld_key_lines": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, fp, fp, fp, i32p, fp, fp]),
        "plstvo_track_stereo_images_batch": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig), C.POINTER(T.PlStereoConfig),
                                                       C.POINTER(T.PlOrbDetectConfig), C.POINTER(T.PlStereoImages),
                                                       C.POINTER(T.PlStereoImages), vp, vp, i32p]),
        "plstvo_track_stereo_images_sequence": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig),
                                                          C.POINTER(T.PlStereoConfig), C.POINTER(T.PlOrbDetectConfig),
                                                          C.POINTER(T.PlStereoImages), vp, vp, i32p]),
        "plstvo_track_stereo_images_lsd_batch": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig),
                                                           C.POINTER(T.PlStereoConfig), C.POINTER(T.PlOrbDetectConfig),
                                                           C.POINTER(T.PlLsdConfig), C.POINTER(T.PlStereoImages),
                                                           C.POINTER(T.PlStereoImages), vp, vp, i32p]),
        "plstvo_track_stereo_images_lsd_sequence": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig),
                                                              C.POINTER(T.PlStereoConfig), C.POINTER(T.PlOrbDetectConfig),
                                                              C.POINTER(T.PlLsdConfig), C.POINTER(T.PlStereoImages), vp, vp, i32p]),
        "plstvo_track_stereo_images_stage_times": (C.c_int, [vp, fp]),
        "plstvo_init_undistort_rectify_map": (C.c_int, [C.POINTER(T.PlRectifyModel), C.c_int, C.c_int, i16p, u16p]),
        "plstvo_rectifier_create": (vp, [vp, C.c_int, C.c_int, i16p, u16p, i16p, u16p]),
        "plstvo_rectifier_create_color": (vp, [vp, C.c_int, C.c_int, C.c_int, i16p, u16p, i16p, u16p]),
        "plstvo_rectifier_destroy": (None, [vp]),
        "plstvo_rectify_batch": (C.c_int, [vp, vp, C.c_int, u8p, u8p, u8p, u8p]),
        "plstvo_rectify_kernel_times": (C.c_int, [vp, fp]),
        "plstvo_track_stereo_raw_images_batch": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig),
                                                           C.POINTER(T.PlStereoConfig), C.POINTER(T.PlOrbDetectConfig),
                                                           C.POINTER(T.PlLsdConfig), vp, C.POINTER(T.PlStereoImages),
                                                           C.POINTER(T.PlStereoImages), vp, vp, i32p]),
        "plstvo_track_stereo_raw_images_sequence": (C.c_int, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig),
                                                              C.POINTER(T.PlStereoConfig), C.POINTER(T.PlOrbDetectConfig),
                                                              C.POINTER(T.PlLsdConfig), vp, C.POINTER(T.PlStereoImages), vp, vp,
                                                              i32p]),
        "plstvo_stereo_session_create": (vp, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig), C.POINTER(T.PlStereoConfig),
                                              C.POINTER(T.PlOrbDetectConfig), C.POINTER(T.PlLsdConfig), vp, C.c_int]),
        "plstvo_stereo_session_create_cams": (vp, [vp, cam, cfg, C.POINTER(T.PlStereoMatchConfig),
                                                   C.POINTER(T.PlStereoConfig), C.POINTER(T.PlOrbDetectConfig),
                                                   C.POINTER(T.PlLsdConfig), C.POINTER(vp), C.c_int]),
        "plstvo_stereo_session_destroy": (None, [vp]),
        "plstvo_stereo_session_device_bytes": (C.c_int64, [vp]),
        "plstvo_stereo_session_initialize": (C.c_int, [vp, vp, C.c_int, i32p, C.POINTER(T.PlStereoImages), i32p]),
        "plstvo_stereo_session_insert": (C.c_int, [vp, vp, C.c_int, i32p, C.POINTER(T.PlStereoImages), vp, vp, i32p]),
        "plstvo_stereo_session_retain": (C.c_int, [vp, vp, C.c_int]),
        "plstvo_stereo_session_use_fld_lines": (C.c_int, [vp, vp, C.c_int]),
        "plstvo_stereo_session_read": (C.c_int, [vp, vp, C.POINTER(T.PlStereoFrameOut)]),
        "plstvo_stereo_session_plot": (C.c_int, [vp, vp, C.c_int]),
        "plstvo_stereo_session_read_plot": (C.c_int, [vp, vp, C.POINTER(C.c_uint8)]),
        "plstvo_default_handler_config": (None, [C.POINTER(T.PlHandlerConfig)]),
        "plstvo_kitti_handler_config": (None, [C.POINTER(T.PlHandlerConfig)]),
        "plstvo_stereo_session_run": (C.c_int, [vp, vp, C.POINTER(T.PlHandlerConfig), C.c_int, i32p, C.c_int,
                                                C.POINTER(T.PlStereoImages), i32p, vp, vp, i32p, i32p]),
        "plstvo_default_keyframe_config": (None, [vp]),
        "plstvo_initial_keyframe_state": (None, [vp]),
        "plstvo_stereo_session_run_keyframes": (C.c_int, [vp, vp, C.POINTER(T.PlHandlerConfig), vp, C.c_int, i32p, C.c_int,
                                                          C.POINTER(T.PlStereoImages), i32p, vp, vp, vp, vp, i32p, i32p]),
        "plstvo_stereo_session_read_keyframes": (C.c_int, [vp, vp, C.POINTER(T.PlStereoFrameOut), i32p]),
        "plstvo_stereo_session_run_schedule": (C.c_int, [vp, vp, C.POINTER(T.PlHandlerConfig), vp, C.c_int, i32p, C.c_int,
                                                         C.POINTER(C.c_uint8), C.POINTER(T.PlStereoImages), i32p, vp, vp, vp,
                                                         vp, i32p, i32p]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)   # AttributeError if the library does not export a declared symbol
        fn.restype, fn.argtypes = res, args
    return L


EXPORTED_SYMBOLS = [
    "plstvo_version", "plstvo_create", "plstvo_destroy", "plstvo_last_error", "plstvo_default_config",
    "plstvo_kitti_config", "plstvo_match_nnr", "plstvo_match", "plstvo_match_batch", "plstvo_match_grid_points",
    "plstvo_match_grid_lines", "plstvo_default_stereo_config", "plstvo_stereo_lift_points", "plstvo_stereo_lift_lines",
    "plstvo_default_stereo_match_config", "plstvo_match_stereo_points", "plstvo_match_stereo_lines", "plstvo_track_stereo_batch",
    "plstvo_track_stereo_sequence", "plstvo_track_stereo_batch_async", "plstvo_track_stereo_sequence_async",
    "plstvo_f2f_tracking",
    "plstvo_optimize_pose", "plstvo_track_batch", "plstvo_track_batch_async", "plstvo_wait", "plstvo_batch_upload", "plstvo_batch_run",
    "plstvo_batch_run_timed", "plstvo_batch_download", "plstvo_batch_free", "plstvo_synchronize",
    "plstvo_host_alloc", "plstvo_host_free", "plstvo_launch_count", "plstvo_batch_kernel_times", "plstvo_batch_stage_times",
    "plstvo_batch_phase_cycles",
    "plstvo_gn_eval_stream", "plstvo_popc_rate", "plstvo_debug_algebra", "plstvo_debug_pose_helpers",
    "plstvo_debug_keyframe", "plstvo_debug_select", "plstvo_debug_tc_partials", "plstvo_debug_color_planes",
    "plstvo_default_orb_config", "plstvo_orb_compute_batch", "plstvo_orb_kernel_times",
    "plstvo_default_orb_detect_config", "plstvo_orb_detect_and_compute_batch", "plstvo_orb_detect_kernel_times",
    "plstvo_lbd_compute_batch", "plstvo_lbd_kernel_times", "plstvo_default_lsd_config", "plstvo_lsd_detect_batch",
    "plstvo_lsd_kernel_times", "plstvo_track_stereo_images_batch",
    "plstvo_track_stereo_images_sequence", "plstvo_track_stereo_images_lsd_batch", "plstvo_track_stereo_images_lsd_sequence",
    "plstvo_track_stereo_images_stage_times", "plstvo_init_undistort_rectify_map", "plstvo_rectifier_create",
    "plstvo_rectifier_destroy", "plstvo_rectify_batch", "plstvo_rectify_kernel_times", "plstvo_track_stereo_raw_images_batch",
    "plstvo_track_stereo_raw_images_sequence", "plstvo_stereo_session_create", "plstvo_stereo_session_destroy",
    "plstvo_stereo_session_device_bytes", "plstvo_stereo_session_initialize", "plstvo_stereo_session_insert",
    "plstvo_rectifier_create_color", "plstvo_stereo_session_retain", "plstvo_stereo_session_read",
    "plstvo_track_batch_cams", "plstvo_stereo_session_create_cams", "plstvo_default_handler_config",
    "plstvo_kitti_handler_config", "plstvo_stereo_session_run", "plstvo_default_keyframe_config",
    "plstvo_initial_keyframe_state", "plstvo_stereo_session_run_keyframes", "plstvo_stereo_session_read_keyframes",
    "plstvo_fld_key_lines", "plstvo_stereo_session_use_fld_lines", "plstvo_stereo_session_run_schedule",
    "plstvo_stereo_session_plot", "plstvo_stereo_session_read_plot"]


def _p(a: Optional[np.ndarray], typ):
    return C.cast(None, typ) if a is None else a.ctypes.data_as(typ)


def _record_ptrs(out: dict, records):
    """Pointers to out's arrays (Engine.stereo_outputs' keys) of the given lifted records, in their C argument order."""
    return [_p(out[r.key], r.ctype) for r in records]


def fld_key_lines(width: int, height: int, n_features: int, seg, lib: Optional[C.CDLL] = None):
    """plstvo_fld_key_lines (host code, no GPU): the reference's FLD-branch key lines of one width x height image from
    FastLineDetector's segments seg float32[n, 4] in its order.  Returns dict(seg [m, 4], angle, npix, response, length), m =
    min(n, n_features) (n where n_features is 0), in the reference's order."""
    lib = lib or load_library()
    seg = np.ascontiguousarray(seg, np.float32).reshape(-1, 4)
    m = len(seg) if n_features == 0 else min(len(seg), max(int(n_features), 0))
    out = dict(seg=np.zeros((m, 4), np.float32), angle=np.zeros(m, np.float32), npix=np.zeros(m, np.int32),
               response=np.zeros(m, np.float32), length=np.zeros(m, np.float32))
    rc = lib.plstvo_fld_key_lines(width, height, n_features, len(seg), _p(seg, T.c_float_p), _p(out["seg"], T.c_float_p),
                                  _p(out["angle"], T.c_float_p), _p(out["npix"], T.c_int32_p),
                                  _p(out["response"], T.c_float_p), _p(out["length"], T.c_float_p))
    if rc < 0:
        raise PlstvoError(rc, "plstvo_fld_key_lines rejected the size, n_features or the segments")
    assert rc == m
    return out


def init_undistort_rectify_map(model: int, K, D, R, P, width: int, height: int, lib: Optional[C.CDLL] = None):
    """plstvo_init_undistort_rectify_map (host code, no GPU): (map1 int16[h, w, 2], map2 uint16[h, w]) as OpenCV 4.13 builds
    them for CV_16SC2.  model: T.RECTIFY_PINHOLE or T.RECTIFY_FISHEYE."""
    lib = lib or load_library()
    m = T.rectify_model(model, K, D, R, P)
    map1 = np.zeros((max(height, 0), max(width, 0), 2), np.int16)
    map2 = np.zeros((max(height, 0), max(width, 0)), np.uint16)
    rc = lib.plstvo_init_undistort_rectify_map(C.byref(m), width, height, _p(map1, C.POINTER(C.c_int16)),
                                               _p(map2, C.POINTER(C.c_uint16)))
    if rc < 0:
        raise PlstvoError(rc, "plstvo_init_undistort_rectify_map rejected the model or the size")
    return map1, map2


class Rectifier:
    """A PlRectifier: a rig's maps resident in HBM (Engine.rectifier_create), or for colour images (channels 3 or 4) the
    conversion to grey with or without maps (Engine.rectifier_create_color); close() or the owning Engine frees it."""

    def __init__(self, lib: C.CDLL, handle, width: int, height: int, channels: int = 1):
        self.lib, self.handle, self.width, self.height, self.channels = lib, handle, width, height, channels

    def image_shape(self, B: int):
        """The shape of B raw images this rectifier takes: uint8[B, H, W] grey, uint8[B, H, W, C] colour."""
        return (B, self.height, self.width) + ((self.channels,) if self.channels > 1 else ())

    def check_frames(self, *frame_sets):
        """ValueError unless each dict's img_l / img_r hold images of this rectifier's size and channels."""
        for fs in frame_sets:
            il, ir = (np.asarray(fs[k]) for k in ("img_l", "img_r"))
            if il.shape != ir.shape or il.shape != self.image_shape(il.shape[0] if il.ndim else 0):
                raise ValueError(f"images must be uint8{list(self.image_shape(il.shape[0] if il.ndim else 0))} "
                                 "(B images of the rectifier's size and channels), both sides alike")

    def close(self):
        if self.handle:
            self.lib.plstvo_rectifier_destroy(self.handle)
            self.handle = None


class StereoSession:
    """A PlStereoSession: n_streams stereo streams, each stream's previous frame kept in HBM as its stereo features
    (Engine.stereo_session_create).  initialize / insert name any subset of the streams; close() or the owning Engine frees it."""

    def __init__(self, eng: "Engine", handle, n_streams: int, rect: Optional[Rectifier] = None, size=(0, 0)):
        self.eng, self.handle, self.n_streams, self.rect = eng, handle, n_streams, rect
        self.width, self.height = size   # the cameras' image size, which sizes read_plot()'s images
        self.last = None   # the last call, if it succeeded: (insert, n_stereo), which sizes read()'s arrays

    def check_frames(self, frames: dict):
        """ValueError unless a colour session's frames are colour images of its rectifier's size and channels."""
        if self.rect is not None and self.rect.channels > 1:
            self.rect.check_frames(frames)

    def initialize(self, ids, frames: dict):
        """initialize(img_l, img_r) for streams ids: frames holds len(ids) frames (img_l / img_r uint8[n, H, W], or
        uint8[n, H, W, C] with a colour rectifier, optionally fast_th [n]).  Returns n_stereo [n, 2]."""
        return self.eng.stereo_session_initialize(self, ids, frames)

    def insert(self, ids, frames: dict, priors=None, results=None):
        """insertStereoPair + optimizePose for streams ids against their kept frames, which the new frames then replace.
        Returns (results [n], n_stereo [n, 4])."""
        return self.eng.stereo_session_insert(self, ids, frames, priors, results)

    def run(self, hcfg, ids, T_: int, frames: dict, fast_th0=None, priors=None):
        """plstvo_stereo_session_run: T_ steps of the handler's loop (insert, optimizePose, updateFrame) for streams ids, the
        FAST threshold and the prior carried from step to step on the device.  hcfg: a T.PlHandlerConfig or a
        handler.HandlerConfig.  frames holds T_ * len(ids) frames, step-major (no fast_th); fast_th0 and priors (optional)
        one entry per stream.  Returns (results [T_, n], fast_th [T_ + 1, n], n_stereo [T_, n, 4]); fast_th's last row is
        the next frame's threshold (for T_ = 0, fast_th0 with 0 mapped to the configured threshold)."""
        return self.eng.stereo_session_run(self, hcfg, ids, T_, frames, fast_th0, priors)

    def run_keyframes(self, hcfg, kcfg, ids, T_: int, frames: dict, kf_state, fast_th0=None, priors=None):
        """plstvo_stereo_session_run_keyframes: run() with the key-frame test (needNewKF, then currFrameIsKF where it fires)
        after each step's optimizePose.  kcfg: a T.KEYFRAME_CONFIG_DTYPE record or a handler.HandlerConfig; kf_state: one
        T.KEYFRAME_STATE_DTYPE record per stream (handler.KeyframeTest.to_state()), updated in place on success.  Returns
        (results [T_, n], kf [T_, n] of T.KEYFRAME_RESULT_DTYPE, fast_th [T_ + 1, n], n_stereo [T_, n, 4])."""
        return self.eng.stereo_session_run_keyframes(self, hcfg, kcfg, ids, T_, frames, kf_state, fast_th0, priors)

    def run_schedule(self, hcfg, ids, schedule, frames: dict, fast_th0=None, priors=None, kcfg=None, kf_state=None):
        """plstvo_stereo_session_run_schedule: run() / run_keyframes() over uneven streams.  schedule uint8 [T_, len(ids)]: 0
        the stream idles at that step, 1 insert, 2 initialize; frames holds one frame per non-zero entry, step-major and in ids
        order within a step (handler.schedule_frames packs them), fast_th optional (initialize entries' thresholds, 0 for
        inserts).  kcfg None: no key-frame test (kf_state must be None); else kf_state as for run_keyframes, updated in place.
        Returns (results [T_, n], fast_th [T_ + 1, n], n_stereo [T_, n, 4]), with kcfg (results, kf [T_, n], fast_th,
        n_stereo); the rows of entries that are not inserts are zero in results and kf, and in n_stereo where the stream
        idles."""
        return self.eng.stereo_session_run_schedule(self, hcfg, ids, schedule, frames, fast_th0, priors, kcfg, kf_state)

    def read_keyframes(self):
        """plstvo_stereo_session_read_keyframes: (rows [n_kf, 4] of step, stream id, points, lines; pt; ls), pt / ls holding
        the key frames' records in (step, call position) order under the keys of read()'s."""
        lib, ctx = self.eng.lib, self.eng.ctx
        empty = T.PlStereoFrameOut()
        n_kf = self.eng._ck(lib.plstvo_stereo_session_read_keyframes(ctx, self.handle, C.byref(empty), None))
        rows = np.zeros((n_kf, 4), np.int32)
        self.eng._ck(lib.plstvo_stereo_session_read_keyframes(ctx, self.handle, C.byref(empty), _p(rows, T.c_int32_p)))
        pt, ls, o = self._frame_out(rows[:, 2:])
        got = self.eng._ck(lib.plstvo_stereo_session_read_keyframes(ctx, self.handle, C.byref(o), None))
        if got != n_kf:
            raise PlstvoError(-1, f"plstvo_stereo_session_read_keyframes returned {got} key frames, then {n_kf}")
        return rows, pt, ls

    def use_fld_lines(self, on: bool):
        """plstvo_stereo_session_use_fld_lines: the reference's FLD line branch.  On, every call takes each frame's key lines
        from frames under the images call's keys (ll_off / lr_off, seg_l / seg_r, angle_l / angle_r, npix_l / npix_r, e.g.
        from fld_key_lines; step-major for run / run_keyframes) instead of running LSD.  Only while no stream holds a frame."""
        self.eng._ck(self.eng.lib.plstvo_stereo_session_use_fld_lines(self.eng.ctx, self.handle, 1 if on else 0))

    def retain(self, on: bool):
        """plstvo_stereo_session_retain: from the next initialize / insert on, keep each call's new frames and matches on the
        device for read(); off frees them."""
        self.eng._ck(self.eng.lib.plstvo_stereo_session_retain(self.eng.ctx, self.handle, 1 if on else 0))

    def plot(self, on: bool):
        """plstvo_stereo_session_plot: from the next initialize / insert on, draw each new frame's plotStereoFrame image on the
        device for read_plot() (retention must be on); off frees them."""
        self.eng._ck(self.eng.lib.plstvo_stereo_session_plot(self.eng.ctx, self.handle, 1 if on else 0))

    def read_plot(self) -> np.ndarray:
        """plstvo_stereo_session_read_plot of the last initialize / insert: uint8[n, H, W, 3], each new frame's left image
        (rectified, in BGR) with its stereo points' circles and stereo lines drawn in (0, 200, 0), in call order."""
        n = len(self.last[1]) if self.last is not None else 0
        out = np.zeros((max(n, 1), self.height, self.width, 3), np.uint8)
        got = self.eng._ck(self.eng.lib.plstvo_stereo_session_read_plot(self.eng.ctx, self.handle, _p(out, T.c_uint8_p)))
        if got != n:
            raise PlstvoError(-1, f"plstvo_stereo_session_read_plot returned {got} frames, the last call had {n}")
        return out[:n]

    def read(self):
        """plstvo_stereo_session_read of the last call: (pt, ls, m12_pt, inlier_pt, m12_ls, inlier_ls).  pt / ls hold the new
        frames' records in call order under the keys of Engine.match_stereo_points / _lines (counts: each frame's rows); the
        tracker's rows are indexed by the kept frames' features in call order, and are None after an initialize."""
        track, ns = self.last if self.last is not None else (False, np.zeros((0, 2), np.int32))
        n = len(ns)
        pt, ls, o = self._frame_out(ns[:, -2:])
        kp, kl = (int(ns[:, 0].sum()), int(ns[:, 1].sum())) if track else (0, 0)
        m12_pt, m12_ls = np.full(kp, -1, np.int32), np.full(kl, -1, np.int32)
        inl_pt, inl_ls = np.zeros(kp, np.uint8), np.zeros(kl, np.uint8)
        o.m12_pt, o.m12_ls = m12_pt.ctypes.data_as(T.c_int32_p), m12_ls.ctypes.data_as(T.c_int32_p)
        o.inlier_pt, o.inlier_ls = inl_pt.ctypes.data_as(T.c_uint8_p), inl_ls.ctypes.data_as(T.c_uint8_p)
        got = self.eng._ck(self.eng.lib.plstvo_stereo_session_read(self.eng.ctx, self.handle, C.byref(o)))
        if got != n:
            raise PlstvoError(-1, f"plstvo_stereo_session_read returned {got} frames, the last call had {n}")
        if not track:
            return pt, ls, None, None, None, None
        return pt, ls, m12_pt, inl_pt, m12_ls, inl_ls

    def _frame_out(self, counts):
        """The point and line dicts of read() for frames of counts [n, 2] (points, lines each) and a PlStereoFrameOut whose
        lifted fields point at them (the tracker's left NULL)."""
        pt = self.eng.stereo_outputs(int(counts[:, 0].sum()), len(counts), lines=False)
        ls = self.eng.stereo_outputs(int(counts[:, 1].sum()), len(counts), lines=True)
        for d, col in ((pt, 0), (ls, 1)):
            del d["m12"]
            d["counts"][...] = counts[:, col]
        o = T.PlStereoFrameOut()
        for r in T.FRAME_OUT_RECORDS:
            setattr(o, r.field, (pt if r.point else ls)[r.key].ctypes.data_as(r.ctype))
        return pt, ls, o

    @property
    def device_bytes(self) -> int:
        return int(self.eng.lib.plstvo_stereo_session_device_bytes(self.handle)) if self.handle else 0

    def close(self):
        if self.handle:
            self.eng.lib.plstvo_stereo_session_destroy(self.handle)
            self.handle = None


def bind_to_gpu_numa(device: int) -> Optional[int]:
    """Restricts the calling process to the CPUs of the NUMA node the GPU hangs off, so that pinned buffers allocated afterwards
    are local to the GPU's PCIe root (matters with one process per GPU on a two-socket host: the e2e path moves ~40 GB/s per
    GPU).  Returns the node, or None when the topology cannot be read (nothing is changed then)."""
    import os
    try:
        import torch
        bus = torch.cuda.get_device_properties(device).pci_bus_id
        dom = torch.cuda.get_device_properties(device).pci_domain_id
        dev = torch.cuda.get_device_properties(device).pci_device_id
        path = f"/sys/bus/pci/devices/{dom:04x}:{bus:02x}:{dev:02x}.0/numa_node"
        node = int(open(path).read().strip())
        if node < 0:
            return None
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        cpus &= os.sched_getaffinity(0)
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return node
    except Exception:
        return None


class PinnedPool:
    """Pinned host arrays (cudaMallocHost) so that H2D/D2H run at full PCIe rate without staging."""

    def __init__(self, lib):
        self.lib = lib
        self._ptrs = []

    def empty(self, shape, dtype) -> np.ndarray:
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        ptr = self.lib.plstvo_host_alloc(max(n, 1))
        if not ptr:
            raise MemoryError("cudaMallocHost failed")
        self._ptrs.append(ptr)
        buf = (C.c_uint8 * max(n, 1)).from_address(ptr)
        return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def copy(self, a: Optional[np.ndarray]) -> Optional[np.ndarray]:
        if a is None:
            return None
        out = self.empty(a.shape, a.dtype)
        out[...] = a
        return out

    def pin_frames(self, f: T.FrameBatch) -> T.FrameBatch:
        return T.FrameBatch(**{k: self.copy(getattr(f, k)) for k in (
            "pt_off", "ls_off", "pdesc", "ldesc", "pt_P", "pt_pl", "pt_sigma2", "ls_sP", "ls_eP", "ls_le",
            "ls_spl", "ls_epl", "ls_sigma2", "ls_level")})

    def close(self):
        for p in self._ptrs:
            self.lib.plstvo_host_free(p)
        self._ptrs = []


class DeviceBatch:
    """Inputs resident in HBM (PlDeviceBatch)."""

    def __init__(self, eng: "Engine", handle, prev: T.FrameBatch):
        self.eng, self.handle = eng, handle
        self.B, self.n_pt, self.n_ls = prev.B, prev.n_pt, prev.n_ls

    def run(self):
        self.eng._ck(self.eng.lib.plstvo_batch_run(self.eng.ctx, self.handle))

    def run_timed(self, iters: int, flush_l2: bool = False) -> float:
        ms = C.c_float(0)
        self.eng._ck(self.eng.lib.plstvo_batch_run_timed(self.eng.ctx, self.handle, iters, int(flush_l2), C.byref(ms)))
        return float(ms.value)

    def kernel_times(self, iters: int = 3):
        a, b = np.zeros(1), np.zeros(1)
        nt, npairs = np.zeros(1, np.int32), np.zeros(1, np.int32)
        self.eng._ck(self.eng.lib.plstvo_batch_kernel_times(
            self.eng.ctx, self.handle, iters, a.ctypes.data_as(T.c_double_p), b.ctypes.data_as(T.c_double_p),
            nt.ctypes.data_as(T.c_int32_p), npairs.ctypes.data_as(T.c_int32_p)))
        return dict(ms_match=float(a[0]), ms_solve=float(b[0]), n_tiles=int(nt[0]), n_pairs=int(npairs[0]))

    def stage_times(self, iters: int = 3):
        ms, cnt = np.zeros(8), np.zeros(4, np.int32)
        self.eng._ck(self.eng.lib.plstvo_batch_stage_times(self.eng.ctx, self.handle, iters, ms.ctypes.data_as(T.c_double_p),
                                                           cnt.ctypes.data_as(T.c_int32_p)))
        return dict(ms_expand=float(ms[0]), ms_distance=float(ms[1]), ms_resolve=float(ms[2]), ms_lists=float(ms[3]),
                    ms_solve=float(ms[3] + ms[4]), ms_optimize_pose=float(ms[4]), ms_gn_stage1=float(ms[5]),
                    ms_outliers=float(ms[6]), ms_gn_stage2=float(ms[7]),
                    tensor_core_form=bool(cnt[0] & 1), streamed_solver=bool(cnt[0] & 2), delegated_to_fp64=int(cnt[0] >> 8), n_items=int(cnt[1]),
                    n_problems=int(cnt[2]), n_pairs=int(cnt[3]))

    def phase_cycles(self):
        """One solve pass with the solver kernels' cycle counters on: [B][PHASE_SLOTS] int64 (layout in include/plstvo.h)."""
        out = np.zeros((self.B, PHASE_SLOTS), np.int64)
        self.eng._ck(self.eng.lib.plstvo_batch_phase_cycles(self.eng.ctx, self.handle, out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def download(self):
        res = np.zeros(self.B, dtype=T.POSE_RESULT_DTYPE)
        m12_pt, m12_ls = np.full(self.n_pt, -1, np.int32), np.full(self.n_ls, -1, np.int32)
        inl_pt, inl_ls = np.zeros(self.n_pt, np.uint8), np.zeros(self.n_ls, np.uint8)
        self.eng._ck(self.eng.lib.plstvo_batch_download(
            self.eng.ctx, self.handle, res.ctypes.data, _p(m12_pt, T.c_int32_p), _p(m12_ls, T.c_int32_p),
            _p(inl_pt, T.c_uint8_p), _p(inl_ls, T.c_uint8_p)))
        return dict(results=res, m12_pt=m12_pt, m12_ls=m12_ls, inlier_pt=inl_pt, inlier_ls=inl_ls)

    def free(self):
        if self.handle:
            self.eng.lib.plstvo_batch_free(self.eng.ctx, self.handle)
            self.handle = None


class Engine:
    """One PlContext (one GPU)."""

    def __init__(self, device: int = -1):
        self.lib = load_library()
        ctx = C.c_void_p()
        rc = self.lib.plstvo_create(device, C.byref(ctx))
        if rc != 0:
            raise PlstvoError(rc, "plstvo_create failed: no sm_90 CUDA device visible (no CPU fallback exists)")
        self.ctx = ctx
        self.pinned = PinnedPool(self.lib)
        self._rectifiers = []
        self._sessions = []

    def close(self):
        if self.ctx:
            for ss in self._sessions:
                ss.close()
            for r in self._rectifiers:
                r.close()
            self.pinned.close()
            self.lib.plstvo_destroy(self.ctx)
            self.ctx = None

    def _ck(self, rc: int) -> int:
        if rc < 0:
            raise PlstvoError(rc, (self.lib.plstvo_last_error(self.ctx) or b"").decode())
        return rc

    @property
    def launches(self) -> int:
        return int(self.lib.plstvo_launch_count(self.ctx))

    # ---- matching.h surface ----
    def match_nnr(self, d1, d2, nnr):
        d1, d2 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32), np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
        m12 = np.full(len(d1), -1, np.int32)
        n = self._ck(self.lib.plstvo_match_nnr(self.ctx, _p(d1, T.c_uint8_p), len(d1), _p(d2, T.c_uint8_p), len(d2),
                                               32, C.c_float(nnr), _p(m12, T.c_int32_p)))
        return n, m12

    def match(self, d1, d2, nnr, best_lr=True):
        d1, d2 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32), np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
        m12 = np.full(len(d1), -1, np.int32)
        n = self._ck(self.lib.plstvo_match(self.ctx, _p(d1, T.c_uint8_p), len(d1), _p(d2, T.c_uint8_p), len(d2), 32,
                                           C.c_float(nnr), int(best_lr), _p(m12, T.c_int32_p)))
        return n, m12

    def match_batch(self, d1, off1, d2, off2, nnr, best_lr=True):
        d1, d2 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32), np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
        off1, off2 = np.ascontiguousarray(off1, np.int32), np.ascontiguousarray(off2, np.int32)
        B = len(off1) - 1
        m12 = np.full(len(d1), -1, np.int32)
        counts = np.zeros(B, np.int32)
        n = self._ck(self.lib.plstvo_match_batch(self.ctx, B, _p(d1, T.c_uint8_p), _p(off1, T.c_int32_p),
                                                 _p(d2, T.c_uint8_p), _p(off2, T.c_int32_p), C.c_float(nnr),
                                                 int(best_lr), _p(m12, T.c_int32_p), _p(counts, T.c_int32_p)))
        return n, m12, counts

    def match_grid_points(self, q_off, q_cell, d1, t_off, t_cell, d2, window: T.PlGridWindow, ratio: float,
                          best_lr=True, rows=T.GRID_ROWS, cols=T.GRID_COLS):
        """StVO::matchGrid, points overload (src/matching.cpp:111-177), batched over frames."""
        q_off, t_off = np.ascontiguousarray(q_off, np.int32), np.ascontiguousarray(t_off, np.int32)
        q_cell, t_cell = np.ascontiguousarray(q_cell, np.int32).reshape(-1, 2), np.ascontiguousarray(t_cell, np.int32).reshape(-1, 2)
        d1, d2 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32), np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
        B = len(q_off) - 1
        m12, counts = np.full(len(d1), -1, np.int32), np.zeros(B, np.int32)
        n = self._ck(self.lib.plstvo_match_grid_points(
            self.ctx, B, rows, cols, window, int(best_lr), float(ratio), _p(q_off, T.c_int32_p), _p(q_cell, T.c_int32_p),
            _p(d1, T.c_uint8_p), _p(t_off, T.c_int32_p), _p(t_cell, T.c_int32_p), _p(d2, T.c_uint8_p),
            _p(m12, T.c_int32_p), _p(counts, T.c_int32_p)))
        return n, m12, counts

    def match_grid_lines(self, q_off, q_line, d1, t_off, t_line, t_dir, d2, window: T.PlGridWindow, ratio: float,
                         line_sim_th: float, best_lr=True, rows=T.GRID_ROWS, cols=T.GRID_COLS):
        """StVO::matchGrid, lines overload (src/matching.cpp:179-258), batched over frames."""
        q_off, t_off = np.ascontiguousarray(q_off, np.int32), np.ascontiguousarray(t_off, np.int32)
        q_line = np.ascontiguousarray(q_line, np.int32).reshape(-1, 4)
        t_line = np.ascontiguousarray(t_line, np.float64).reshape(-1, 4)
        t_dir = np.ascontiguousarray(t_dir, np.float64).reshape(-1, 2)
        d1, d2 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32), np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
        B = len(q_off) - 1
        m12, counts = np.full(len(d1), -1, np.int32), np.zeros(B, np.int32)
        n = self._ck(self.lib.plstvo_match_grid_lines(
            self.ctx, B, rows, cols, window, int(best_lr), float(ratio), float(line_sim_th), _p(q_off, T.c_int32_p),
            _p(q_line, T.c_int32_p), _p(d1, T.c_uint8_p), _p(t_off, T.c_int32_p), _p(t_line, T.c_double_p),
            _p(t_dir, T.c_double_p), _p(d2, T.c_uint8_p), _p(m12, T.c_int32_p), _p(counts, T.c_int32_p)))
        return n, m12, counts

    def stereo_lift_points(self, cam, scfg: T.PlStereoConfig, l_off, kp_l, octave_l, desc_l, r_off, kp_r, m12):
        """Stereo matches -> PointFeature records (src/stereoFrame.cpp:149-172), batched over frames.  Every output array has
        one slot per left keypoint; frame p's survivors are dense from l_off[p], counts[p] of them."""
        l_off, r_off = np.ascontiguousarray(l_off, np.int32), np.ascontiguousarray(r_off, np.int32)
        kp_l, kp_r = np.ascontiguousarray(kp_l, np.float32).reshape(-1, 2), np.ascontiguousarray(kp_r, np.float32).reshape(-1, 2)
        octave_l, m12 = np.ascontiguousarray(octave_l, np.int32), np.ascontiguousarray(m12, np.int32)
        desc_l = np.ascontiguousarray(desc_l, np.uint8).reshape(-1, 32)
        B, n = len(l_off) - 1, len(kp_l)
        out = self.stereo_outputs(n, B, lines=False)
        del out["m12"]
        total = self._ck(self.lib.plstvo_stereo_lift_points(
            self.ctx, C.byref(cam), C.byref(scfg), B, _p(l_off, T.c_int32_p), _p(kp_l, T.c_float_p), _p(octave_l, T.c_int32_p),
            _p(desc_l, T.c_uint8_p), _p(r_off, T.c_int32_p), _p(kp_r, T.c_float_p), _p(m12, T.c_int32_p),
            *_record_ptrs(out, T.FRAME_OUT_POINT_RECORDS), _p(out["counts"], T.c_int32_p)))
        return total, out

    def orb_compute_batch(self, cfg: T.PlOrbConfig, images, kp_off, kp_xy, kp_octave, kp_angle=None):
        """ORB angles and descriptors of given key points on images uint8[n, H, W] (OpenCV's ORB after key-point selection;
        kp_angle None: angles computed, as detectAndCompute does; else used as given, as ORB::compute does).  Image i's
        survivors of the border filter are rows kp_off[i] .. kp_off[i] + counts[i] of every output, in input order; later rows
        keep their initial value (angle 0, desc 0, src_idx -1)."""
        images = np.ascontiguousarray(images, np.uint8)
        n_img, H, W = images.shape
        kp_off = np.ascontiguousarray(kp_off, np.int32)
        kp_xy = np.ascontiguousarray(kp_xy, np.float32).reshape(-1, 2)
        kp_octave = np.ascontiguousarray(kp_octave, np.int32)
        kp_angle = None if kp_angle is None else np.ascontiguousarray(kp_angle, np.float32)
        n = len(kp_xy)
        out = dict(angle=np.zeros(n, np.float32), desc=np.zeros((n, 32), np.uint8), src_idx=np.full(n, -1, np.int32),
                   counts=np.zeros(n_img, np.int32))
        total = self._ck(self.lib.plstvo_orb_compute_batch(
            self.ctx, C.byref(cfg), n_img, W, H, _p(images, T.c_uint8_p), _p(kp_off, T.c_int32_p), _p(kp_xy, T.c_float_p),
            _p(kp_octave, T.c_int32_p), _p(kp_angle, T.c_float_p), _p(out["angle"], T.c_float_p), _p(out["desc"], T.c_uint8_p),
            _p(out["src_idx"], T.c_int32_p), _p(out["counts"], T.c_int32_p)))
        return total, out

    def orb_kernel_times(self):
        """Device ms of the last orb_compute_batch: pyramid + blur, border filter, angles + descriptors."""
        ms = np.zeros(3, np.float32)
        self._ck(self.lib.plstvo_orb_kernel_times(self.ctx, _p(ms, T.c_float_p)))
        return ms

    def orb_detect_and_compute_batch(self, cfg: T.PlOrbDetectConfig, images, fast_th=None, capacity: Optional[int] = None):
        """ORB::detectAndCompute on each of images uint8[n, H, W] (empty mask).  fast_th: per-image FAST thresholds, or None
        for cfg.fast_threshold.  Returns (total, dict(off [n + 1], xy [total, 2], octave, angle, response, desc [total, 32]));
        image i's key points are rows off[i] .. off[i + 1], ordered by level, then y, then x on the level.  Without a
        capacity the call sizes its buffers from the feature budget and, if more key points come out (ties), calls again
        with the exact count; with one, more than capacity raises PLSTVO_E_TOO_LARGE."""
        images = np.ascontiguousarray(images, np.uint8)
        n_img, H, W = images.shape
        th = None if fast_th is None else np.ascontiguousarray(np.broadcast_to(np.asarray(fast_th, np.int32), (n_img,)))
        cap = int(capacity) if capacity is not None else n_img * (2 * max(int(cfg.n_features), 0) + 64)
        while True:
            off = np.zeros(n_img + 1, np.int32)
            out = dict(off=off, xy=np.zeros((cap, 2), np.float32), octave=np.zeros(cap, np.int32),
                       angle=np.zeros(cap, np.float32), response=np.zeros(cap, np.float32), desc=np.zeros((cap, 32), np.uint8))
            rc = self.lib.plstvo_orb_detect_and_compute_batch(
                self.ctx, C.byref(cfg), n_img, W, H, _p(images, T.c_uint8_p), _p(th, T.c_int32_p), cap,
                _p(off, T.c_int32_p), _p(out["xy"], T.c_float_p), _p(out["octave"], T.c_int32_p), _p(out["angle"], T.c_float_p),
                _p(out["response"], T.c_float_p), _p(out["desc"], T.c_uint8_p))
            if rc == -2 and capacity is None and off[-1] > cap and np.diff(off).max() <= 65535:
                cap = int(off[-1])
                continue
            total = self._ck(rc)
            break
        for k in ("xy", "octave", "angle", "response", "desc"):
            out[k] = out[k][:total]
        return total, out

    def orb_detect_kernel_times(self):
        """Device ms of the last orb_detect_and_compute_batch: pyramid + blur, FAST + NMS, selection (with Harris),
        angles + descriptors."""
        ms = np.zeros(4, np.float32)
        self._ck(self.lib.plstvo_orb_detect_kernel_times(self.ctx, _p(ms, T.c_float_p)))
        return ms

    def lbd_compute_batch(self, images, kl_off, kl_seg, kl_angle, kl_npix):
        """LBD descriptors (BinaryDescriptor::compute, default Params) of octave-0 key lines on images uint8[n, H, W].  Image
        i's lines are rows kl_off[i] .. kl_off[i + 1] of kl_seg ([m, 4] float sPointInOctaveX, sPointInOctaveY,
        ePointInOctaveX, ePointInOctaveY), kl_angle ([m] radians) and kl_npix ([m] numOfPixels).  Returns desc uint8[m, 32],
        row i being line i's descriptor."""
        images = np.ascontiguousarray(images, np.uint8)
        n_img, H, W = images.shape
        kl_off = np.ascontiguousarray(kl_off, np.int32)
        kl_seg = np.ascontiguousarray(kl_seg, np.float32).reshape(-1, 4)
        kl_angle, kl_npix = np.ascontiguousarray(kl_angle, np.float32), np.ascontiguousarray(kl_npix, np.int32)
        desc = np.zeros((len(kl_seg), 32), np.uint8)
        self._ck(self.lib.plstvo_lbd_compute_batch(
            self.ctx, n_img, W, H, _p(images, T.c_uint8_p), _p(kl_off, T.c_int32_p), _p(kl_seg, T.c_float_p),
            _p(kl_angle, T.c_float_p), _p(kl_npix, T.c_int32_p), _p(desc, T.c_uint8_p)))
        return desc

    def lbd_kernel_times(self):
        """Device ms of the last lbd_compute_batch: blur + Sobel, descriptors."""
        ms = np.zeros(2, np.float32)
        self._ck(self.lib.plstvo_lbd_kernel_times(self.ctx, _p(ms, T.c_float_p)))
        return ms

    def lsd_detect_batch(self, cfg: T.PlLsdConfig, images, capacity: Optional[int] = None):
        """detectLineFeatures' LSD key lines of each of images uint8[n, H, W].  Returns (total, dict(off [n + 1], seg [total, 4]
        sPointInOctave / ePointInOctave, angle, npix, response, length)); image i's lines are rows off[i] .. off[i + 1], in
        the reference's order.  Without a capacity the call sizes its buffers from n_features (or calls again with the exact
        count); with one, more than capacity raises PLSTVO_E_TOO_LARGE."""
        images = np.ascontiguousarray(images, np.uint8)
        n_img, H, W = images.shape
        cap = int(capacity) if capacity is not None else n_img * (max(int(cfg.n_features), 0) or 1024)
        while True:
            off = np.zeros(n_img + 1, np.int32)
            out = dict(off=off, seg=np.zeros((cap, 4), np.float32), angle=np.zeros(cap, np.float32),
                       npix=np.zeros(cap, np.int32), response=np.zeros(cap, np.float32), length=np.zeros(cap, np.float32))
            rc = self.lib.plstvo_lsd_detect_batch(
                self.ctx, C.byref(cfg), n_img, W, H, _p(images, T.c_uint8_p), cap, _p(off, T.c_int32_p),
                _p(out["seg"], T.c_float_p), _p(out["angle"], T.c_float_p), _p(out["npix"], T.c_int32_p),
                _p(out["response"], T.c_float_p), _p(out["length"], T.c_float_p))
            if rc == -2 and capacity is None and off[-1] > cap and np.diff(off).max() <= 65535:
                cap = int(off[-1])
                continue
            total = self._ck(rc)
            break
        for k in ("seg", "angle", "npix", "response", "length"):
            out[k] = out[k][:total]
        return total, out

    def fld_key_lines(self, width: int, height: int, n_features: int, seg):
        """Module-level fld_key_lines on this engine's library."""
        return fld_key_lines(width, height, n_features, seg, self.lib)

    def lsd_kernel_times(self):
        """Device ms of the last lsd_detect_batch: blur + resize, gradient + seed order, region growing, the host's region
        angles (with its round trip), rectangles."""
        ms = np.zeros(5, np.float32)
        self._ck(self.lib.plstvo_lsd_kernel_times(self.ctx, _p(ms, T.c_float_p)))
        return ms

    def stereo_lift_lines(self, cam, scfg: T.PlStereoConfig, l_off, seg_l, angle_l, octave_l, desc_l, r_off, seg_r, m12):
        """Stereo matches -> LineFeature records (src/stereoFrame.cpp:348-397), batched over frames."""
        l_off, r_off = np.ascontiguousarray(l_off, np.int32), np.ascontiguousarray(r_off, np.int32)
        seg_l, seg_r = np.ascontiguousarray(seg_l, np.float32).reshape(-1, 4), np.ascontiguousarray(seg_r, np.float32).reshape(-1, 4)
        angle_l = np.ascontiguousarray(angle_l, np.float32)
        octave_l, m12 = np.ascontiguousarray(octave_l, np.int32), np.ascontiguousarray(m12, np.int32)
        desc_l = np.ascontiguousarray(desc_l, np.uint8).reshape(-1, 32)
        B, n = len(l_off) - 1, len(seg_l)
        out = self.stereo_outputs(n, B, lines=True)
        del out["m12"]
        total = self._ck(self.lib.plstvo_stereo_lift_lines(
            self.ctx, C.byref(cam), C.byref(scfg), B, _p(l_off, T.c_int32_p), _p(seg_l, T.c_float_p), _p(angle_l, T.c_float_p),
            _p(octave_l, T.c_int32_p), _p(desc_l, T.c_uint8_p), _p(r_off, T.c_int32_p), _p(seg_r, T.c_float_p),
            _p(m12, T.c_int32_p), *_record_ptrs(out, T.FRAME_OUT_LINE_RECORDS), _p(out["counts"], T.c_int32_p)))
        return total, out

    def match_stereo_points(self, cam, mcfg: T.PlStereoMatchConfig, scfg: T.PlStereoConfig, l_off, kp_l, octave_l, desc_l,
                            r_off, kp_r, desc_r, out=None):
        """StereoFrame::matchStereoPoints (src/stereoFrame.cpp:120-173): grid cells, matchGrid and the lifting in one device
        pass.  Returns (total, out) like stereo_lift_points, plus out["m12"]."""
        l_off, r_off = np.ascontiguousarray(l_off, np.int32), np.ascontiguousarray(r_off, np.int32)
        kp_l, kp_r = np.ascontiguousarray(kp_l, np.float32).reshape(-1, 2), np.ascontiguousarray(kp_r, np.float32).reshape(-1, 2)
        octave_l = np.ascontiguousarray(octave_l, np.int32)
        desc_l, desc_r = np.ascontiguousarray(desc_l, np.uint8).reshape(-1, 32), np.ascontiguousarray(desc_r, np.uint8).reshape(-1, 32)
        B, n = len(l_off) - 1, len(kp_l)
        if out is None:
            out = self.stereo_outputs(n, B, lines=False)
        total = self._ck(self.lib.plstvo_match_stereo_points(
            self.ctx, C.byref(cam), C.byref(mcfg), C.byref(scfg), B, _p(l_off, T.c_int32_p), _p(kp_l, T.c_float_p),
            _p(octave_l, T.c_int32_p), _p(desc_l, T.c_uint8_p), _p(r_off, T.c_int32_p), _p(kp_r, T.c_float_p),
            _p(desc_r, T.c_uint8_p), _p(out["m12"], T.c_int32_p), *_record_ptrs(out, T.FRAME_OUT_POINT_RECORDS),
            _p(out["counts"], T.c_int32_p)))
        return total, out

    def stereo_outputs(self, n: int, B: int, lines: bool, pinned: bool = False) -> dict:
        """Output arrays of match_stereo_points / _lines for n left features in B frames (pinned=True: cudaMallocHost)."""
        mk = (lambda shape, dt: self.pinned.empty(shape, dt)) if pinned else (lambda shape, dt: np.zeros(shape, dt))
        out = dict(m12=mk((n,), np.int32))
        for r in T.FRAME_OUT_LINE_RECORDS if lines else T.FRAME_OUT_POINT_RECORDS:
            out[r.key] = mk((n,) + r.row, r.dtype)
        out["counts"] = mk((B,), np.int32)
        out["m12"][...] = -1
        out["src_idx"][...] = -1
        return out

    def match_stereo_lines(self, cam, mcfg: T.PlStereoMatchConfig, scfg: T.PlStereoConfig, l_off, seg_l, angle_l, octave_l,
                           desc_l, r_off, seg_r, desc_r, out=None):
        """StereoFrame::matchStereoLines (src/stereoFrame.cpp:309-398) in one device pass."""
        l_off, r_off = np.ascontiguousarray(l_off, np.int32), np.ascontiguousarray(r_off, np.int32)
        seg_l, seg_r = np.ascontiguousarray(seg_l, np.float32).reshape(-1, 4), np.ascontiguousarray(seg_r, np.float32).reshape(-1, 4)
        angle_l, octave_l = np.ascontiguousarray(angle_l, np.float32), np.ascontiguousarray(octave_l, np.int32)
        desc_l, desc_r = np.ascontiguousarray(desc_l, np.uint8).reshape(-1, 32), np.ascontiguousarray(desc_r, np.uint8).reshape(-1, 32)
        B, n = len(l_off) - 1, len(seg_l)
        if out is None:
            out = self.stereo_outputs(n, B, lines=True)
        total = self._ck(self.lib.plstvo_match_stereo_lines(
            self.ctx, C.byref(cam), C.byref(mcfg), C.byref(scfg), B, _p(l_off, T.c_int32_p), _p(seg_l, T.c_float_p),
            _p(angle_l, T.c_float_p), _p(octave_l, T.c_int32_p), _p(desc_l, T.c_uint8_p), _p(r_off, T.c_int32_p),
            _p(seg_r, T.c_float_p), _p(desc_r, T.c_uint8_p), _p(out["m12"], T.c_int32_p),
            *_record_ptrs(out, T.FRAME_OUT_LINE_RECORDS), _p(out["counts"], T.c_int32_p)))
        return total, out

    def _track_stereo(self, fn, cam, cfg, mcfg, scfg, more, frame_sets, as_c, priors, results):
        """One blocking track_stereo_* call: fn(ctx, cam, cfg, mcfg, scfg, *more, one struct per frame set, priors, results,
        n_stereo).  frame_sets: (prev, curr) of B pairs, giving results [B] and n_stereo [B, 4], or (frames,) of NF
        consecutive frames, giving results [NF - 1] and n_stereo [NF, 2]; as_c makes each set's struct and keep-alive arrays."""
        structs = [as_c(f) for f in frame_sets]
        B, pairs = structs[0][0].B, len(frame_sets) == 2
        if results is None:
            results = np.zeros(B if pairs else max(B - 1, 0), dtype=T.POSE_RESULT_DTYPE)
        n_stereo = np.zeros((B, 4 if pairs else 2), np.int32)
        self._ck(fn(self.ctx, C.byref(cam), C.byref(cfg), C.byref(mcfg), C.byref(scfg), *more,
                    *(C.byref(s) for s, _ in structs), priors.ctypes.data if priors is not None else None, results.ctypes.data,
                    _p(n_stereo, T.c_int32_p)))
        return results, n_stereo

    def track_stereo_batch(self, cam, cfg, mcfg, scfg, prev: dict, curr: dict, priors=None, results=None):
        """Raw stereo features of B (prev, curr) frame pairs -> poses: matchStereoPoints / Lines for both frames, f2fTracking and
        optimizePose, the lifted records resident in HBM.  prev / curr: dicts with the PlStereoFeatures fields.
        Returns (results, n_stereo[B, 4])."""
        return self._track_stereo(self.lib.plstvo_track_stereo_batch, cam, cfg, mcfg, scfg, (), (prev, curr),
                                  T.stereo_features_as_c, priors, results)

    def track_stereo_batch_async(self, cam, cfg, mcfg, scfg, prev_c, curr_c, results, n_stereo, priors=None) -> int:
        """Streaming form: prev_c / curr_c are PlStereoFeatures structs built once by T.stereo_features_as_c over PINNED arrays
        (keep the returned keep-alive dicts); results / n_stereo are caller-owned (pinned) arrays, valid after wait(ticket)."""
        return self._ck(self.lib.plstvo_track_stereo_batch_async(
            self.ctx, C.byref(cam), C.byref(cfg), C.byref(mcfg), C.byref(scfg), C.byref(prev_c), C.byref(curr_c),
            priors.ctypes.data if priors is not None else None, results.ctypes.data, _p(n_stereo, T.c_int32_p)))

    def track_stereo_sequence_async(self, cam, cfg, mcfg, scfg, frames_c, results, n_stereo, priors=None) -> int:
        return self._ck(self.lib.plstvo_track_stereo_sequence_async(
            self.ctx, C.byref(cam), C.byref(cfg), C.byref(mcfg), C.byref(scfg), C.byref(frames_c),
            priors.ctypes.data if priors is not None else None, results.ctypes.data, _p(n_stereo, T.c_int32_p)))

    def track_stereo_sequence(self, cam, cfg, mcfg, scfg, frames: dict, priors=None, results=None):
        """NF consecutive frames of raw stereo features -> NF - 1 poses (pair p = frames p, p + 1); every frame goes through the
        stereo step once.  Returns (results, n_stereo[NF, 2])."""
        return self._track_stereo(self.lib.plstvo_track_stereo_sequence, cam, cfg, mcfg, scfg, (), (frames,),
                                  T.stereo_features_as_c, priors, results)

    def track_stereo_images_batch(self, cam, cfg, mcfg, scfg, ocfg, prev: dict, curr: dict, priors=None, results=None):
        """Stereo images and key lines of B (prev, curr) frame pairs -> poses: ORB detection, LBD description, the stereo step,
        f2fTracking and optimizePose, feature data resident in HBM.  prev / curr: dicts with img_l / img_r uint8[B, H, W] and
        the other PlStereoImages fields (see T.stereo_images_as_c).  Returns (results, n_stereo[B, 4])."""
        return self._track_stereo(self.lib.plstvo_track_stereo_images_batch, cam, cfg, mcfg, scfg, (C.byref(ocfg),),
                                  (prev, curr), T.stereo_images_as_c, priors, results)

    def track_stereo_images_sequence(self, cam, cfg, mcfg, scfg, ocfg, frames: dict, priors=None, results=None):
        """NF consecutive stereo frames (images and key lines) -> NF - 1 poses; every frame's images are detected and described
        once.  Returns (results, n_stereo[NF, 2])."""
        return self._track_stereo(self.lib.plstvo_track_stereo_images_sequence, cam, cfg, mcfg, scfg, (C.byref(ocfg),),
                                  (frames,), T.stereo_images_as_c, priors, results)

    def track_stereo_images_lsd_batch(self, cam, cfg, mcfg, scfg, ocfg, lcfg, prev: dict, curr: dict, priors=None, results=None):
        """Stereo images alone of B (prev, curr) frame pairs -> poses: LSD detection inside the call, then what
        track_stereo_images_batch does.  prev / curr: dicts with img_l / img_r uint8[B, H, W] and optionally fast_th [B], no
        key-line arrays.  lcfg may be None where cfg.has_lines is 0.  Returns (results, n_stereo[B, 4])."""
        return self._track_stereo(self.lib.plstvo_track_stereo_images_lsd_batch, cam, cfg, mcfg, scfg,
                                  (C.byref(ocfg), None if lcfg is None else C.byref(lcfg)), (prev, curr), T.stereo_images_as_c,
                                  priors, results)

    def track_stereo_images_lsd_sequence(self, cam, cfg, mcfg, scfg, ocfg, lcfg, frames: dict, priors=None, results=None):
        """NF consecutive stereo frames (images alone) -> NF - 1 poses, LSD inside the call; every frame's images are detected
        and described once.  Returns (results, n_stereo[NF, 2])."""
        return self._track_stereo(self.lib.plstvo_track_stereo_images_lsd_sequence, cam, cfg, mcfg, scfg,
                                  (C.byref(ocfg), None if lcfg is None else C.byref(lcfg)), (frames,), T.stereo_images_as_c,
                                  priors, results)

    # ---- rectification: PinholeStereoCamera::rectifyImagesLR ----
    def rectifier_create(self, map1_l, map2_l, map1_r=None, map2_r=None) -> Rectifier:
        """Uploads a rig's CV_16SC2 map pairs once (map1 int16[h, w, 2], map2 uint16[h, w]); the right pair defaults to the
        left one, which is then held once (the reference's cam_d0 branch)."""
        m1l = np.ascontiguousarray(map1_l, np.int16)
        m2l = np.ascontiguousarray(map2_l, np.uint16)
        m1r = m1l if map1_r is None else np.ascontiguousarray(map1_r, np.int16)
        m2r = m2l if map2_r is None else np.ascontiguousarray(map2_r, np.uint16)
        H, W = m2l.shape
        if m1l.shape != (H, W, 2) or m1r.shape != (H, W, 2) or m2r.shape != (H, W):
            raise ValueError("map shapes differ")
        i16p, u16p = C.POINTER(C.c_int16), C.POINTER(C.c_uint16)
        h = self.lib.plstvo_rectifier_create(self.ctx, W, H, _p(m1l, i16p), _p(m2l, u16p), _p(m1r, i16p), _p(m2r, u16p))
        if not h:
            raise PlstvoError(-1, (self.lib.plstvo_last_error(self.ctx) or b"").decode())
        r = Rectifier(self.lib, h, W, H)
        self._rectifiers.append(r)
        return r

    def rectifier_create_color(self, width: int, height: int, channels: int, map1_l=None, map2_l=None, map1_r=None,
                               map2_r=None) -> Rectifier:
        """A rectifier of colour images (channels 3: BGR, 4: BGRA): cvtColor(remap(img), COLOR_BGR2GRAY) with the maps, the
        conversion alone without them.  The right pair defaults to the left one (held once); no maps at all is the map-less
        form."""
        i16p, u16p = C.POINTER(C.c_int16), C.POINTER(C.c_uint16)
        m1l = None if map1_l is None else np.ascontiguousarray(map1_l, np.int16)
        m2l = None if map2_l is None else np.ascontiguousarray(map2_l, np.uint16)
        m1r = m1l if map1_r is None else np.ascontiguousarray(map1_r, np.int16)
        m2r = m2l if map2_r is None else np.ascontiguousarray(map2_r, np.uint16)
        for m, shape in ((m1l, (height, width, 2)), (m2l, (height, width)), (m1r, (height, width, 2)), (m2r, (height, width))):
            if m is not None and m.shape != shape:
                raise ValueError("map shapes differ from the size")
        h = self.lib.plstvo_rectifier_create_color(self.ctx, width, height, channels, _p(m1l, i16p), _p(m2l, u16p),
                                                   _p(m1r, i16p), _p(m2r, u16p))
        if not h:
            raise PlstvoError(-1, (self.lib.plstvo_last_error(self.ctx) or b"").decode())
        r = Rectifier(self.lib, h, width, height, channels)
        self._rectifiers.append(r)
        return r

    def rectifier_destroy(self, rect: Rectifier):
        rect.close()
        self._rectifiers = [r for r in self._rectifiers if r is not rect]

    def rectify_batch(self, rect: Rectifier, img_l, img_r):
        """rectifyImagesLR on B pairs: (rectified left uint8[B, H, W], rectified right).  A colour rectifier takes
        uint8[B, H, W, C] and returns the grey images the reference's detectors see."""
        il = np.ascontiguousarray(img_l, np.uint8)
        ir = np.ascontiguousarray(img_r, np.uint8)
        if il.ndim == len(rect.image_shape(0)) - 1:
            il, ir = il[None], ir[None]
        if il.shape != ir.shape or il.shape != rect.image_shape(il.shape[0]):
            if rect.channels > 1:
                raise ValueError("images must be uint8[B, H, W, C] of the rectifier's size and channels, both sides alike")
            raise ValueError("images must be uint8[B, H, W] of the rectifier's size, both sides alike")
        ol, orr = np.empty(il.shape[:3], np.uint8), np.empty(ir.shape[:3], np.uint8)
        self._ck(self.lib.plstvo_rectify_batch(self.ctx, rect.handle, il.shape[0], _p(il, T.c_uint8_p), _p(ir, T.c_uint8_p),
                                               _p(ol, T.c_uint8_p), _p(orr, T.c_uint8_p)))
        return ol, orr

    def rectify_kernel_times(self) -> float:
        """Device ms of the last remap (rectify_batch or a raw-images call)."""
        ms = np.zeros(1, np.float32)
        self._ck(self.lib.plstvo_rectify_kernel_times(self.ctx, _p(ms, T.c_float_p)))
        return float(ms[0])

    def track_stereo_raw_images_batch(self, cam, cfg, mcfg, scfg, ocfg, lcfg, rect: Optional[Rectifier], prev: dict, curr: dict,
                                      priors=None, results=None):
        """track_stereo_images_lsd_batch on raw (distorted) images: rect's remap runs on the device first; rect None: the
        _lsd_ call.  A colour rectifier takes img_l / img_r uint8[B, H, W, C].  Returns (results, n_stereo[B, 4])."""
        if rect is not None and rect.channels > 1:
            rect.check_frames(prev, curr)
        return self._track_stereo(self.lib.plstvo_track_stereo_raw_images_batch, cam, cfg, mcfg, scfg,
                                  (C.byref(ocfg), None if lcfg is None else C.byref(lcfg), None if rect is None else rect.handle),
                                  (prev, curr), T.stereo_images_as_c, priors, results)

    def track_stereo_raw_images_sequence(self, cam, cfg, mcfg, scfg, ocfg, lcfg, rect: Optional[Rectifier], frames: dict,
                                         priors=None, results=None):
        """track_stereo_images_lsd_sequence on raw images, rectified on the device (colour ones converted to grey there).
        Returns (results, n_stereo[NF, 2])."""
        if rect is not None and rect.channels > 1:
            rect.check_frames(frames)
        return self._track_stereo(self.lib.plstvo_track_stereo_raw_images_sequence, cam, cfg, mcfg, scfg,
                                  (C.byref(ocfg), None if lcfg is None else C.byref(lcfg), None if rect is None else rect.handle),
                                  (frames,), T.stereo_images_as_c, priors, results)

    # ---- stereo sessions: many streams, each stream's previous frame kept on the device ----
    def stereo_session_create(self, cam, cfg, mcfg, scfg, ocfg, lcfg, rect: Optional[Rectifier], n_streams: int) -> StereoSession:
        """A session of n_streams streams with these configs (copied; lcfg may be None where cfg.has_lines is 0) and rect
        (None: the images are already rectified; it must outlive the session).  With a colour rectifier the session takes
        colour frames, uint8[n, H, W, C]."""
        h = self.lib.plstvo_stereo_session_create(self.ctx, C.byref(cam), C.byref(cfg), C.byref(mcfg), C.byref(scfg),
                                                  C.byref(ocfg), None if lcfg is None else C.byref(lcfg),
                                                  None if rect is None else rect.handle, n_streams)
        if not h:
            raise PlstvoError(-1, (self.lib.plstvo_last_error(self.ctx) or b"").decode())
        ss = StereoSession(self, h, n_streams, rect, (cam.width, cam.height))
        self._sessions.append(ss)
        return ss

    def stereo_session_create_cams(self, cams, cfg, mcfg, scfg, ocfg, lcfg, rects, n_streams: int) -> StereoSession:
        """A session whose stream i is tracked under cams[i] (n_streams PlCamera of one image size) and prepared by rects[i]
        (rects None: no stream is remapped; in a grey session an entry None takes that stream's images as given; a colour
        session needs a colour rectifier for every stream).  The rectifiers must outlive the session."""
        cams = list(cams)
        if len(cams) != n_streams:
            raise ValueError("one camera per stream")
        carr = (T.PlCamera * max(n_streams, 1))(*cams)
        rarr = None
        first = None
        if rects is not None:
            rects = list(rects)
            if len(rects) != n_streams:
                raise ValueError("one rectifier (or None) per stream")
            rarr = (C.c_void_p * n_streams)(*[None if r is None else r.handle for r in rects])
            first = next((r for r in rects if r is not None), None)
        h = self.lib.plstvo_stereo_session_create_cams(self.ctx, carr, C.byref(cfg), C.byref(mcfg), C.byref(scfg),
                                                       C.byref(ocfg), None if lcfg is None else C.byref(lcfg), rarr, n_streams)
        if not h:
            raise PlstvoError(-1, (self.lib.plstvo_last_error(self.ctx) or b"").decode())
        ss = StereoSession(self, h, n_streams, first, (cams[0].width, cams[0].height))
        self._sessions.append(ss)
        return ss

    def stereo_session_destroy(self, ss: StereoSession):
        ss.close()
        self._sessions = [x for x in self._sessions if x is not ss]

    def stereo_session_initialize(self, ss: StereoSession, ids, frames: dict):
        ss.check_frames(frames)
        ids = np.ascontiguousarray(ids, np.int32)
        fs, keep = T.stereo_images_as_c(frames)
        n_stereo = np.zeros((len(ids), 2), np.int32)
        ss.last = None
        self._ck(self.lib.plstvo_stereo_session_initialize(self.ctx, ss.handle, len(ids), _p(ids, T.c_int32_p), C.byref(fs),
                                                           _p(n_stereo, T.c_int32_p)))
        del keep
        ss.last = (False, n_stereo.copy())
        return n_stereo

    def stereo_session_insert(self, ss: StereoSession, ids, frames: dict, priors=None, results=None):
        ss.check_frames(frames)
        ids = np.ascontiguousarray(ids, np.int32)
        fs, keep = T.stereo_images_as_c(frames)
        n = len(ids)
        if results is None:
            results = np.zeros(n, dtype=T.POSE_RESULT_DTYPE)
        n_stereo = np.zeros((n, 4), np.int32)
        ss.last = None
        self._ck(self.lib.plstvo_stereo_session_insert(self.ctx, ss.handle, n, _p(ids, T.c_int32_p), C.byref(fs),
                                                       priors.ctypes.data if priors is not None else None, results.ctypes.data,
                                                       _p(n_stereo, T.c_int32_p)))
        del keep
        ss.last = (True, n_stereo.copy())
        return results, n_stereo

    def handler_config(self, kitti: bool = False):
        """plstvo_default_handler_config / plstvo_kitti_handler_config."""
        h = T.PlHandlerConfig()
        (self.lib.plstvo_kitti_handler_config if kitti else self.lib.plstvo_default_handler_config)(C.byref(h))
        return h

    def stereo_session_run(self, ss: StereoSession, hcfg, ids, T_: int, frames: dict, fast_th0=None, priors=None):
        ss.check_frames(frames)
        h = hcfg if isinstance(hcfg, T.PlHandlerConfig) else T.handler_config(hcfg)
        ids = np.ascontiguousarray(ids, np.int32)
        fs, keep = T.stereo_images_as_c(frames)
        n = len(ids)
        th0 = None if fast_th0 is None else np.ascontiguousarray(fast_th0, np.int32).reshape(-1)
        pri = None if priors is None else np.ascontiguousarray(priors, T.PRIOR_DTYPE).reshape(-1)
        if (th0 is not None and len(th0) != n) or (pri is not None and len(pri) != n):
            raise ValueError("fast_th0 and priors take one entry per stream of ids")
        results = np.zeros((T_, n), dtype=T.POSE_RESULT_DTYPE)
        fast_th = np.zeros((T_ + 1, n), np.int32)
        n_stereo = np.zeros((T_, n, 4), np.int32)
        last, ss.last = ss.last, None
        self._ck(self.lib.plstvo_stereo_session_run(self.ctx, ss.handle, C.byref(h), n, _p(ids, T.c_int32_p), T_, C.byref(fs),
                                                    _p(th0, T.c_int32_p), None if pri is None else pri.ctypes.data,
                                                    results.ctypes.data, _p(fast_th, T.c_int32_p), _p(n_stereo, T.c_int32_p)))
        del keep
        # read() returns the last step, as if it had been an insert; T_ = 0 changes nothing
        ss.last = (True, n_stereo[-1].copy()) if T_ > 0 else last
        return results, fast_th, n_stereo

    def keyframe_config(self):
        """plstvo_default_keyframe_config: one T.KEYFRAME_CONFIG_DTYPE record."""
        k = np.zeros(1, T.KEYFRAME_CONFIG_DTYPE)
        self.lib.plstvo_default_keyframe_config(k.ctypes.data)
        return k

    def initial_keyframe_state(self, n: int = 1):
        """plstvo_initial_keyframe_state for n streams: T.KEYFRAME_STATE_DTYPE [n]."""
        s = np.zeros(n, T.KEYFRAME_STATE_DTYPE)
        for i in range(n):
            self.lib.plstvo_initial_keyframe_state(s[i:].ctypes.data)
        return s

    def stereo_session_run_keyframes(self, ss: StereoSession, hcfg, kcfg, ids, T_: int, frames: dict, kf_state, fast_th0=None,
                                     priors=None):
        ss.check_frames(frames)
        h = hcfg if isinstance(hcfg, T.PlHandlerConfig) else T.handler_config(hcfg)
        k = (np.ascontiguousarray(kcfg, T.KEYFRAME_CONFIG_DTYPE).reshape(-1) if isinstance(kcfg, np.ndarray)
             else T.keyframe_config(kcfg))
        ids = np.ascontiguousarray(ids, np.int32)
        fs, keep = T.stereo_images_as_c(frames)
        n = len(ids)
        th0 = None if fast_th0 is None else np.ascontiguousarray(fast_th0, np.int32).reshape(-1)
        pri = None if priors is None else np.ascontiguousarray(priors, T.PRIOR_DTYPE).reshape(-1)
        if not (isinstance(kf_state, np.ndarray) and kf_state.dtype == T.KEYFRAME_STATE_DTYPE and kf_state.flags.c_contiguous):
            raise ValueError("kf_state: a contiguous T.KEYFRAME_STATE_DTYPE array, updated in place")
        if (th0 is not None and len(th0) != n) or (pri is not None and len(pri) != n) or kf_state.size != n:
            raise ValueError("fast_th0, priors and kf_state take one entry per stream of ids")
        results = np.zeros((T_, n), dtype=T.POSE_RESULT_DTYPE)
        kf = np.zeros((T_, n), dtype=T.KEYFRAME_RESULT_DTYPE)
        fast_th = np.zeros((T_ + 1, n), np.int32)
        n_stereo = np.zeros((T_, n, 4), np.int32)
        last, ss.last = ss.last, None
        self._ck(self.lib.plstvo_stereo_session_run_keyframes(
            self.ctx, ss.handle, C.byref(h), k.ctypes.data, n, _p(ids, T.c_int32_p), T_, C.byref(fs), _p(th0, T.c_int32_p),
            None if pri is None else pri.ctypes.data, kf_state.ctypes.data, results.ctypes.data, kf.ctypes.data,
            _p(fast_th, T.c_int32_p), _p(n_stereo, T.c_int32_p)))
        del keep
        ss.last = (True, n_stereo[-1].copy()) if T_ > 0 else last
        return results, kf, fast_th, n_stereo

    def stereo_session_run_schedule(self, ss: StereoSession, hcfg, ids, schedule, frames: dict, fast_th0=None, priors=None,
                                    kcfg=None, kf_state=None):
        ss.check_frames(frames)
        h = hcfg if isinstance(hcfg, T.PlHandlerConfig) else T.handler_config(hcfg)
        ids = np.ascontiguousarray(ids, np.int32)
        n = len(ids)
        raw = np.asarray(schedule)
        if raw.size and (not np.issubdtype(raw.dtype, np.integer) or raw.min() < 0 or raw.max() > 255):
            raise ValueError("schedule: integers, 0 idle, 1 insert, 2 initialize (the library refuses other values)")
        sched = np.ascontiguousarray(raw, np.uint8).reshape(-1, n) if n else np.zeros((len(raw), 0), np.uint8)
        T_ = sched.shape[0]
        fs, keep = T.stereo_images_as_c(frames)
        th0 = None if fast_th0 is None else np.ascontiguousarray(fast_th0, np.int32).reshape(-1)
        pri = None if priors is None else np.ascontiguousarray(priors, T.PRIOR_DTYPE).reshape(-1)
        if (th0 is not None and len(th0) != n) or (pri is not None and len(pri) != n):
            raise ValueError("fast_th0 and priors take one entry per stream of ids")
        k = kf = None
        if kcfg is not None:
            k = (np.ascontiguousarray(kcfg, T.KEYFRAME_CONFIG_DTYPE).reshape(-1) if isinstance(kcfg, np.ndarray)
                 else T.keyframe_config(kcfg))
            if not (isinstance(kf_state, np.ndarray) and kf_state.dtype == T.KEYFRAME_STATE_DTYPE
                    and kf_state.flags.c_contiguous and kf_state.size == n):
                raise ValueError("kf_state: a contiguous T.KEYFRAME_STATE_DTYPE array of one entry per stream, updated in place")
            kf = np.zeros((T_, n), dtype=T.KEYFRAME_RESULT_DTYPE)
        elif kf_state is not None:
            raise ValueError("kf_state without a key-frame config")
        results = np.zeros((T_, n), dtype=T.POSE_RESULT_DTYPE)
        fast_th = np.zeros((T_ + 1, n), np.int32)
        n_stereo = np.zeros((T_, n, 4), np.int32)
        last, ss.last = ss.last, None
        self._ck(self.lib.plstvo_stereo_session_run_schedule(
            self.ctx, ss.handle, C.byref(h), None if k is None else k.ctypes.data, n, _p(ids, T.c_int32_p), T_,
            sched.ctypes.data_as(C.POINTER(C.c_uint8)), C.byref(fs), _p(th0, T.c_int32_p),
            None if pri is None else pri.ctypes.data, None if kf_state is None else kf_state.ctypes.data,
            results.ctypes.data, None if kf is None else kf.ctypes.data, _p(fast_th, T.c_int32_p), _p(n_stereo, T.c_int32_p)))
        del keep
        # read() returns the last step with entries as its last chain call (the insert where the step has both kinds)
        steps = np.nonzero(sched.any(axis=1))[0]
        if len(steps):
            row = sched[steps[-1]]
            ss.last = ((True, n_stereo[steps[-1]][row == 1].copy()) if (row == 1).any()
                       else (False, n_stereo[steps[-1]][row == 2][:, 2:].copy()))
        else:
            ss.last = last
        return (results, fast_th, n_stereo) if k is None else (results, kf, fast_th, n_stereo)

    def track_stereo_images_stage_times(self):
        """Device ms of the last images call: uploads, ORB, LBD (overlaps ORB; after the LSD form, the lines: LSD's first launch
        to LBD's last), stereo step, f2fTracking + optimizePose."""
        ms = np.zeros(5, np.float32)
        self._ck(self.lib.plstvo_track_stereo_images_stage_times(self.ctx, _p(ms, T.c_float_p)))
        return ms

    # ---- stereoFrameHandler.h surface ----
    def f2f_tracking(self, cfg, prev: T.FrameBatch, curr: T.FrameBatch):
        m12_pt, m12_ls = np.full(prev.n_pt, -1, np.int32), np.full(prev.n_ls, -1, np.int32)
        n = np.zeros((prev.B, 2), np.int32)
        pc, cc = prev.as_c(), curr.as_c()
        self._ck(self.lib.plstvo_f2f_tracking(self.ctx, C.byref(cfg), C.byref(pc), C.byref(cc),
                                              _p(m12_pt, T.c_int32_p), _p(m12_ls, T.c_int32_p), _p(n, T.c_int32_p)))
        return m12_pt, m12_ls, n

    def optimize_pose(self, cam, cfg, matched: T.MatchedBatch, priors=None):
        res = np.zeros(matched.B, dtype=T.POSE_RESULT_DTYPE)
        inl_pt = np.zeros(int(matched.pt_off[-1]), np.uint8)
        inl_ls = np.zeros(int(matched.ls_off[-1]), np.uint8)
        mc = matched.as_c()
        self._ck(self.lib.plstvo_optimize_pose(self.ctx, C.byref(cam), C.byref(cfg), C.byref(mc),
                                               priors.ctypes.data if priors is not None else None, res.ctypes.data,
                                               _p(inl_pt, T.c_uint8_p), _p(inl_ls, T.c_uint8_p)))
        return res, inl_pt, inl_ls

    def track_batch(self, cam, cfg, prev: T.FrameBatch, curr: T.FrameBatch, priors=None, out=None):
        """insertStereoPair's f2fTracking + optimizePose for B pairs, host buffers in / out."""
        if out is None:
            out = dict(results=np.zeros(prev.B, dtype=T.POSE_RESULT_DTYPE),
                       m12_pt=np.full(prev.n_pt, -1, np.int32), m12_ls=np.full(prev.n_ls, -1, np.int32),
                       inlier_pt=np.zeros(prev.n_pt, np.uint8), inlier_ls=np.zeros(prev.n_ls, np.uint8))
        pc, cc = prev.as_c(), curr.as_c()
        self._ck(self.lib.plstvo_track_batch(
            self.ctx, C.byref(cam), C.byref(cfg), C.byref(pc), C.byref(cc),
            priors.ctypes.data if priors is not None else None, out["results"].ctypes.data,
            _p(out["m12_pt"], T.c_int32_p), _p(out["m12_ls"], T.c_int32_p), _p(out["inlier_pt"], T.c_uint8_p),
            _p(out["inlier_ls"], T.c_uint8_p)))
        return out

    def track_batch_cams(self, cams, cfg, prev: T.FrameBatch, curr: T.FrameBatch, priors=None, out=None):
        """track_batch with pair p solved under cams[p] (B PlCamera)."""
        cams = list(cams)
        if len(cams) != prev.B:
            raise ValueError("one camera per pair")
        carr = (T.PlCamera * max(prev.B, 1))(*cams)
        if out is None:
            out = dict(results=np.zeros(prev.B, dtype=T.POSE_RESULT_DTYPE),
                       m12_pt=np.full(prev.n_pt, -1, np.int32), m12_ls=np.full(prev.n_ls, -1, np.int32),
                       inlier_pt=np.zeros(prev.n_pt, np.uint8), inlier_ls=np.zeros(prev.n_ls, np.uint8))
        pc, cc = prev.as_c(), curr.as_c()
        self._ck(self.lib.plstvo_track_batch_cams(
            self.ctx, carr, C.byref(cfg), C.byref(pc), C.byref(cc),
            priors.ctypes.data if priors is not None else None, out["results"].ctypes.data,
            _p(out["m12_pt"], T.c_int32_p), _p(out["m12_ls"], T.c_int32_p), _p(out["inlier_pt"], T.c_uint8_p),
            _p(out["inlier_ls"], T.c_uint8_p)))
        return out

    def track_batch_async(self, cam, cfg, prev: T.FrameBatch, curr: T.FrameBatch, out, priors=None) -> int:
        """Streaming form: returns a ticket; `prev`, `curr`, `priors` and `out` must stay alive and untouched until
        wait(ticket).  Use pinned arrays (self.pinned) so that the copies really are asynchronous."""
        pc, cc = prev.as_c(), curr.as_c()
        self._keep = getattr(self, "_keep", {})
        t = self._ck(self.lib.plstvo_track_batch_async(
            self.ctx, C.byref(cam), C.byref(cfg), C.byref(pc), C.byref(cc),
            priors.ctypes.data if priors is not None else None, out["results"].ctypes.data,
            _p(out["m12_pt"], T.c_int32_p), _p(out["m12_ls"], T.c_int32_p), _p(out["inlier_pt"], T.c_uint8_p),
            _p(out["inlier_ls"], T.c_uint8_p)))
        self._keep[t] = (prev, curr, priors, out)
        return t

    def wait(self, ticket: int):
        self._ck(self.lib.plstvo_wait(self.ctx, ticket))
        getattr(self, "_keep", {}).pop(ticket, None)

    def pinned_outputs(self, prev: T.FrameBatch):
        e = self.pinned.empty
        return dict(results=e((prev.B,), T.POSE_RESULT_DTYPE), m12_pt=e((prev.n_pt,), np.int32),
                    m12_ls=e((prev.n_ls,), np.int32), inlier_pt=e((prev.n_pt,), np.uint8),
                    inlier_ls=e((prev.n_ls,), np.uint8))

    def upload(self, cam, cfg, prev: T.FrameBatch, curr: T.FrameBatch, priors=None) -> DeviceBatch:
        h = C.c_void_p()
        pc, cc = prev.as_c(), curr.as_c()
        self._ck(self.lib.plstvo_batch_upload(self.ctx, C.byref(cam), C.byref(cfg), C.byref(pc), C.byref(cc),
                                              priors.ctypes.data if priors is not None else None, C.byref(h)))
        return DeviceBatch(self, h, prev)

    def gn_eval_stream(self, cam, cfg, matched: T.MatchedBatch, DT, iters: int = 1):
        """optimizeFunctions for B problems streamed from HBM (C5 roofline kernel); returns H, g, e, ms_total."""
        B = matched.B
        DT = np.ascontiguousarray(DT, np.float64).reshape(B, 16)
        H, g, e = np.zeros((B, 6, 6)), np.zeros((B, 6)), np.zeros(B)
        ms = C.c_float(0)
        mc = matched.as_c()
        self._ck(self.lib.plstvo_gn_eval_stream(self.ctx, C.byref(cam), C.byref(cfg), C.byref(mc), _p(DT, T.c_double_p),
                                                iters, _p(H, T.c_double_p), _p(g, T.c_double_p), _p(e, T.c_double_p),
                                                C.byref(ms)))
        return H, g, e, float(ms.value)

    def debug_select(self, lists, ks, pivots=None):
        """Block-wide radix selection (test hook): the ks[p]-th smallest of lists[p]; with pivots, of |x - pivot| rounded to float."""
        off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)
        v = np.ascontiguousarray(np.concatenate([np.asarray(x, np.float64) for x in lists]) if len(lists) else np.zeros(0))
        ks = np.ascontiguousarray(ks, np.int32)
        out = np.zeros(len(lists))
        pv = None if pivots is None else np.ascontiguousarray(pivots, np.float64)
        self._ck(self.lib.plstvo_debug_select(self.ctx, len(lists), _p(off, T.c_int32_p), _p(v, T.c_double_p), _p(ks, T.c_int32_p),
                                              _p(pv, T.c_double_p) if pv is not None else None, 0 if pv is None else 1,
                                              _p(out, T.c_double_p)))
        return out

    def debug_tc_partials(self, d1, off1, d2, off2, nnr):
        """Tensor-core matcher's intermediate words (test hook) for a match_batch problem set: rowp (per problem
        [ceil(n2 / 256)][n1], flattened), colp [sum n2], rowkey [sum n1, 2], colkey [sum n2, 2], all uint32."""
        d1, d2 = np.ascontiguousarray(d1, np.uint8).reshape(-1, 32), np.ascontiguousarray(d2, np.uint8).reshape(-1, 32)
        off1, off2 = np.ascontiguousarray(off1, np.int32), np.ascontiguousarray(off2, np.int32)
        B = len(off1) - 1
        n1, n2 = np.diff(off1).astype(np.int64), np.diff(off2).astype(np.int64)
        u32p = C.POINTER(C.c_uint32)
        rowp = np.zeros(int(((n2 + 255) // 256 * n1).sum()), np.uint32)
        colp = np.zeros(len(d2), np.uint32)
        rowkey, colkey = np.zeros((len(d1), 2), np.uint32), np.zeros((len(d2), 2), np.uint32)
        self._ck(self.lib.plstvo_debug_tc_partials(self.ctx, B, _p(d1, T.c_uint8_p), _p(off1, T.c_int32_p), _p(d2, T.c_uint8_p),
                                                   _p(off2, T.c_int32_p), C.c_float(nnr), _p(rowp, u32p), _p(colp, u32p),
                                                   _p(rowkey, u32p), _p(colkey, u32p)))
        return rowp, colp, rowkey, colkey

    def debug_color_planes(self, rect: Rectifier, img_l, img_r, rects=None):
        """Both grey planes of a colour FLD session's preparation (test hook) on B pairs uint8[B, H, W, C] of the colour
        rectifier rect; rects (None, or one Rectifier or None per pair): pair b prepared by rects[b], None converting only.
        Returns (grey, rgb), each uint8[2, B, H, W] (left images, then right): COLOR_BGR2GRAY and COLOR_RGB2GRAY of each
        remapped image."""
        il = np.ascontiguousarray(img_l, np.uint8)
        ir = np.ascontiguousarray(img_r, np.uint8)
        B = il.shape[0] if il.ndim else 0
        if il.shape != ir.shape or il.shape != rect.image_shape(B):
            raise ValueError("images must be uint8[B, H, W, C] of the rectifier's size and channels, both sides alike")
        H, W = rect.height, rect.width
        rarr = None
        if rects is not None:
            if len(rects) != B:
                raise ValueError("one rectifier (or None) per pair")
            rarr = (C.c_void_p * max(B, 1))(*[None if r is None else r.handle for r in rects])
        grey, rgb = np.zeros((2, B, H, W), np.uint8), np.zeros((2, B, H, W), np.uint8)
        self._ck(self.lib.plstvo_debug_color_planes(self.ctx, rect.handle, rarr, B, _p(il, T.c_uint8_p), _p(ir, T.c_uint8_p),
                                                    _p(grey, T.c_uint8_p), _p(rgb, T.c_uint8_p)))
        return grey, rgb

    def debug_algebra(self, H, g):
        """On-chip 6x6 routines (test hook): returns x = H^-1 g (col-pivot QR), log|det H|, inv(H), eigvals(H)."""
        H = np.ascontiguousarray(H, np.float64).reshape(-1, 36)
        g = np.ascontiguousarray(g, np.float64).reshape(-1, 6)
        n = len(H)
        x, lad, inv, eig = np.zeros((n, 6)), np.zeros(n), np.zeros((n, 36)), np.zeros((n, 6))
        self._ck(self.lib.plstvo_debug_algebra(self.ctx, n, _p(H, T.c_double_p), _p(g, T.c_double_p), _p(x, T.c_double_p),
                                               _p(lad, T.c_double_p), _p(inv, T.c_double_p), _p(eig, T.c_double_p)))
        return x, lad, inv.reshape(n, 6, 6), eig

    # plstvo_debug_pose_helpers' record layouts (include/plstvo.h, PLSTVO_PH_*): name -> (offset, shape)
    PH_IN = {"H": (0, (6, 6)), "g": (36, (6,)), "cov": (42, (6, 6)), "DT": (78, (4, 4)), "err": (94, ()),
             "Tfw_prev": (95, (4, 4)), "Tfw_cov_prev": (111, (6, 6)), "xi": (147, (6,)), "T": (153, (4, 4))}
    PH_IN_SIZE = 169
    PH_OUT = {"chol_x": (0, (6,)), "chol_lad": (6, ()), "chol_ok": (7, ()), "chol0_x": (8, (6,)), "chol0_ok": (14, ()),
              "regs_x": (15, (6,)), "regs_ok": (21, ()), "qr_x": (22, (6,)), "qr_lad": (28, ()), "surely": (29, ()),
              "good_fast": (30, ()), "good_full": (31, ()), "eig": (32, (6,)), "inv": (38, (4, 4)), "log": (54, (6,)),
              "exp": (60, (4, 4)), "fin_good": (76, ()), "fin_err": (77, ()), "fin_DT": (78, (4, 4)), "fin_Tfw": (94, (4, 4)),
              "fin_Tfw_cov": (110, (6, 6)), "fin_eig": (146, (6,))}
    PH_OUT_SIZE = 152

    def debug_pose_helpers(self, **inputs):
        """The pose solvers' decision and finishing helpers (test hook), one case per row of the inputs: keyword arrays named as
        in PH_IN with a leading case axis (missing ones are zero; Tfw_prev and T default to the identity).  Returns a dict of
        the PH_OUT quantities with the same leading axis; flags as bool."""
        n = len(next(iter(inputs.values())))
        rec = np.zeros((n, self.PH_IN_SIZE))
        for name in ("Tfw_prev", "T"):
            rec[:, self.PH_IN[name][0]:self.PH_IN[name][0] + 16] = np.eye(4).ravel()
        for name, a in inputs.items():
            off, shape = self.PH_IN[name]
            size = int(np.prod(shape, dtype=np.int64))
            rec[:, off:off + size] = np.asarray(a, np.float64).reshape(n, size)
        out = np.zeros((n, self.PH_OUT_SIZE))
        self._ck(self.lib.plstvo_debug_pose_helpers(self.ctx, n, _p(rec, T.c_double_p), _p(out, T.c_double_p)))
        res = {}
        for name, (off, shape) in self.PH_OUT.items():
            size = int(np.prod(shape, dtype=np.int64))
            v = out[:, off:off + size].reshape((n,) + shape)
            res[name] = v.astype(bool) if name in ("chol_ok", "chol0_ok", "regs_ok", "surely", "good_fast", "good_full",
                                                   "fin_good") else v
        return res

    def debug_keyframe(self, kcfg, results, state, priors=None):
        """One launch of the session run's key-frame test (test hook) on n placed streams: kcfg one T.KEYFRAME_CONFIG_DTYPE
        record (not checked), results [n] of T.POSE_RESULT_DTYPE (Tfw, DT and DT_cov read), state [n] of
        T.KEYFRAME_STATE_DTYPE updated in place, priors None or [n] of T.PRIOR_DTYPE updated in place (a stream that fires
        takes Tfw = I, Tfw_cov = I).  Returns the [n] T.KEYFRAME_RESULT_DTYPE rows."""
        k = np.ascontiguousarray(kcfg, T.KEYFRAME_CONFIG_DTYPE).reshape(-1)
        res = np.ascontiguousarray(results, T.POSE_RESULT_DTYPE).reshape(-1)
        n = len(res)
        for name, a, dt in (("state", state, T.KEYFRAME_STATE_DTYPE), ("priors", priors, T.PRIOR_DTYPE)):
            if a is not None and not (isinstance(a, np.ndarray) and a.dtype == dt and a.flags.c_contiguous and a.size == n):
                raise ValueError(f"{name}: a contiguous array of {n} {dt} records, updated in place")
        if state is None:
            raise ValueError("state: one T.KEYFRAME_STATE_DTYPE record per stream")
        out = np.zeros(n, T.KEYFRAME_RESULT_DTYPE)
        self._ck(self.lib.plstvo_debug_keyframe(self.ctx, k.ctypes.data, n, res.ctypes.data, state.ctypes.data, out.ctypes.data,
                                                None if priors is None else priors.ctypes.data))
        return out

    def synchronize(self):
        self._ck(self.lib.plstvo_synchronize(self.ctx))

    def popc_rate(self) -> float:
        r = np.zeros(1)
        self._ck(self.lib.plstvo_popc_rate(self.ctx, r.ctypes.data_as(T.c_double_p)))
        return float(r[0])
