"""ctypes mirror of include/plstvo.h plus numpy-backed containers.

The containers keep the numpy arrays alive for as long as the C struct built from them is in use.
Field names follow the reference's classes (PointFeature / LineFeature, include/stereoFeatures.h:30-121;
StereoFrame::pdesc_l / ldesc_l, include/stereoFrame.h:59-115).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import NamedTuple, Optional, Sequence

import numpy as np

DESC_BYTES = 32
MAX_FEATURES = 65535

c_double_p = C.POINTER(C.c_double)
c_float_p = C.POINTER(C.c_float)
c_int32_p = C.POINTER(C.c_int32)
c_uint8_p = C.POINTER(C.c_uint8)


class PlCamera(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("b", C.c_double), ("width", C.c_int32), ("height", C.c_int32)]


class PlConfig(C.Structure):
    _fields_ = [("has_points", C.c_int32), ("has_lines", C.c_int32), ("best_lr_matches", C.c_int32),
                ("use_motion_model", C.c_int32), ("min_features", C.c_int32), ("max_iters", C.c_int32),
                ("max_iters_ref", C.c_int32), ("solver_mode", C.c_int32),
                ("min_ratio_12_p", C.c_double), ("min_ratio_12_l", C.c_double), ("homog_th", C.c_double),
                ("min_error", C.c_double), ("min_error_change", C.c_double), ("inlier_k", C.c_double),
                ("lsd_scale", C.c_double)]


class PlFrameBatch(C.Structure):
    _fields_ = [("B", C.c_int32), ("pt_off", c_int32_p), ("ls_off", c_int32_p),
                ("pdesc", c_uint8_p), ("ldesc", c_uint8_p),
                ("pt_P", c_double_p), ("pt_pl", c_double_p), ("pt_sigma2", c_double_p),
                ("ls_sP", c_double_p), ("ls_eP", c_double_p), ("ls_le", c_double_p),
                ("ls_spl", c_double_p), ("ls_epl", c_double_p), ("ls_sigma2", c_double_p),
                ("ls_level", c_int32_p)]


class PlMatchedBatch(C.Structure):
    _fields_ = [("B", C.c_int32), ("pt_off", c_int32_p), ("ls_off", c_int32_p),
                ("pt_P", c_double_p), ("pt_pl_obs", c_double_p), ("pt_sigma2", c_double_p),
                ("pt_inlier", c_uint8_p),
                ("ls_sP", c_double_p), ("ls_eP", c_double_p), ("ls_le_obs", c_double_p),
                ("ls_spl", c_double_p), ("ls_epl", c_double_p), ("ls_sigma2", c_double_p),
                ("ls_inlier", c_uint8_p)]


class PlGridWindow(C.Structure):
    """GridWindow: width = (left, right), height = (up, down) — include/gridStructure.h:39-41."""
    _fields_ = [("left", C.c_int32), ("right", C.c_int32), ("up", C.c_int32), ("down", C.c_int32)]


class PlStereoConfig(C.Structure):
    """Config values read by the 3-D lifting step (include/config.h:72-96, src/config.cpp:58-106)."""
    _fields_ = [(k, C.c_double) for k in ("max_dist_epip", "min_disp", "ls_min_disp_ratio", "line_horiz_th",
                                          "stereo_overlap_th", "orb_scale_factor", "lsd_scale")]


def default_stereo_config() -> "PlStereoConfig":
    return PlStereoConfig(1.0, 1.0, 0.7, 0.1, 0.75, 1.2, 1.2)   # src/config.cpp:58-69, :96, :106


class PlOrbConfig(C.Structure):
    """cv::ORB parameters of plstvo_orb_compute_batch (src/config.cpp:95-102); patch_size 31 and wta_k 2 only."""
    _fields_ = [("n_levels", C.c_int32), ("scale_factor", C.c_double), ("edge_threshold", C.c_int32),
                ("patch_size", C.c_int32), ("wta_k", C.c_int32)]


def default_orb_config(n_levels: int = 4, scale_factor: float = 1.2) -> "PlOrbConfig":
    return PlOrbConfig(n_levels, scale_factor, 19, 31, 2)   # config_kitti.yaml: 1 level


class PlOrbDetectConfig(C.Structure):
    """cv::ORB parameters of plstvo_orb_detect_and_compute_batch: score_type 1 FAST_SCORE, 0 HARRIS_SCORE."""
    _fields_ = [("orb", PlOrbConfig), ("n_features", C.c_int32), ("score_type", C.c_int32), ("fast_threshold", C.c_int32)]


class PlLsdConfig(C.Structure):
    """LineSegmentDetector parameters of plstvo_lsd_detect_batch (Config::lsd*), min_line_length relative to min(W, H)."""
    _fields_ = [("refine", C.c_int32), ("scale", C.c_double), ("sigma_scale", C.c_double), ("quant", C.c_double),
                ("ang_th", C.c_double), ("n_bins", C.c_int32), ("min_line_length", C.c_double), ("n_features", C.c_int32)]


def default_lsd_config(n_features: int = 300, **kw) -> "PlLsdConfig":
    """The shipped configs' LSD options: refine 0, scale 1.2, sigma_scale 0.6, quant 2.0, ang_th 22.5, n_bins 1024,
    min_line_length 0.025; keyword arguments override any field."""
    c = PlLsdConfig(0, 1.2, 0.6, 2.0, 22.5, 1024, 0.025, n_features)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


RECTIFY_PINHOLE, RECTIFY_FISHEYE = 0, 1


class PlRectifyModel(C.Structure):
    """One camera's undistort-rectify model (PlRectifyModel, include/plstvo.h): model 0 pinhole / 1 fisheye, n_dist
    coefficients of D, K 3x3, R 3x3 and P 3x4, row-major; every field double."""
    _fields_ = [("model", C.c_double), ("n_dist", C.c_double), ("K", C.c_double * 9), ("D", C.c_double * 8),
                ("R", C.c_double * 9), ("P", C.c_double * 12)]


def rectify_model(model: int, K, D, R, P) -> "PlRectifyModel":
    """PlRectifyModel from arrays: K 3x3, D of 4 / 5 / 8 coefficients, R 3x3, P 3x3 or 3x4 (a 3x3 P gets a zero column)."""
    D = np.asarray(D, np.float64).ravel()
    P = np.asarray(P, np.float64)
    if P.shape == (3, 3):
        P = np.hstack([P, np.zeros((3, 1))])
    m = PlRectifyModel()
    m.model, m.n_dist = float(model), float(D.size)
    m.K[:] = np.asarray(K, np.float64).ravel().tolist()
    m.D[:min(D.size, 8)] = D[:8].tolist()   # a longer D keeps its count, which the library rejects
    m.R[:] = np.asarray(R, np.float64).ravel().tolist()
    m.P[:] = P.ravel().tolist()
    return m


ORB_HARRIS_SCORE, ORB_FAST_SCORE = 0, 1


def default_orb_detect_config(n_features: int = 1200, n_levels: int = 4, scale_factor: float = 1.2,
                              score_type: int = ORB_FAST_SCORE, fast_threshold: int = 20) -> "PlOrbDetectConfig":
    """src/config.cpp:95-102 defaults: 1200 features, scale 1.2, 4 levels, edge 19, FAST score, patch 31, WTA_K 2, FAST 20."""
    return PlOrbDetectConfig(default_orb_config(n_levels, scale_factor), n_features, score_type, fast_threshold)


class PlStereoMatchConfig(C.Structure):
    """Grid / matcher values of matchStereoPoints / matchStereoLines (include/stereoFrame.h:51-52, src/config.cpp:51, :60, :63, :91)."""
    _fields_ = [("grid_rows", C.c_int32), ("grid_cols", C.c_int32), ("matching_s_ws", C.c_int32), ("best_lr_matches", C.c_int32),
                ("min_ratio_12_p", C.c_double), ("line_sim_th", C.c_double)]


def default_stereo_match_config() -> "PlStereoMatchConfig":
    return PlStereoMatchConfig(48, 64, 10, 1, 0.9, 0.75)


class PlStereoFeatures(C.Structure):
    """Raw stereo features of B frames (PlStereoFeatures, include/plstvo.h)."""
    _fields_ = [("B", C.c_int32), ("pl_off", c_int32_p), ("pr_off", c_int32_p), ("kp_l", c_float_p), ("kp_r", c_float_p),
                ("poct_l", c_int32_p), ("pdesc_l", c_uint8_p), ("pdesc_r", c_uint8_p), ("ll_off", c_int32_p), ("lr_off", c_int32_p),
                ("seg_l", c_float_p), ("seg_r", c_float_p), ("angle_l", c_float_p), ("loct_l", c_int32_p), ("ldesc_l", c_uint8_p),
                ("ldesc_r", c_uint8_p)]


STEREO_FEATURE_DTYPES = dict(pl_off=np.int32, pr_off=np.int32, kp_l=np.float32, kp_r=np.float32, poct_l=np.int32, pdesc_l=np.uint8,
                             pdesc_r=np.uint8, ll_off=np.int32, lr_off=np.int32, seg_l=np.float32, seg_r=np.float32,
                             angle_l=np.float32, loct_l=np.int32, ldesc_l=np.uint8, ldesc_r=np.uint8)


def stereo_features_as_c(d: dict):
    """dict of arrays (keys of STEREO_FEATURE_DTYPES) -> (PlStereoFeatures, keep-alive list)."""
    keep = {k: np.ascontiguousarray(d[k], dt) for k, dt in STEREO_FEATURE_DTYPES.items()}
    s = PlStereoFeatures()
    s.B = len(keep["pl_off"]) - 1
    for k, a in keep.items():
        typ = dict(PlStereoFeatures._fields_)[k]
        setattr(s, k, a.ctypes.data_as(typ))
    return s, keep


class PlStereoImages(C.Structure):
    """Stereo images and their key lines of B frames (PlStereoImages, include/plstvo.h)."""
    _fields_ = [("B", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("img_l", c_uint8_p), ("img_r", c_uint8_p),
                ("fast_th", c_int32_p), ("ll_off", c_int32_p), ("lr_off", c_int32_p), ("seg_l", c_float_p), ("seg_r", c_float_p),
                ("angle_l", c_float_p), ("angle_r", c_float_p), ("npix_l", c_int32_p), ("npix_r", c_int32_p)]


_C_PTR = {np.float64: c_double_p, np.int32: c_int32_p, np.uint8: c_uint8_p}


class FrameRecord(NamedTuple):
    """One lifted array: its PlStereoFrameOut field, its key in Engine.stereo_outputs' dicts, dtype, shape of one row, and
    whether it is a point (True) or a line array."""
    field: str
    key: str
    dtype: type
    row: tuple
    point: bool

    @property
    def ctype(self):
        return _C_PTR[self.dtype]


# The 19 lifted arrays, once, in PlStereoFrameOut's field order (include/plstvo.h): the lifting and matchStereo calls write
# them in this order, and plstvo_stereo_session_read / _read_keyframes fill them.
FRAME_OUT_RECORDS = tuple(FrameRecord(*r) for r in (
    ("pt_pl", "pl", np.float64, (2,), True), ("pt_disp", "disp", np.float64, (), True),
    ("pt_P", "P", np.float64, (3,), True), ("pt_sigma2", "sigma2", np.float64, (), True),
    ("pt_level", "level", np.int32, (), True), ("pdesc", "desc", np.uint8, (DESC_BYTES,), True),
    ("pt_src", "src_idx", np.int32, (), True),
    ("ls_spl", "spl", np.float64, (2,), False), ("ls_epl", "epl", np.float64, (2,), False),
    ("ls_sdisp", "sdisp", np.float64, (), False), ("ls_edisp", "edisp", np.float64, (), False),
    ("ls_sP", "sP", np.float64, (3,), False), ("ls_eP", "eP", np.float64, (3,), False),
    ("ls_le", "le", np.float64, (3,), False), ("ls_angle", "angle", np.float64, (), False),
    ("ls_sigma2", "sigma2", np.float64, (), False), ("ls_level", "level", np.int32, (), False),
    ("ldesc", "desc", np.uint8, (DESC_BYTES,), False), ("ls_src", "src_idx", np.int32, (), False)))
FRAME_OUT_POINT_RECORDS = tuple(r for r in FRAME_OUT_RECORDS if r.point)
FRAME_OUT_LINE_RECORDS = tuple(r for r in FRAME_OUT_RECORDS if not r.point)


class PlStereoFrameOut(C.Structure):
    """Destinations of plstvo_stereo_session_read (PlStereoFrameOut, include/plstvo.h); a NULL field is not copied."""
    _fields_ = [(r.field, r.ctype) for r in FRAME_OUT_RECORDS] + [
        ("m12_pt", c_int32_p), ("inlier_pt", c_uint8_p), ("m12_ls", c_int32_p), ("inlier_ls", c_uint8_p)]


# PlStereoFrameOut's point / line fields and the keys of Engine.match_stereo_points / _lines' outputs they correspond to
FRAME_OUT_POINT_KEYS = {r.field: r.key for r in FRAME_OUT_POINT_RECORDS}
FRAME_OUT_LINE_KEYS = {r.field: r.key for r in FRAME_OUT_LINE_RECORDS}


STEREO_IMAGE_DTYPES = dict(img_l=np.uint8, img_r=np.uint8, fast_th=np.int32, ll_off=np.int32, lr_off=np.int32, seg_l=np.float32,
                           seg_r=np.float32, angle_l=np.float32, angle_r=np.float32, npix_l=np.int32, npix_r=np.int32)


def stereo_images_as_c(d: dict):
    """dict with img_l / img_r uint8[B, H, W] (uint8[B, H, W, C] for a colour rectifier) and optionally fast_th [B] and the
    key-line arrays (keys of STEREO_IMAGE_DTYPES; a missing or None entry is passed as NULL) -> (PlStereoImages, keep-alive
    dict)."""
    keep = {k: None if d.get(k) is None else np.ascontiguousarray(d[k], dt) for k, dt in STEREO_IMAGE_DTYPES.items()}
    s = PlStereoImages()
    B, H, W = keep["img_l"].shape[:3]
    s.B, s.width, s.height = B, W, H
    for k, a in keep.items():
        typ = dict(PlStereoImages._fields_)[k]
        setattr(s, k, C.cast(None, typ) if a is None else a.ctypes.data_as(typ))
    return s, keep


GRID_ROWS, GRID_COLS = 48, 64     # include/stereoFrame.h:51-52


class PlPrior(C.Structure):
    _fields_ = [("Tfw", C.c_double * 16), ("Tfw_cov", C.c_double * 36), ("DT", C.c_double * 16),
                ("DT_cov", C.c_double * 36), ("err_norm", C.c_double)]


class PlPoseResult(C.Structure):
    _fields_ = [("DT", C.c_double * 16), ("DT_cov", C.c_double * 36), ("DT_cov_eig", C.c_double * 6),
                ("err_norm", C.c_double), ("Tfw", C.c_double * 16), ("Tfw_cov", C.c_double * 36),
                ("DT_opt", C.c_double * 16),
                ("n_matched_pt", C.c_int32), ("n_matched_ls", C.c_int32), ("n_inliers_pt", C.c_int32),
                ("n_inliers_ls", C.c_int32), ("n_inliers", C.c_int32), ("good", C.c_int32),
                ("status", C.c_int32), ("iters_stage1", C.c_int32), ("iters_stage2", C.c_int32),
                ("reserved", C.c_int32)]


# numpy view of PlPoseResult (same layout; C struct has no padding: 147 doubles + 10 int32)
POSE_RESULT_DTYPE = np.dtype([
    ("DT", "f8", (4, 4)), ("DT_cov", "f8", (6, 6)), ("DT_cov_eig", "f8", (6,)), ("err_norm", "f8"),
    ("Tfw", "f8", (4, 4)), ("Tfw_cov", "f8", (6, 6)), ("DT_opt", "f8", (4, 4)),
    ("n_matched_pt", "i4"), ("n_matched_ls", "i4"), ("n_inliers_pt", "i4"), ("n_inliers_ls", "i4"),
    ("n_inliers", "i4"), ("good", "i4"), ("status", "i4"), ("iters_stage1", "i4"),
    ("iters_stage2", "i4"), ("reserved", "i4")])
assert POSE_RESULT_DTYPE.itemsize == C.sizeof(PlPoseResult)

class PlHandlerConfig(C.Structure):
    """updateFrame's adaptive FAST threshold (Config::adaptativeFAST, fastMinTh .. fastErrTh) of plstvo_stereo_session_run."""
    _fields_ = [("adaptative_fast", C.c_int32), ("fast_min_th", C.c_int32), ("fast_max_th", C.c_int32),
                ("fast_inc_th", C.c_int32), ("fast_feat_th", C.c_int32), ("fast_err_th", C.c_float)]


def handler_config(h) -> "PlHandlerConfig":
    """The PlHandlerConfig of a handler.HandlerConfig (or any object with its fields)."""
    return PlHandlerConfig(int(bool(h.adaptative_fast)), h.fast_min_th, h.fast_max_th, h.fast_inc_th, h.fast_feat_th,
                           float(h.fast_err_th))


PRIOR_DTYPE = np.dtype([("Tfw", "f8", (4, 4)), ("Tfw_cov", "f8", (6, 6)), ("DT", "f8", (4, 4)),
                        ("DT_cov", "f8", (6, 6)), ("err_norm", "f8")])
assert PRIOR_DTYPE.itemsize == C.sizeof(PlPrior)

# plstvo_stereo_session_run_keyframes: needNewKF's thresholds, one stream's key-frame state, one stream's test at one step
KEYFRAME_CONFIG_DTYPE = np.dtype([("min_entropy_ratio", "f8"), ("max_kf_t_dist", "f8"), ("max_kf_r_dist", "f8")])
KEYFRAME_STATE_DTYPE = np.dtype([("prev_f_iskf", "i4"), ("N_prevKF_currF", "i4"), ("entropy_first_prevKF", "f8"),
                                 ("T_prevKF", "f8", (4, 4)), ("cov_prevKF_currF", "f8", (6, 6))])
KEYFRAME_RESULT_DTYPE = np.dtype([("new_kf", "i4"), ("N_prevKF_currF", "i4"), ("entropy_curr", "f8"), ("entropy_ratio", "f8"),
                                  ("t", "f8"), ("r", "f8")])


def keyframe_config(h) -> np.ndarray:
    """The PlKeyframeConfig (KEYFRAME_CONFIG_DTYPE, one record) of a handler.HandlerConfig (or any object with its fields)."""
    return np.array([(h.min_entropy_ratio, h.max_kf_t_dist, h.max_kf_r_dist)], KEYFRAME_CONFIG_DTYPE)

ST_REFINED, ST_ROBUST_FALLBACK, ST_FEW_BEFORE, ST_FEW_AFTER = 0, 1, 2, 3


def _ptr(a: Optional[np.ndarray], typ):
    if a is None:
        return C.cast(None, typ)
    return a.ctypes.data_as(typ)


def _arr(a, dtype, shape_tail=()):
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=dtype)
    if shape_tail:
        a = a.reshape((-1,) + tuple(shape_tail))
    return a


# ---- Config presets -------------------------------------------------------------------------------
def default_config() -> PlConfig:
    """Config::Config() defaults, src/config.cpp:36-113."""
    return PlConfig(has_points=1, has_lines=1, best_lr_matches=1, use_motion_model=0, min_features=10,
                    max_iters=5, max_iters_ref=10, solver_mode=0, min_ratio_12_p=0.9, min_ratio_12_l=0.9,
                    homog_th=1e-7, min_error=1e-7, min_error_change=1e-7, inlier_k=4.0, lsd_scale=1.2)


def kitti_config() -> PlConfig:
    """config/config/config_kitti.yaml:3-45."""
    c = default_config()
    c.min_ratio_12_p = 0.75
    c.min_ratio_12_l = 0.75
    c.inlier_k = 1.2
    return c


def euroc_config() -> PlConfig:
    """config/config/config_euroc.yaml optimisation block = the defaults (ratios 0.9, inlier_k 4.0)."""
    return default_config()


def kitti_camera() -> PlCamera:
    """config/dataset_params/kitti00-02.yaml:2-13."""
    return PlCamera(fx=718.856, fy=718.856, cx=607.1928, cy=185.2157, b=0.537165719, width=1241, height=376)


def euroc_camera() -> PlCamera:
    """752x480, baseline config/dataset_params/euroc_params.yaml:8-11; rectified intrinsics are produced
    at run time by stereoRectify in the reference and are not in the repo: assumed values (SURVEY 8(d))."""
    return PlCamera(fx=435.2047, fy=435.2047, cx=367.4517, cy=252.2009, b=0.110077842, width=752, height=480)


def hd_camera() -> PlCamera:
    """High-density roofline config C5 (assumed, SURVEY 8(d))."""
    return PlCamera(fx=1000.0, fy=1000.0, cx=960.0, cy=540.0, b=0.12, width=1920, height=1080)


# ---- containers -----------------------------------------------------------------------------------
@dataclass
class FrameBatch:
    """B stereo frames with pre-extracted features, SoA, concatenated (PlFrameBatch)."""
    pt_off: np.ndarray
    ls_off: np.ndarray
    pdesc: np.ndarray
    ldesc: np.ndarray
    pt_P: Optional[np.ndarray] = None
    pt_pl: Optional[np.ndarray] = None
    pt_sigma2: Optional[np.ndarray] = None
    ls_sP: Optional[np.ndarray] = None
    ls_eP: Optional[np.ndarray] = None
    ls_le: Optional[np.ndarray] = None
    ls_spl: Optional[np.ndarray] = None
    ls_epl: Optional[np.ndarray] = None
    ls_sigma2: Optional[np.ndarray] = None
    ls_level: Optional[np.ndarray] = None

    def __post_init__(self):
        self.pt_off = _arr(self.pt_off, np.int32)
        self.ls_off = _arr(self.ls_off, np.int32)
        self.pdesc = _arr(self.pdesc, np.uint8, (DESC_BYTES,))
        self.ldesc = _arr(self.ldesc, np.uint8, (DESC_BYTES,))
        self.pt_P = _arr(self.pt_P, np.float64, (3,))
        self.pt_pl = _arr(self.pt_pl, np.float64, (2,))
        self.pt_sigma2 = _arr(self.pt_sigma2, np.float64)
        self.ls_sP = _arr(self.ls_sP, np.float64, (3,))
        self.ls_eP = _arr(self.ls_eP, np.float64, (3,))
        self.ls_le = _arr(self.ls_le, np.float64, (3,))
        self.ls_spl = _arr(self.ls_spl, np.float64, (2,))
        self.ls_epl = _arr(self.ls_epl, np.float64, (2,))
        self.ls_sigma2 = _arr(self.ls_sigma2, np.float64)
        self.ls_level = _arr(self.ls_level, np.int32)
        assert self.pt_off.shape == self.ls_off.shape and self.pt_off[0] == 0 and self.ls_off[0] == 0
        assert self.pdesc.shape[0] == self.pt_off[-1] and self.ldesc.shape[0] == self.ls_off[-1]

    @property
    def B(self) -> int:
        return int(self.pt_off.shape[0] - 1)

    @property
    def n_pt(self) -> int:
        return int(self.pt_off[-1])

    @property
    def n_ls(self) -> int:
        return int(self.ls_off[-1])

    def as_c(self) -> PlFrameBatch:
        return PlFrameBatch(
            B=self.B, pt_off=_ptr(self.pt_off, c_int32_p), ls_off=_ptr(self.ls_off, c_int32_p),
            pdesc=_ptr(self.pdesc, c_uint8_p), ldesc=_ptr(self.ldesc, c_uint8_p),
            pt_P=_ptr(self.pt_P, c_double_p), pt_pl=_ptr(self.pt_pl, c_double_p),
            pt_sigma2=_ptr(self.pt_sigma2, c_double_p),
            ls_sP=_ptr(self.ls_sP, c_double_p), ls_eP=_ptr(self.ls_eP, c_double_p),
            ls_le=_ptr(self.ls_le, c_double_p), ls_spl=_ptr(self.ls_spl, c_double_p),
            ls_epl=_ptr(self.ls_epl, c_double_p), ls_sigma2=_ptr(self.ls_sigma2, c_double_p),
            ls_level=_ptr(self.ls_level, c_int32_p))

    def select(self, idx: Sequence[int]) -> "FrameBatch":
        """Sub-batch made of the frames `idx` (copies)."""
        idx = list(idx)
        pt = [np.arange(self.pt_off[i], self.pt_off[i + 1]) for i in idx]
        ls = [np.arange(self.ls_off[i], self.ls_off[i + 1]) for i in idx]
        pi = np.concatenate(pt) if pt else np.zeros(0, np.int64)
        li = np.concatenate(ls) if ls else np.zeros(0, np.int64)

        def take(a, ii):
            return None if a is None else a[ii]
        return FrameBatch(
            pt_off=np.concatenate([[0], np.cumsum([len(x) for x in pt])]),
            ls_off=np.concatenate([[0], np.cumsum([len(x) for x in ls])]),
            pdesc=self.pdesc[pi], ldesc=self.ldesc[li], pt_P=take(self.pt_P, pi), pt_pl=take(self.pt_pl, pi),
            pt_sigma2=take(self.pt_sigma2, pi), ls_sP=take(self.ls_sP, li), ls_eP=take(self.ls_eP, li),
            ls_le=take(self.ls_le, li), ls_spl=take(self.ls_spl, li), ls_epl=take(self.ls_epl, li),
            ls_sigma2=take(self.ls_sigma2, li), ls_level=take(self.ls_level, li))

    def input_bytes(self, role: str) -> int:
        """Bytes of the arrays the given role ('prev' / 'curr') uploads."""
        n, m = self.n_pt, self.n_ls
        if role == "prev":
            return 32 * (n + m) + 8 * (3 + 1) * n + (8 * (3 + 3 + 2 + 2 + 1) + 4) * m
        return 32 * (n + m) + 16 * n + 24 * m


@dataclass
class MatchedBatch:
    """Explicit matched_pt / matched_ls lists for B problems (PlMatchedBatch)."""
    pt_off: np.ndarray
    ls_off: np.ndarray
    pt_P: np.ndarray
    pt_pl_obs: np.ndarray
    pt_sigma2: np.ndarray
    ls_sP: np.ndarray
    ls_eP: np.ndarray
    ls_le_obs: np.ndarray
    ls_spl: np.ndarray
    ls_epl: np.ndarray
    ls_sigma2: np.ndarray
    pt_inlier: Optional[np.ndarray] = None
    ls_inlier: Optional[np.ndarray] = None

    def __post_init__(self):
        self.pt_off = _arr(self.pt_off, np.int32)
        self.ls_off = _arr(self.ls_off, np.int32)
        self.pt_P = _arr(self.pt_P, np.float64, (3,))
        self.pt_pl_obs = _arr(self.pt_pl_obs, np.float64, (2,))
        self.pt_sigma2 = _arr(self.pt_sigma2, np.float64)
        self.ls_sP = _arr(self.ls_sP, np.float64, (3,))
        self.ls_eP = _arr(self.ls_eP, np.float64, (3,))
        self.ls_le_obs = _arr(self.ls_le_obs, np.float64, (3,))
        self.ls_spl = _arr(self.ls_spl, np.float64, (2,))
        self.ls_epl = _arr(self.ls_epl, np.float64, (2,))
        self.ls_sigma2 = _arr(self.ls_sigma2, np.float64)
        self.pt_inlier = _arr(self.pt_inlier, np.uint8)
        self.ls_inlier = _arr(self.ls_inlier, np.uint8)

    @property
    def B(self) -> int:
        return int(self.pt_off.shape[0] - 1)

    def as_c(self) -> PlMatchedBatch:
        return PlMatchedBatch(
            B=self.B, pt_off=_ptr(self.pt_off, c_int32_p), ls_off=_ptr(self.ls_off, c_int32_p),
            pt_P=_ptr(self.pt_P, c_double_p), pt_pl_obs=_ptr(self.pt_pl_obs, c_double_p),
            pt_sigma2=_ptr(self.pt_sigma2, c_double_p), pt_inlier=_ptr(self.pt_inlier, c_uint8_p),
            ls_sP=_ptr(self.ls_sP, c_double_p), ls_eP=_ptr(self.ls_eP, c_double_p),
            ls_le_obs=_ptr(self.ls_le_obs, c_double_p), ls_spl=_ptr(self.ls_spl, c_double_p),
            ls_epl=_ptr(self.ls_epl, c_double_p), ls_sigma2=_ptr(self.ls_sigma2, c_double_p),
            ls_inlier=_ptr(self.ls_inlier, c_uint8_p))


def matched_from_frames(prev: FrameBatch, curr: FrameBatch, m12_pt: np.ndarray, m12_ls: np.ndarray,
                        lsd_scale: float = 1.2) -> MatchedBatch:
    """Host restatement of the f2fTracking glue (src/stereoFrameHandler.cpp:144-152, :167-179):
    matched lists in ascending prev index with the LineFeature::safeCopy sigma2 rule
    (src/stereoFeatures.cpp:117-135).  Used by tests to feed the explicit-list API."""
    pt_off, ls_off = [0], [0]
    P, obs, s2 = [], [], []
    sP, eP, le, spl, epl, ls2 = [], [], [], [], [], []
    for p in range(prev.B):
        a0, a1, b0 = prev.pt_off[p], prev.pt_off[p + 1], curr.pt_off[p]
        m = np.asarray(m12_pt[a0:a1])
        i1 = np.nonzero(m >= 0)[0]
        P.append(prev.pt_P[a0 + i1]); obs.append(curr.pt_pl[b0 + m[i1]]); s2.append(prev.pt_sigma2[a0 + i1])
        pt_off.append(pt_off[-1] + len(i1))
        a0, a1, b0 = prev.ls_off[p], prev.ls_off[p + 1], curr.ls_off[p]
        m = np.asarray(m12_ls[a0:a1])
        i1 = np.nonzero(m >= 0)[0]
        sP.append(prev.ls_sP[a0 + i1]); eP.append(prev.ls_eP[a0 + i1]); le.append(curr.ls_le[b0 + m[i1]])
        spl.append(prev.ls_spl[a0 + i1]); epl.append(prev.ls_epl[a0 + i1])
        s = prev.ls_sigma2[a0 + i1].copy()
        lev = prev.ls_level[a0 + i1] if prev.ls_level is not None else np.zeros(len(i1), np.int32)
        for k in range(int(lev.max()) if len(lev) else 0):
            s = np.where(lev > k, s * lsd_scale, s)
        ls2.append(1.0 / (s * s))
        ls_off.append(ls_off[-1] + len(i1))
    cat = lambda xs, w: (np.concatenate(xs) if xs else np.zeros((0, w))).reshape(-1, w) if w > 1 else \
        (np.concatenate(xs) if xs else np.zeros(0))
    return MatchedBatch(pt_off=pt_off, ls_off=ls_off, pt_P=cat(P, 3), pt_pl_obs=cat(obs, 2), pt_sigma2=cat(s2, 1),
                        ls_sP=cat(sP, 3), ls_eP=cat(eP, 3), ls_le_obs=cat(le, 3), ls_spl=cat(spl, 2),
                        ls_epl=cat(epl, 2), ls_sigma2=cat(ls2, 1))


def identity_priors(B: int) -> np.ndarray:
    """prev_frame state after initialize(): Tfw = I, Tfw_cov = I, DT = I (src/stereoFrameHandler.cpp:43-45)."""
    pr = np.zeros(B, dtype=PRIOR_DTYPE)
    pr["Tfw"] = np.eye(4)
    pr["Tfw_cov"] = np.eye(6)
    pr["DT"] = np.eye(4)
    pr["DT_cov"] = 0.0
    pr["err_norm"] = 0.0
    return pr
