"""StVO::StereoFrameHandler surface (include/stereoFrameHandler.h:34-101) over the C-ABI, for frames of
pre-extracted features (feature extraction is the reference's own, out of scope here).

Call sequence of app/imagesStVO.cpp:88-124:
    h = StereoFrameHandler(cam, cfg); h.initialize(frame0)
    for frame in frames: h.insertStereoPair(frame); h.optimizePose(); ...read h.curr_frame...; h.updateFrame()
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from . import types as T
from .engine import Engine


@dataclass
class HandlerConfig:
    """Config values of the host-side state machine (src/config.cpp:40-42, :52, :72-76, :102)."""
    adaptative_fast: bool = True
    fast_min_th: int = 5
    fast_max_th: int = 50
    fast_inc_th: int = 5
    fast_feat_th: int = 50
    fast_err_th: float = 0.5
    orb_fast_th: int = 20
    min_entropy_ratio: float = 0.85
    max_kf_t_dist: float = 5.0
    max_kf_r_dist: float = 15.0


def update_fast_threshold(c: HandlerConfig, orb_fast_th: int, DT, err_norm: float, n_inliers_pt: int) -> int:
    """updateFrame's adaptive FAST threshold (src/stereoFrameHandler.cpp:66-86)."""
    if not c.adaptative_fast:
        return orb_fast_th
    inc, feat = c.fast_inc_th, c.fast_feat_th
    if np.array_equal(np.asarray(DT).reshape(4, 4), np.eye(4)) or err_norm > float(np.float32(c.fast_err_th)):
        return max(c.fast_min_th, orb_fast_th - 2 * inc)
    if n_inliers_pt < feat:
        return max(c.fast_min_th, orb_fast_th - 2 * inc)
    if n_inliers_pt < 2 * feat:
        return max(c.fast_min_th, orb_fast_th - inc)
    if n_inliers_pt > 3 * feat:
        return min(c.fast_max_th, orb_fast_th + inc)
    return orb_fast_th          # the reference's "> 4 feat" branch (:84-85) sits behind "> 3 feat": unreachable


def _inverse_se3(T):
    Ti = np.eye(4)
    Ti[:3, :3] = T[:3, :3].T
    Ti[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return Ti


def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], float)


def _adjoint_se3(T):
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = T[:3, :3]
    A[:3, 3:] = _skew(T[:3, 3]) @ T[:3, :3]
    return A


def _logmap_se3(T):
    """src/auxiliar.cpp:143-173."""
    R = T[:3, :3]
    cosine = min(1.0, max(-1.0, (np.trace(R) - 1.0) / 2.0))
    sine = min(1.0, np.sqrt(1.0 - cosine * cosine))
    theta = np.arccos(cosine)
    w, V = np.zeros(3), np.eye(3)
    if theta > 1e-6:
        w_hat = theta * (R - R.T) / (2.0 * sine)
        w = np.array([w_hat[2, 1], w_hat[0, 2], w_hat[1, 0]])
        s = _skew(w) / theta
        V = np.eye(3) + s * (1.0 - cosine) / theta + s @ s * (theta - sine) / theta
    return np.concatenate([np.linalg.solve(V, T[:3, 3]), w])


def chain_poses(results, Tfw0=None, cov0=None):
    """World poses of a sequence from per-pair results solved with identity priors (plstvo_track_stereo_sequence), chained like
    optimizePose's tail (src/stereoFrameHandler.cpp:377-378, :388-389).  Writes results["Tfw"], results["Tfw_cov"] in place."""
    from .synth import expmap_se3
    T_ = np.eye(4) if Tfw0 is None else np.asarray(Tfw0, float).reshape(4, 4).copy()
    cov = np.eye(6) if cov0 is None else np.asarray(cov0, float).reshape(6, 6).copy()
    for k in range(len(results)):
        if results["good"][k]:
            A = _adjoint_se3(T_)
            cov = cov + A @ results["DT_cov"][k].reshape(6, 6) @ A.T
            T_ = expmap_se3(_logmap_se3(T_ @ results["DT"][k].reshape(4, 4)))
        results["Tfw"][k] = T_
        results["Tfw_cov"][k] = cov
    return results


class KeyframeTest:
    """needNewKF / currFrameIsKF (src/stereoFrameHandler.cpp:1136-1218; state include/stereoFrameHandler.h:81-86)."""
    K_ENTROPY = 3.0 * (1.0 + np.log(2.0 * np.arccos(-1.0)))

    def __init__(self):
        self.reset()

    def reset(self):
        self.prev_f_iskf, self.N_prevKF_currF = True, 0
        self.entropy_first_prevKF = 0.0
        self.T_prevKF, self.cov_prevKF_currF = np.eye(4), np.zeros((6, 6))
        self.entropy_curr = self.entropy_ratio = self.t = self.r = 0.0

    def needNewKF(self, c: HandlerConfig, Tfw, DT, DT_cov) -> bool:
        Tfw, DT, DT_cov = np.asarray(Tfw).reshape(4, 4), np.asarray(DT).reshape(4, 4), np.asarray(DT_cov).reshape(6, 6)
        with np.errstate(all="ignore"):
            if self.prev_f_iskf:
                d = np.linalg.det(DT_cov)
                self.entropy_first_prevKF = self.K_ENTROPY + 0.5 * np.log(d) if d != 0.0 else -999999999.99
                self.prev_f_iskf = False
            dX = _logmap_se3(_inverse_se3(Tfw) @ self.T_prevKF)
            self.t = float(np.linalg.norm(dX[:3]))
            self.r = float(np.linalg.norm(dX[3:]) * 180.0 / np.pi)
            adj_inv = _adjoint_se3(_inverse_se3(DT))
            adj_kf = _adjoint_se3(self.T_prevKF)
            self.cov_prevKF_currF = self.cov_prevKF_currF + adj_kf @ (adj_inv @ DT_cov @ adj_inv.T) @ adj_kf.T
            self.entropy_curr = float(self.K_ENTROPY + 0.5 * np.log(np.linalg.det(self.cov_prevKF_currF)))
            self.entropy_ratio = float(self.entropy_curr / self.entropy_first_prevKF)
        degenerate = not DT_cov.any() and np.array_equal(DT, np.eye(4))
        if (self.entropy_ratio < c.min_entropy_ratio or not np.isfinite(self.entropy_ratio) or degenerate
                or self.t > c.max_kf_t_dist or self.r > c.max_kf_r_dist or self.N_prevKF_currF > 10):
            return True
        self.N_prevKF_currF += 1
        return False

    def to_state(self) -> np.ndarray:
        """This test's state as one PlKeyframeState record (T.KEYFRAME_STATE_DTYPE), for StereoSession.run_keyframes."""
        s = np.zeros(1, T.KEYFRAME_STATE_DTYPE)
        s["prev_f_iskf"], s["N_prevKF_currF"] = int(bool(self.prev_f_iskf)), self.N_prevKF_currF
        s["entropy_first_prevKF"], s["T_prevKF"][0], s["cov_prevKF_currF"][0] = self.entropy_first_prevKF, self.T_prevKF, self.cov_prevKF_currF
        return s

    @classmethod
    def from_state(cls, s) -> "KeyframeTest":
        """The test standing in PlKeyframeState s (a T.KEYFRAME_STATE_DTYPE record); the diagnostics start at 0."""
        s = np.asarray(s, T.KEYFRAME_STATE_DTYPE).reshape(-1)[0]
        k = cls()
        k.prev_f_iskf, k.N_prevKF_currF = bool(s["prev_f_iskf"]), int(s["N_prevKF_currF"])
        k.entropy_first_prevKF = float(s["entropy_first_prevKF"])
        k.T_prevKF, k.cov_prevKF_currF = np.array(s["T_prevKF"], float), np.array(s["cov_prevKF_currF"], float)
        return k

    def currFrameIsKF(self, frame):
        frame.Tfw, frame.Tfw_cov = np.eye(4), np.eye(6)
        self.T_prevKF, self.cov_prevKF_currF = np.eye(4), np.zeros((6, 6))
        self.prev_f_iskf, self.N_prevKF_currF = True, 0


@dataclass
class StereoFrame:
    """What the path reads of StereoFrame (include/stereoFrame.h:59-115) + the per-frame results."""
    features: T.FrameBatch                    # a batch of exactly one frame
    frame_idx: int = 0
    Tfw: np.ndarray = field(default_factory=lambda: np.eye(4))
    Tfw_cov: np.ndarray = field(default_factory=lambda: np.eye(6))
    DT: np.ndarray = field(default_factory=lambda: np.eye(4))
    DT_cov: np.ndarray = field(default_factory=lambda: np.zeros((6, 6)))
    DT_cov_eig: np.ndarray = field(default_factory=lambda: np.zeros(6))
    err_norm: float = -1.0


def stereo_features(engine: Engine, cam: T.PlCamera, raw: dict, mcfg: Optional[T.PlStereoMatchConfig] = None,
                    scfg: Optional[T.PlStereoConfig] = None) -> T.FrameBatch:
    """The matching half of StereoFrame::extractStereoFeatures (matchStereoPoints + matchStereoLines, src/stereoFrame.cpp:120-173,
    :309-398) for ONE frame of raw stereo features (a dict with the PlStereoFeatures fields): the frame's stereo_pt / stereo_ls
    records as the FrameBatch the handler consumes."""
    mcfg, scfg = mcfg or T.default_stereo_match_config(), scfg or T.default_stereo_config()
    assert len(raw["pl_off"]) == 2, "one frame"
    kp, op = engine.match_stereo_points(cam, mcfg, scfg, raw["pl_off"], raw["kp_l"], raw["poct_l"], raw["pdesc_l"], raw["pr_off"],
                                        raw["kp_r"], raw["pdesc_r"])
    kl, ol = engine.match_stereo_lines(cam, mcfg, scfg, raw["ll_off"], raw["seg_l"], raw["angle_l"], raw["loct_l"], raw["ldesc_l"],
                                       raw["lr_off"], raw["seg_r"], raw["ldesc_r"])
    return T.FrameBatch(pt_off=[0, kp], ls_off=[0, kl], pdesc=op["desc"][:kp], ldesc=ol["desc"][:kl], pt_P=op["P"][:kp],
                        pt_pl=op["pl"][:kp], pt_sigma2=op["sigma2"][:kp], ls_sP=ol["sP"][:kl], ls_eP=ol["eP"][:kl],
                        ls_le=ol["le"][:kl], ls_spl=ol["spl"][:kl], ls_epl=ol["epl"][:kl], ls_sigma2=ol["sigma2"][:kl],
                        ls_level=ol["level"][:kl])


class StereoFrameHandler:
    def __init__(self, cam: T.PlCamera, cfg: Optional[T.PlConfig] = None, engine: Optional[Engine] = None,
                 hcfg: Optional[HandlerConfig] = None):
        self.cam, self.cfg = cam, cfg or T.default_config()
        self.hcfg = hcfg or HandlerConfig()
        self.orb_fast_th = self.hcfg.orb_fast_th         # src/stereoFrameHandler.cpp:38
        self.kf = KeyframeTest()
        self.engine = engine or Engine()
        self.prev_frame: Optional[StereoFrame] = None
        self.curr_frame: Optional[StereoFrame] = None
        self.matched_pt = np.zeros(0, np.int64)     # prev indices of matched_pt, ascending (list order)
        self.matched_ls = np.zeros(0, np.int64)
        self.n_inliers = self.n_inliers_pt = self.n_inliers_ls = 0
        self._pending = None

    def initialize(self, features: T.FrameBatch, idx: int = 0):
        """src/stereoFrameHandler.cpp:35-52: Tfw = I, Tfw_cov = I, DT = I."""
        assert features.B == 1
        self.prev_frame = StereoFrame(features, idx)
        self.curr_frame = self.prev_frame
        self.orb_fast_th = self.hcfg.orb_fast_th
        self.kf.reset()                                  # :48-51

    def insertStereoPair(self, features: T.FrameBatch, idx: int = 0):
        """src/stereoFrameHandler.cpp:54-60: new frame + f2fTracking.  The fused device call already computes the
        pose; optimizePose() publishes it."""
        assert features.B == 1 and self.prev_frame is not None
        self.curr_frame = StereoFrame(features, idx)
        self.f2fTracking()

    def f2fTracking(self):
        """src/stereoFrameHandler.cpp:106-129."""
        p = self.prev_frame
        pri = np.zeros(1, dtype=T.PRIOR_DTYPE)
        pri["Tfw"][0], pri["Tfw_cov"][0] = p.Tfw, p.Tfw_cov
        pri["DT"][0], pri["DT_cov"][0], pri["err_norm"][0] = p.DT, p.DT_cov, p.err_norm
        out = self.engine.track_batch(self.cam, self.cfg, p.features, self.curr_frame.features, priors=pri)
        self._pending = out
        self.m12_pt, self.m12_ls = out["m12_pt"], out["m12_ls"]
        self.matched_pt = np.nonzero(self.m12_pt >= 0)[0]
        self.matched_ls = np.nonzero(self.m12_ls >= 0)[0]
        self.n_inliers_pt, self.n_inliers_ls = len(self.matched_pt), len(self.matched_ls)   # :126-128
        self.n_inliers = self.n_inliers_pt + self.n_inliers_ls

    def optimizePose(self):
        """src/stereoFrameHandler.cpp:307-392."""
        r = self._pending["results"][0]
        c = self.curr_frame
        c.DT, c.DT_cov, c.DT_cov_eig, c.err_norm = r["DT"].copy(), r["DT_cov"].copy(), r["DT_cov_eig"].copy(), float(r["err_norm"])
        c.Tfw, c.Tfw_cov = r["Tfw"].copy(), r["Tfw_cov"].copy()
        self.inlier_pt = self._pending["inlier_pt"][self.matched_pt].astype(bool)    # flags in matched_pt order
        self.inlier_ls = self._pending["inlier_ls"][self.matched_ls].astype(bool)
        self.n_inliers_pt, self.n_inliers_ls, self.n_inliers = int(r["n_inliers_pt"]), int(r["n_inliers_ls"]), int(r["n_inliers"])
        self.status = int(r["status"])

    def needNewKF(self) -> bool:
        """src/stereoFrameHandler.cpp:1136-1187."""
        c = self.curr_frame
        return self.kf.needNewKF(self.hcfg, c.Tfw, c.DT, c.DT_cov)

    def currFrameIsKF(self):
        """src/stereoFrameHandler.cpp:1189-1218."""
        self.kf.currFrameIsKF(self.curr_frame)

    def updateFrame(self):
        """src/stereoFrameHandler.cpp:62-102: orb_fast_th is the threshold the caller's detector uses for the next frame."""
        c = self.curr_frame
        self.orb_fast_th = update_fast_threshold(self.hcfg, self.orb_fast_th, c.DT, c.err_norm, self.n_inliers_pt)
        self.matched_pt = np.zeros(0, np.int64)
        self.matched_ls = np.zeros(0, np.int64)
        self.prev_frame, self.curr_frame = self.curr_frame, None


# ---- scheduled session runs (plstvo_stereo_session_run_schedule): frames packing and the per-stream chain ----
SCHEDULE_IDLE, SCHEDULE_INSERT, SCHEDULE_INITIALIZE = 0, 1, 2
_LINE_SIDES = (("ll_off", "seg_l", "angle_l", "npix_l"), ("lr_off", "seg_r", "angle_r", "npix_r"))


def take_frames(frames: dict, idx) -> dict:
    """Frames idx (in that order) of a frames dict: images and fast_th sliced, and each side's key lines (FLD branch:
    ll_off / seg_l / angle_l / npix_l and the right side's) cut per frame and re-based to one CSR."""
    idx = np.asarray(idx, np.int64)
    out = {k: np.asarray(frames[k])[idx] for k in ("img_l", "img_r")}
    if frames.get("fast_th") is not None:
        out["fast_th"] = np.asarray(frames["fast_th"], np.int32)[idx]
    for off_k, seg_k, ang_k, npix_k in _LINE_SIDES:
        if frames.get(off_k) is None:
            continue
        off = np.asarray(frames[off_k], np.int64)
        rows = np.concatenate([np.arange(off[i], off[i + 1]) for i in idx]) if len(idx) else np.zeros(0, np.int64)
        out[off_k] = np.concatenate([[0], np.cumsum(off[idx + 1] - off[idx])]).astype(np.int32)
        out[seg_k] = np.asarray(frames[seg_k], np.float32).reshape(-1, 4)[rows]
        out[ang_k] = np.asarray(frames[ang_k], np.float32)[rows]
        out[npix_k] = np.asarray(frames[npix_k], np.int32)[rows]
    return out


def join_frames(parts) -> dict:
    """The frames dicts parts concatenated in order (take_frames' keys), key lines re-based to one CSR per side."""
    parts = list(parts)
    out = {k: np.concatenate([np.asarray(p[k]) for p in parts]) for k in ("img_l", "img_r")}
    if all(p.get("fast_th") is not None for p in parts) and parts:
        out["fast_th"] = np.concatenate([np.asarray(p["fast_th"], np.int32) for p in parts])
    for off_k, seg_k, ang_k, npix_k in _LINE_SIDES:
        if not parts or parts[0].get(off_k) is None:
            continue
        counts = np.concatenate([np.diff(np.asarray(p[off_k], np.int64)) for p in parts])
        out[off_k] = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        out[seg_k] = np.concatenate([np.asarray(p[seg_k], np.float32).reshape(-1, 4) for p in parts])
        out[ang_k] = np.concatenate([np.asarray(p[ang_k], np.float32) for p in parts])
        out[npix_k] = np.concatenate([np.asarray(p[npix_k], np.int32) for p in parts])
    return out


def schedule_frames(schedule, frame_of) -> dict:
    """The frames of a schedule [T, n], packed as plstvo_stereo_session_run_schedule takes them: one per non-zero entry,
    step-major and in call order within a step.  frame_of(t, k) gives entry (t, k)'s frame as a one-frame dict."""
    sched = np.asarray(schedule)
    return join_frames(frame_of(t, k) for t in range(sched.shape[0]) for k in range(sched.shape[1]) if sched[t, k])


def schedule_groups(schedule):
    """Per step t, the chain's two calls: (t, initialize positions, insert positions, their frames' indices in the packed
    frames, in the same order).  Steps with no entries are skipped."""
    sched = np.asarray(schedule)
    b, out = 0, []
    for t in range(sched.shape[0]):
        where = {}
        for k in range(sched.shape[1]):
            if sched[t, k]:
                where[k] = b
                b += 1
        init = [k for k in where if sched[t, k] == SCHEDULE_INITIALIZE]
        ins = [k for k in where if sched[t, k] == SCHEDULE_INSERT]
        if where:
            out.append((t, init, ins, [where[k] for k in init], [where[k] for k in ins]))
    return out


def fresh_prior() -> np.ndarray:
    """priorOf of a freshly initialised frame (Tfw = I, Tfw_cov = I, DT = I, DT_cov = 0, err_norm = -1): one T.PRIOR_DTYPE."""
    p = np.zeros(1, T.PRIOR_DTYPE)
    p["Tfw"], p["Tfw_cov"], p["DT"], p["err_norm"] = np.eye(4), np.eye(6), np.eye(4), -1.0
    return p


class ScheduleStreams:
    """The per-stream state a scheduled run carries, on the host: the FAST threshold the stream's next frame takes, its prior
    and, with the key-frame test, its state.  An idle step changes nothing; initialize resets all three to what
    HandlerState's initialize leaves; an insert takes them and leaves updateFrame's threshold, priorOf the published result
    and the test's state (currFrameIsKF's Tfw = I, Tfw_cov = I where it fired)."""

    def __init__(self, hcfg: HandlerConfig, th0, priors=None, kf_state=None):
        self.hcfg = hcfg
        self.th = np.asarray(th0, np.int32).copy()
        n = len(self.th)
        self.prior = np.repeat(fresh_prior(), n) if priors is None else np.array(priors, T.PRIOR_DTYPE).reshape(-1).copy()
        self.kf = None if kf_state is None else np.array(kf_state, T.KEYFRAME_STATE_DTYPE).reshape(-1).copy()

    def initialize(self, k: int, th: int):
        self.th[k] = th
        self.prior[k] = fresh_prior()[0]
        if self.kf is not None:
            self.kf[k] = KeyframeTest().to_state()[0]

    def inserted(self, k: int, r, kf_state=None, new_kf: bool = False):
        """Stream k's insert gave result r (and, with the test, the state after it and whether the frame became a key frame)."""
        self.th[k] = update_fast_threshold(self.hcfg, int(self.th[k]), r["DT"], float(r["err_norm"]), int(r["n_inliers_pt"]))
        for f in ("Tfw", "Tfw_cov", "DT", "DT_cov", "err_norm"):
            self.prior[k][f] = r[f]
        if self.kf is not None and kf_state is not None:
            self.kf[k] = kf_state
        if new_kf:
            self.prior[k]["Tfw"], self.prior[k]["Tfw_cov"] = np.eye(4), np.eye(6)
