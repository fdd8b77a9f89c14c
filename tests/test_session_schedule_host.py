"""plstvo_stereo_session_run_schedule without a GPU: the call is declared, exported and bound with the header's signature;
the Python packing of a schedule's frames (images, thresholds and the FLD branch's key lines) and the chain's groups; the
host mirror's per-stream chaining (an idle step carries the state, initialize resets it); and examples/schedule_cpp.cpp
(StereoStreamsHandler::insertStereoSequences with a schedule) compiles and links.  The call's own argument checks need a
context, so a GPU: tests/test_gpu_session_schedule.py pins each of them by its message."""
import ctypes as C
import os
import subprocess

import numpy as np

from conftest import ROOT
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import EXPORTED_SYMBOLS, LIB_PATH, load_library
from stvo_pl_b200.handler import (HandlerConfig, KeyframeTest, ScheduleStreams, fresh_prior, join_frames, schedule_frames,
                                  schedule_groups, take_frames, update_fast_threshold)
from test_stereo_session_host import declaration

LIBDIR = os.path.dirname(LIB_PATH)
NAME = "plstvo_stereo_session_run_schedule"


def test_schedule_call_is_declared_exported_and_bound():
    assert hasattr(C.CDLL(LIB_PATH), NAME)
    assert NAME in EXPORTED_SYMBOLS
    ret, params = declaration(NAME)
    fn = getattr(load_library(), NAME)
    assert ret == "int" and fn.restype is C.c_int
    assert len(fn.argtypes) == len(params) == 16
    # run_keyframes' arguments with the schedule after T and the key-frame state before the results
    _, rk = declaration("plstvo_stereo_session_run_keyframes")
    assert params[:7] == rk[:7]
    assert params[7].startswith("const uint8_t* schedule") and params[8] == rk[7]
    assert fn.argtypes[7] == C.POINTER(C.c_uint8) and fn.argtypes[8] == C.POINTER(T.PlStereoImages)


def frame(t, k, lines=True):
    """A one-frame dict whose pixels and key lines name (t, k)."""
    d = dict(img_l=np.full((1, 2, 3), 10 * t + k, np.uint8), img_r=np.full((1, 2, 3), 100 + 10 * t + k, np.uint8),
             fast_th=np.int32([t + k]))
    if lines:
        for side, m in (("l", k % 3), ("r", (k + 1) % 3)):
            d[f"l{side}_off"] = np.int32([0, m])
            d[f"seg_{side}"] = np.full((m, 4), 10 * t + k + (0.5 if side == "r" else 0), np.float32)
            d[f"angle_{side}"] = np.full(m, t - k, np.float32)
            d[f"npix_{side}"] = np.full(m, 3 + k, np.int32)
    return d


def test_schedule_frames_pack_step_major_with_key_lines():
    sched = np.uint8([[1, 0, 2], [0, 0, 0], [2, 1, 1]])
    f = schedule_frames(sched, frame)
    entries = [(t, k) for t in range(3) for k in range(3) if sched[t, k]]
    assert len(f["img_l"]) == len(entries) == 5
    for b, (t, k) in enumerate(entries):
        one = frame(t, k)
        assert f["img_l"][b].tobytes() == one["img_l"][0].tobytes() and f["img_r"][b].tobytes() == one["img_r"][0].tobytes()
        assert f["fast_th"][b] == t + k
        for off, seg, ang, npix in (("ll_off", "seg_l", "angle_l", "npix_l"), ("lr_off", "seg_r", "angle_r", "npix_r")):
            rows = slice(f[off][b], f[off][b + 1])
            np.testing.assert_array_equal(f[seg][rows], one[seg])
            np.testing.assert_array_equal(f[ang][rows], one[ang])
            np.testing.assert_array_equal(f[npix][rows], one[npix])
    # the chain's groups, and take_frames cutting a group's frames (key lines re-based) back out of the packing
    groups = schedule_groups(sched)
    assert [(t, init, ins) for t, init, ins, _, _ in groups] == [(0, [2], [0]), (2, [0], [1, 2])]
    t, init, ins, bi, bn = groups[1]
    assert bi == [2] and bn == [3, 4]
    g = take_frames(f, bn)
    want = join_frames([frame(2, 1), frame(2, 2)])
    assert g.keys() == want.keys()
    for key in g:
        np.testing.assert_array_equal(g[key], want[key], key)
    assert take_frames(f, [])["ll_off"].tolist() == [0]


def test_mirror_idle_carries_and_initialize_resets():
    h = HandlerConfig(fast_feat_th=20)
    pri = np.repeat(fresh_prior(), 2)
    pri["err_norm"] = [0.25, 0.5]
    kf = np.concatenate([KeyframeTest().to_state(), KeyframeTest().to_state()])
    kf["N_prevKF_currF"] = [3, 4]
    m = ScheduleStreams(h, [12, 30], pri, kf)
    r = np.zeros(1, T.POSE_RESULT_DTYPE)[0]
    r["DT"], r["DT_cov"], r["Tfw"], r["Tfw_cov"] = np.eye(4) * 2, np.eye(6) * 3, np.eye(4) * 4, np.eye(6) * 5
    r["err_norm"], r["n_inliers_pt"] = 0.125, 70
    after = KeyframeTest().to_state()[0]
    after["N_prevKF_currF"] = 9
    before1 = (m.th[1], m.prior[1].tobytes(), m.kf[1].tobytes())
    m.inserted(0, r, after, new_kf=False)
    # stream 1 idled: all of its state is carried unchanged
    assert (m.th[1], m.prior[1].tobytes(), m.kf[1].tobytes()) == before1
    assert m.th[0] == update_fast_threshold(h, 12, r["DT"], 0.125, 70) == 17
    for f in ("Tfw", "Tfw_cov", "DT", "DT_cov", "err_norm"):
        np.testing.assert_array_equal(m.prior[0][f], r[f])
    assert m.kf[0]["N_prevKF_currF"] == 9
    m.inserted(0, r, after, new_kf=True)   # currFrameIsKF: the next prior's Tfw, Tfw_cov reset
    np.testing.assert_array_equal(m.prior[0]["Tfw"], np.eye(4))
    np.testing.assert_array_equal(m.prior[0]["Tfw_cov"], np.eye(6))
    np.testing.assert_array_equal(m.prior[0]["DT"], r["DT"])
    m.initialize(0, 25)   # what HandlerState's initialize leaves
    assert m.th[0] == 25
    assert m.prior[0].tobytes() == fresh_prior()[0].tobytes()
    assert m.kf[0].tobytes() == KeyframeTest().to_state()[0].tobytes()
    assert (m.th[1], m.prior[1].tobytes(), m.kf[1].tobytes()) == before1
    # the fresh prior is priorOf of a freshly initialised frame, as the library's initial key-frame state is initialize()'s
    p = fresh_prior()[0]
    assert np.array_equal(p["Tfw"], np.eye(4)) and np.array_equal(p["Tfw_cov"], np.eye(6))
    assert np.array_equal(p["DT"], np.eye(4)) and not p["DT_cov"].any() and p["err_norm"] == -1.0
    s = np.zeros(1, T.KEYFRAME_STATE_DTYPE)
    load_library().plstvo_initial_keyframe_state(s.ctypes.data)
    assert s.tobytes() == KeyframeTest().to_state().tobytes()
    # no priors: every stream starts from the fresh prior; no key-frame state: none is carried
    m2 = ScheduleStreams(h, [5, 6, 7])
    assert m2.kf is None and all(m2.prior[k].tobytes() == p.tobytes() for k in range(3))


def build_schedule_example(tmp_path):
    exe = str(tmp_path / "schedule_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "schedule_cpp.cpp"), "-L", LIBDIR, "-lplstvo_b200",
                    f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    return exe


def test_schedule_example_compiles(tmp_path):
    assert os.path.exists(build_schedule_example(tmp_path))
