"""plstvo_stereo_session_plot / _read_plot on the GPU: every plotted image equals oracle/plot.py's plotStereoFrame over the
oracle's base image of the input frame (rectified, in BGR) and the call's own _read rows, byte for byte.  Grey sessions
with and without a rectifier, colour BGR / BGRA with and without maps, camera-per-stream sessions with a rectifier per
stream (NULL entries in a grey one), the FLD branch with caller segments that leave the image, points or lines off, frames
with no stereo feature, initialize and insert over streams named in any order, KITTI-size and 37 x 23 frames.  Plotting
changes nothing else (results, n_stereo, _read rows, launches, device memory); the error rules; and examples/plot_cpp.cpp
against read_plot.  Needs neither cv2 nor the reference sources."""
import os
import struct
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle import plot as P
from test_gpu_rectify import rig
from test_gpu_session_cams import colour, perturbed_maps, three_cams
from test_gpu_track_images import CAM_SMALL, configs, frames_slice, moving_views
from test_gpu_track_images_lsd import images_only
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, LIB_PATH, PlstvoError
from stvo_pl_b200.handler import HandlerConfig, update_fast_threshold

pytestmark = pytest.mark.gpu

E_INVALID = -1   # PLSTVO_E_INVALID


def with_alpha(frames, seed):
    rng = np.random.default_rng(seed)
    out = dict(frames)
    for k in ("img_l", "img_r"):
        a = rng.integers(0, 256, frames[k].shape[:-1] + (1,), dtype=np.uint8)
        out[k] = np.concatenate([frames[k], a], -1)
    return out


def check_plot(ss, frames, maps):
    """ss.read_plot() against the oracle: frame k's base image from frames['img_l'][k] and maps[k] (None: not remapped),
    then the circles and lines of its _read rows.  Returns the images."""
    pt, ls = ss.read()[:2]
    imgs = ss.read_plot()
    n = len(frames["img_l"])
    assert imgs.shape == (n, ss.height, ss.width, 3)
    po = np.concatenate([[0], np.cumsum(pt["counts"])])
    lo = np.concatenate([[0], np.cumsum(ls["counts"])])
    for k in range(n):
        base = P.base_image(frames["img_l"][k], maps[k])
        want = P.plot_stereo_frame(base, pt["pl"][po[k]:po[k + 1]], ls["spl"][lo[k]:lo[k + 1]], ls["epl"][lo[k]:lo[k + 1]])
        np.testing.assert_array_equal(imgs[k], want, err_msg=f"frame {k}")
    return imgs


def drive(ss, frames_per_call, maps_of):
    """initialize stream 0 with the first frame, then insert the others, checking every plot; returns the stereo counts"""
    counts = []
    for k, f in enumerate(frames_per_call):
        if k == 0:
            ns = ss.initialize([0], f)
            counts.append(ns[0])
        else:
            _, ns = ss.insert([0], f)
            counts.append(ns[0, 2:])
        check_plot(ss, f, [maps_of] * len(f["img_l"]))
    return np.array(counts)


# ---- 1. one stream, KITTI size: grey, grey rectifier, colour with and without maps, points or lines off ----
MODES = ["grey", "grey_rect", "bgr", "bgra", "bgr_maps", "bgra_maps", "no_points", "no_points_rect", "no_lines"]


@pytest.mark.parametrize("mode", MODES)
def test_one_stream(mode):
    cam, maps = rig("kitti")
    W, H = cam.width, cam.height
    fr = images_only(moving_views(4, W, H, 640, 300, fast_th=[20, 12, 20, 0]))
    channels = 4 if "bgra" in mode else 3 if "bgr" in mode else 1
    if channels > 1:
        fr = colour(fr, 7)
        if channels == 4:
            fr = with_alpha(fr, 8)
    mc, sc, tc, oc = configs(1200, 4)
    lc = T.default_lsd_config()
    if mode.startswith("no_points"):
        tc.has_points = 0
    if mode == "no_lines":
        tc.has_lines, lc = 0, None
    e = Engine()
    with_maps = mode in ("grey_rect", "bgr_maps", "bgra_maps", "no_points_rect")
    rect = None
    if channels > 1:
        rect = e.rectifier_create_color(W, H, channels, *(maps if with_maps else ()))
    elif with_maps:
        rect = e.rectifier_create(*maps)
    ss = e.stereo_session_create(cam, tc, mc, sc, oc, lc, rect, 1)
    ss.retain(True)
    ss.plot(True)
    counts = drive(ss, [frames_slice(fr, k, k + 1) for k in range(4)], maps[:2] if with_maps else None)
    if mode.startswith("no_points"):
        assert (counts[:, 0] == 0).all() and counts[:, 1].sum() > 0
    elif mode == "no_lines":
        assert (counts[:, 1] == 0).all() and counts[:, 0].sum() > 0
    else:
        assert counts.min() > 0, counts
    e.close()


# ---- 2. small frames and the FLD branch: caller segments that leave the image ----
def leaving(fr, px):
    """fr's key lines with both ends pushed px pixels outward along the segment, so most leave the image"""
    out = dict(fr)
    for s in ("l", "r"):
        seg = fr[f"seg_{s}"].astype(np.float64).reshape(-1, 4)
        d = seg[:, 2:] - seg[:, :2]
        u = d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-9)
        out[f"seg_{s}"] = np.concatenate([seg[:, :2] - px * u, seg[:, 2:] + px * u], 1).astype(np.float32)
    return out


@pytest.mark.parametrize("size", ["320x240", "101x67", "37x23"])
def test_fld_lines_leaving_the_image(size):
    """every size's odd pixel count ends each frame's base image in a partial group of 4; on the small ones every line
    meets a border (where the stereo step keeps any)"""
    W, H = (int(v) for v in size.split("x"))
    cam = CAM_SMALL if W == 320 else T.PlCamera(fx=30.0, fy=30.0, cx=18.0, cy=11.0, b=0.2, width=W, height=H)
    fr = leaving(moving_views(3, W, H, 77, 60 if W == 320 else 12), 40 if W == 320 else 25)
    mc, sc, tc, oc = configs(500, 4)
    if W < 64:
        tc.has_points = 0   # ORB's border leaves no key point on so small an image
    e = Engine()
    for channels in (1, 3):
        f = fr if channels == 1 else colour(fr, 3)
        rect = None if channels == 1 else e.rectifier_create_color(W, H, 3)
        ss = e.stereo_session_create(cam, tc, mc, sc, oc, T.default_lsd_config(), rect, 1)
        ss.use_fld_lines(True)
        ss.retain(True)
        ss.plot(True)
        counts = drive(ss, [frames_slice(f, k, k + 1) for k in range(3)], None)
        if W == 320:
            assert counts[:, 1].sum() > 0, counts
            pt, ls = ss.read()[:2]
            assert ((ls["spl"] < 0) | (ls["epl"] < 0) | (ls["spl"][:, :1] >= W) | (ls["epl"][:, :1] >= W)).any()
        ss.close()
    e.close()


def test_frames_without_stereo_features():
    """flat frames: no point, no line; the plot is the base image"""
    mc, sc, tc, oc = configs(500, 4)
    e = Engine()
    ss = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, T.default_lsd_config(), None, 2)
    ss.retain(True)
    ss.plot(True)
    fr = images_only(moving_views(2, 320, 240, 5, 60))
    fr["img_l"][1] = 90
    fr["img_r"][1] = 90
    ns = ss.initialize([1, 0], fr)
    assert tuple(ns[1]) == (0, 0) and ns[0].sum() > 0
    imgs = check_plot(ss, fr, [None, None])
    np.testing.assert_array_equal(imgs[1], P.gray2bgr(fr["img_l"][1]))
    e.close()


# ---- 3. camera-per-stream sessions, one rectifier per stream; streams in any order and any subset ----
@pytest.mark.parametrize("kind", ["grey", "bgr", "bgra"])
def test_cams_sessions(kind):
    S, NF = 5, 4
    cam, maps = rig("euroc")
    W, H = cam.width, cam.height
    cams = [three_cams(cam)[s % 3] for s in range(S)]
    e = Engine()
    pm = perturbed_maps(1)
    channels = {"grey": 1, "bgr": 3, "bgra": 4}[kind]
    if channels == 1:
        kinds = [e.rectifier_create(*maps), e.rectifier_create(*pm), None]
        rmaps = [maps[:2], pm[:2], None]
    else:
        kinds = [e.rectifier_create_color(W, H, channels, *maps), e.rectifier_create_color(W, H, channels, *pm),
                 e.rectifier_create_color(W, H, channels)]
        rmaps = [maps[:2], pm[:2], None]
    rects = [kinds[s % 3] for s in range(S)]
    mc, sc, tc, oc = configs(800, 4)
    ss = e.stereo_session_create_cams(cams, tc, mc, sc, oc, T.default_lsd_config(), rects, S)
    ss.retain(True)
    ss.plot(True)
    st = [images_only(moving_views(NF, W, H, 300 + 11 * s, 120)) for s in range(S)]
    if channels > 1:
        st = [colour(d, s) if channels == 3 else with_alpha(colour(d, s), s) for s, d in enumerate(st)]
    t = [0] * S

    def call(ids, insert):
        f = {k: np.stack([st[i][k][t[i]] for i in ids]) for k in ("img_l", "img_r")}
        if insert:
            ss.insert(ids, f)
        else:
            ss.initialize(ids, f)
        check_plot(ss, f, [rmaps[i % 3] for i in ids])
        for i in ids:
            t[i] += 1

    call([3, 0, 4, 1, 2], False)
    call([2, 4], True)
    call([1, 3, 0], True)
    call([4], False)
    call([0, 4, 2, 1, 3], True)
    e.close()


# ---- 4. plotting changes nothing else ----
def test_plotting_changes_nothing_else():
    S = 3
    mc, sc, tc, oc = configs(800, 4)
    e = Engine()
    lc = T.default_lsd_config()
    A = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)   # plotting on, then off again
    B = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)   # never
    for s in (A, B):
        s.retain(True)
    st = [images_only(moving_views(5, 320, 240, 900 + s, 80)) for s in range(S)]
    ids = [2, 0, 1]

    def frames(t):
        return {k: np.stack([st[i][k][t] for i in ids]) for k in ("img_l", "img_r")}

    def call(ss, t):
        l0 = e.launches
        out = ss.initialize(ids, frames(t)) if t == 0 else ss.insert(ids, frames(t))
        return out, e.launches - l0, ss.read()

    def same(a, b):
        if isinstance(a, dict):
            assert a.keys() == b.keys()
            for k in a:
                same(a[k], b[k])
        elif isinstance(a, (tuple, list)):
            assert len(a) == len(b)
            for x, y in zip(a, b):
                same(x, y)
        elif a is None:
            assert b is None
        else:
            np.testing.assert_array_equal(a, b)

    for t in range(5):
        A.plot(t < 3)
        a, la, ra = call(A, t)
        b, lb, rb = call(B, t)
        same(a, b)
        same(ra, rb)
        if t < 3:
            assert la == lb + 2   # the base image and the drawing
            check_plot(A, frames(t), [None] * S)
        else:
            assert la == lb
            assert A.device_bytes == B.device_bytes
    e.close()


# ---- 5. the error rules ----
def read_plot_rc(e, ss, out=True):
    buf = np.zeros(max(ss.height * ss.width * 3 * 4, 1), np.uint8)
    return e.lib.plstvo_stereo_session_read_plot(e.ctx, ss.handle, buf.ctypes.data_as(T.c_uint8_p) if out else None)


def test_errors():
    mc, sc, tc, oc = configs(500, 4)
    e = Engine()
    lc = T.default_lsd_config()
    ss = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, 2)
    fr = images_only(moving_views(6, 320, 240, 31, 60))
    one = lambda k: frames_slice(fr, k, k + 1)  # noqa: E731
    bare = lambda k: dict(img_l=fr["img_l"][k:k + 1], img_r=fr["img_r"][k:k + 1])  # noqa: E731   # a run's frames
    with pytest.raises(PlstvoError):   # plot without retention
        ss.plot(True)
    assert read_plot_rc(e, ss) == E_INVALID   # plotting off
    ss.retain(True)
    ss.plot(True)
    assert read_plot_rc(e, ss) == E_INVALID   # no call since it was turned on
    ss.initialize([0], one(0))
    check_plot(ss, one(0), [None])
    assert read_plot_rc(e, ss, out=False) == E_INVALID
    other = Engine()
    assert other.lib.plstvo_stereo_session_read_plot(other.ctx, ss.handle, np.zeros(1, np.uint8).ctypes.data_as(T.c_uint8_p)) \
        == E_INVALID and other.lib.plstvo_stereo_session_plot(other.ctx, ss.handle, 1) == E_INVALID
    other.close()
    assert e.lib.plstvo_stereo_session_plot(e.ctx, None, 1) == E_INVALID
    # a failed call discards the plot: an insert on a stream with no frame
    with pytest.raises(PlstvoError):
        ss.insert([1], one(1))
    assert read_plot_rc(e, ss) == E_INVALID
    ss.insert([0], one(1))
    check_plot(ss, one(1), [None])
    # retention off turns plotting off and frees the arena; plotting must be turned on again
    b_on = ss.device_bytes
    ss.retain(False)
    assert ss.device_bytes < b_on
    ss.retain(True)
    ss.insert([0], one(2))
    assert read_plot_rc(e, ss) == E_INVALID
    ss.plot(True)
    ss.plot(True)   # already on: stays on
    ss.insert([0], one(3))
    check_plot(ss, one(3), [None])
    # every kind of run discards the plot, a run of T = 0 too
    h = e.handler_config()
    for run in ("run0", "run", "run_keyframes", "run_schedule"):
        ss.insert([0], one(4))
        check_plot(ss, one(4), [None])
        if run == "run0":
            ss.run(h, [0], 0, dict(img_l=fr["img_l"][:0], img_r=fr["img_r"][:0]))
        elif run == "run":
            ss.run(h, [0], 1, bare(5))
        elif run == "run_keyframes":
            ss.run_keyframes(h, e.keyframe_config(), [0], 1, bare(5), e.initial_keyframe_state(1))
        else:
            ss.run_schedule(h, [0], np.ones((1, 1), np.uint8), bare(5))
        assert read_plot_rc(e, ss) == E_INVALID, run
    # plot off frees the arena and reads fail
    ss.insert([0], one(4))
    b_on = ss.device_bytes
    ss.plot(False)
    assert ss.device_bytes < b_on and read_plot_rc(e, ss) == E_INVALID
    ss.read()   # retention itself is untouched
    e.close()


# ---- 6. examples/plot_cpp.cpp (StereoImageHandler::plotFrames) against read_plot ----
def read_ppm(path):
    with open(path, "rb") as f:
        data = f.read()
    head = data.split(b"\n", 3)
    assert head[0] == b"P6" and head[2] == b"255"
    w, h = (int(v) for v in head[1].split())
    return np.frombuffer(head[3], np.uint8).reshape(h, w, 3)


def test_plot_example_equals_read_plot(tmp_path):
    NF, cam, channels = 5, T.kitti_camera(), 3
    fr = colour(images_only(moving_views(NF, cam.width, cam.height, 602, 300)), 80)
    path = tmp_path / "frames.bin"
    with open(path, "wb") as f:
        f.write(struct.pack("<iiiii", cam.width, cam.height, NF, channels, 0))
        f.write(struct.pack("<9d", cam.fx, cam.fy, cam.cx, cam.cy, cam.b, 0.0, 0.0, 0.0, 0.0))
        for k in range(NF):
            f.write(np.ascontiguousarray(fr["img_l"][k]).tobytes())
            f.write(np.ascontiguousarray(fr["img_r"][k]).tobytes())
    libdir = os.path.dirname(LIB_PATH)
    exe = str(tmp_path / "plot_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "plot_cpp.cpp"), "-L", libdir, "-lplstvo_b200", f"-Wl,-rpath,{libdir}",
                    "-o", exe], check=True)
    out = tmp_path / "out"
    out.mkdir()
    subprocess.run([exe, str(path), str(out)], capture_output=True, text=True, check=True)
    # the handler's calls on a session: initialize at orb_fast_th, then inserts at the thresholds updateFrame sets, with
    # priorOf the published frame
    e = Engine()
    rect = e.rectifier_create_color(cam.width, cam.height, channels)
    mc, sc, tc, oc = configs(1200, 4)
    hc = HandlerConfig()
    ss = e.stereo_session_create(cam, tc, mc, sc, oc, T.default_lsd_config(), rect, 1)
    ss.retain(True)
    ss.plot(True)
    th = hc.orb_fast_th
    state = dict(Tfw=np.eye(4), Tfw_cov=np.eye(6), DT=np.eye(4), DT_cov=np.zeros((6, 6)), err_norm=-1.0)
    for k in range(NF):
        f = dict(img_l=fr["img_l"][k:k + 1], img_r=fr["img_r"][k:k + 1], fast_th=np.int32([th]))
        if k == 0:
            ss.initialize([0], f)
        else:
            pri = np.zeros(1, T.PRIOR_DTYPE)
            for key, v in state.items():
                pri[key][0] = v
            res, _ = ss.insert([0], f, pri)
            r = res[0]
            state = dict(Tfw=r["Tfw"], Tfw_cov=r["Tfw_cov"], DT=r["DT"], DT_cov=r["DT_cov"], err_norm=float(r["err_norm"]))
            th = update_fast_threshold(hc, th, r["DT"], float(r["err_norm"]), int(r["n_inliers_pt"]))
        img = check_plot(ss, f, [None])[0]
        np.testing.assert_array_equal(read_ppm(out / f"plot_{k}.ppm"), img[..., ::-1], err_msg=f"frame {k}")
    e.close()
