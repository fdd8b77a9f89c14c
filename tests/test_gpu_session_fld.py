"""Stereo sessions on the reference's FLD line branch (plstvo_stereo_session_use_fld_lines) on the GPU.  LSD's key lines
(plstvo_lsd_detect_batch) stand in for FastLineDetector's, so a session with the switch on, fed them, must equal a plain LSD
session byte for byte: results, n_stereo, threshold rows, key-frame decisions, and _read / _read_keyframes rows, through
initialize, uneven inserts over S = 1, 37 and SMs + 5 streams, a re-initialised stream, runs (whole and split) and
run_keyframes, plain and camera-per-stream sessions (grey rigs, one NULL entry), with points or lines off.  An insert also
equals plstvo_track_stereo_images_batch with the kept frames' images and key lines as prev.  Colour sessions (BGR, BGRA, with
and without maps) equal the chain ORB on the BGR2GRAY remap, LBD on the RGB2GRAY remap (the rectify oracle and cv2's
conversion), then the stereo step.  Errors leave the session usable."""
import subprocess

import numpy as np
import pytest

from test_gpu_session_cams import colour, perturbed_maps, three_cams
from test_gpu_session_frames import assert_frames
from test_gpu_session_run import priors_of, scenes, step_major
from test_fld_keylines_host import LIBDIR, ROOT
from test_gpu_stereo_session import frames_of
from test_gpu_track_images import CAM_SMALL, configs, sm_count
from test_gpu_rectify import rig
from oracle import color as OC
from oracle import fld as OF
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError
from stvo_pl_b200.handler import HandlerConfig, update_fast_threshold

pytestmark = pytest.mark.gpu


def line_fields(e, lc, il, ir):
    """The key-line fields of frames il / ir (grey, as the session's LSD sees them): LSD's lines, frame-major."""
    n = len(il)
    if n == 0:
        return dict(ll_off=np.zeros(1, np.int32), lr_off=np.zeros(1, np.int32))
    _, kl = e.lsd_detect_batch(lc, np.concatenate([il, ir]))
    off = kl["off"]
    a, b = int(off[n]), int(off[2 * n])
    return dict(ll_off=off[:n + 1].copy(), lr_off=(off[n:] - off[n]).astype(np.int32), seg_l=kl["seg"][:a],
                seg_r=kl["seg"][a:b], angle_l=kl["angle"][:a], angle_r=kl["angle"][a:b], npix_l=kl["npix"][:a],
                npix_r=kl["npix"][a:b])


def with_lines(e, lc, frames, grey=None):
    """frames plus the key-line fields of grey (default: frames' own images)"""
    g = frames if grey is None else grey
    return dict(frames, **line_fields(e, lc, g["img_l"], g["img_r"]))


class Twins:
    """An LSD session and an FLD session with the same configs, retention on."""

    def __init__(self, e, S, points=True, lines=True, cams=False, cam=CAM_SMALL):
        self.e = e
        mc, sc, tc, oc = configs(500, 4)
        tc.has_points, tc.has_lines = int(points), int(lines)
        self.lc = T.default_lsd_config()
        self.rects = None
        if cams:
            cam, maps = rig("euroc")
            rs = [e.rectifier_create(*maps), e.rectifier_create(*perturbed_maps(1)), None]
            self.rects = [rs[s % 3] for s in range(S)]
            cs = [three_cams(cam)[s % 3] for s in range(S)]
            mk = lambda: e.stereo_session_create_cams(cs, tc, mc, sc, oc, self.lc, self.rects, S)  # noqa: E731
        else:
            mk = lambda: e.stereo_session_create(cam, tc, mc, sc, oc, self.lc, None, S)  # noqa: E731
        self.W, self.H = cam.width, cam.height
        self.lines = lines
        self.A, self.B = mk(), mk()
        self.B.use_fld_lines(True)
        for s in (self.A, self.B):
            s.retain(True)

    def grey(self, frames, ids):
        """what the sessions' LSD reads: each stream's images through its rectifier"""
        if self.rects is None:
            return frames
        out = dict(frames)
        for side in ("img_l", "img_r"):
            out[side] = frames[side].copy()
        for k, i in enumerate(list(ids) * (len(frames["img_l"]) // max(len(ids), 1))):
            r = self.rects[i]
            if r is not None:
                out["img_l"][k], out["img_r"][k] = (x[0] for x in self.e.rectify_batch(r, frames["img_l"][k:k + 1],
                                                                                      frames["img_r"][k:k + 1]))
        return out

    def fld(self, frames, ids):
        return with_lines(self.e, self.lc, frames, self.grey(frames, ids)) if self.lines else frames

    def initialize(self, ids, frames):
        a = self.A.initialize(ids, frames)
        b = self.B.initialize(ids, self.fld(frames, ids))
        np.testing.assert_array_equal(a, b)
        self.same_read()

    def insert(self, ids, frames, priors=None):
        ra, na = self.A.insert(ids, frames, priors)
        rb, nb = self.B.insert(ids, self.fld(frames, ids), priors)
        assert ra.tobytes() == rb.tobytes()
        np.testing.assert_array_equal(na, nb)
        self.same_read()
        return ra

    def same_read(self):
        a, b = self.A.read(), self.B.read()
        assert_frames(a[0], a[1], b[:2])
        for x, y in zip(a[2:], b[2:]):
            assert (x is None and y is None) or np.array_equal(x, y)


def uneven(tw, S, NF, seed):
    """initialize every stream, then inserts of random subsets with one stream re-initialised part-way"""
    st = scenes(S, NF, seed, tw.W, tw.H)
    rng = np.random.default_rng(seed)
    pos = {i: 0 for i in range(S)}
    ids = rng.permutation(S)
    tw.initialize(ids, frames_of(st, ids, pos))
    for step in range(2 * NF):
        cand = [i for i in range(S) if pos[i] + 1 < NF]
        if not cand:
            break
        ids = rng.permutation(cand)[:max(1, int(rng.integers(1, len(cand) + 1)))]
        for i in ids:
            pos[i] += 1
        if step == 1:   # a stream re-initialised mid-run
            tw.initialize(ids[:1], frames_of(st, ids[:1], pos))
            ids = ids[1:]
            if len(ids) == 0:
                continue
        tw.insert(ids, frames_of(st, ids, pos))


@pytest.mark.parametrize("S", ["1", "37", "sms+5"])
def test_inserts_equal_the_lsd_session(S):
    S = sm_count() + 5 if S == "sms+5" else int(S)
    e = Engine(0)
    uneven(Twins(e, S), S, 4 if S > 1 else 6, 700 + S)
    e.close()


@pytest.mark.parametrize("mode", ["no_points", "no_lines", "cams"])
def test_switches_and_cams(mode):
    e = Engine(0)
    S = 5
    tw = Twins(e, S, points=mode != "no_points", lines=mode != "no_lines", cams=mode == "cams")
    uneven(tw, S, 4, 900 + len(mode))
    e.close()


def test_insert_equals_the_images_call():
    """prev = each stream's kept images and key lines at their thresholds, curr = the new frames, the same priors"""
    e = Engine(0)
    S = 4
    tw = Twins(e, S)
    st = scenes(S, 3, 41)
    ids = np.arange(S)
    f0 = tw.fld(frames_of(st, ids, {i: 0 for i in ids}), ids)
    f1 = tw.fld(frames_of(st, ids, {i: 1 for i in ids}), ids)
    tw.B.initialize(ids, f0)
    pri = np.zeros(S, T.PRIOR_DTYPE)
    pri["Tfw"] = pri["DT"] = np.eye(4)
    pri["Tfw_cov"] = np.eye(6)
    pri["DT"][:, 0, 3] = 0.01
    got, ns = tw.B.insert(ids, f1, pri)
    mc, sc, tc, oc = configs(500, 4)
    want, ns_want = e.track_stereo_images_batch(CAM_SMALL, tc, mc, sc, oc, f0, f1, pri)
    assert got.tobytes() == want.tobytes()
    np.testing.assert_array_equal(ns, ns_want)
    e.close()


@pytest.mark.parametrize("S", ["3", "sms+5"])
def test_runs_equal_the_lsd_session(S):
    """run, a split run and run_keyframes with the switch on equal the LSD session's (which equal T inserts)"""
    S = sm_count() + 5 if S == "sms+5" else int(S)
    e = Engine(0)
    tw = Twins(e, S)
    st = scenes(S, 7, 1300 + S)
    ids = np.arange(S)[::-1].copy()
    tw.initialize(ids, frames_of(st, ids, {i: 0 for i in ids}))
    h = tw.e.handler_config(kitti=True)
    fa = step_major(st, ids, 1, 3)
    ra = tw.A.run(h, ids, 3, fa)
    rb = tw.B.run(h, ids, 3, tw.fld(fa, ids))
    assert ra[0].tobytes() == rb[0].tobytes()
    for x, y in zip(ra[1:], rb[1:]):
        np.testing.assert_array_equal(x, y)
    tw.same_read()
    # split: T = 1 then T = 2 on the FLD session against T = 3 on the LSD session
    fa = step_major(st, ids, 4, 3)
    th0, pri = ra[1][-1], priors_of(ra[0][-1])
    whole = tw.A.run(h, ids, 3, fa, th0, pri)
    part = lambda t0, T_: with_lines(e, tw.lc, step_major(st, ids, 4 + t0, T_))  # noqa: E731
    p1 = tw.B.run(h, ids, 1, part(0, 1), th0, pri)
    p2 = tw.B.run(h, ids, 2, part(1, 2), p1[1][-1], priors_of(p1[0][-1]))
    assert np.concatenate([p1[0], p2[0]]).tobytes() == whole[0].tobytes()
    np.testing.assert_array_equal(np.concatenate([p1[1][:1], p2[1]]), whole[1])
    np.testing.assert_array_equal(np.concatenate([p1[2], p2[2]]), whole[2])
    tw.same_read()
    e.close()


def test_run_keyframes_equals_the_lsd_session():
    e = Engine(0)
    S = 6
    tw = Twins(e, S)
    st = scenes(S, 6, 1700)
    ids = np.arange(S)
    tw.initialize(ids, frames_of(st, ids, {i: 0 for i in ids}))
    h = e.handler_config(kitti=True)
    k = e.keyframe_config()
    k["max_kf_t_dist"] = 0.02   # fires on some steps
    sa, sb = e.initial_keyframe_state(S), e.initial_keyframe_state(S)
    fa = step_major(st, ids, 1, 5)
    ra = tw.A.run_keyframes(h, k, ids, 5, fa, sa)
    rb = tw.B.run_keyframes(h, k, ids, 5, tw.fld(fa, ids), sb)
    assert ra[0].tobytes() == rb[0].tobytes() and ra[1].tobytes() == rb[1].tobytes()
    for x, y in zip(ra[2:], rb[2:]):
        np.testing.assert_array_equal(x, y)
    assert sa.tobytes() == sb.tobytes()
    ka, kb = tw.A.read_keyframes(), tw.B.read_keyframes()
    np.testing.assert_array_equal(ka[0], kb[0])
    assert_frames(ka[1], ka[2], kb[1:])
    tw.same_read()
    e.close()


# ---- colour: ORB on the BGR2GRAY remap, LBD on the RGB2GRAY remap ----
def colour_chain(e, cam, tc, mc, sc, oc, maps, frames, lines, th=None):
    """(pt, ls) of a read: the chain on the host images (the rectify oracle and cv2's conversions) and the feature calls;
    th [n]: each frame's FAST threshold (default oc's)"""
    def grey(img, rgb, side):
        m = (None, None) if maps is None else (maps[2 * side], maps[2 * side + 1])
        return np.stack([(OF.remap_gray_rgb if rgb else OC.remap_gray)(x, *m) for x in img])
    n = len(frames["img_l"])
    bgr = np.concatenate([grey(frames["img_l"], False, 0), grey(frames["img_r"], False, 1)])
    rgb = np.concatenate([grey(frames["img_l"], True, 0), grey(frames["img_r"], True, 1)])
    th = np.full(n, oc.fast_threshold, np.int32) if th is None else np.int32(th)
    _, orb = e.orb_detect_and_compute_batch(oc, bgr, np.concatenate([th, th]))
    off = orb["off"]
    a, b = int(off[n]), int(off[2 * n])
    _, dp = e.match_stereo_points(cam, mc, sc, off[:n + 1], orb["xy"][:a], orb["octave"][:a], orb["desc"][:a], off[n:] - off[n],
                                  orb["xy"][a:b], orb["desc"][a:b])
    loff = np.concatenate([lines["ll_off"], lines["lr_off"][1:] + lines["ll_off"][-1]]).astype(np.int32)
    seg = np.concatenate([lines["seg_l"], lines["seg_r"]])
    desc = e.lbd_compute_batch(rgb, loff, seg, np.concatenate([lines["angle_l"], lines["angle_r"]]),
                               np.concatenate([lines["npix_l"], lines["npix_r"]]))
    c = int(loff[n])
    _, dl = e.match_stereo_lines(cam, mc, sc, loff[:n + 1], seg[:c], lines["angle_l"], np.zeros(c, np.int32), desc[:c],
                                 loff[n:] - loff[n], seg[c:], desc[c:])
    out = []
    for o, d in ((off, dp), (loff, dl)):
        del d["m12"]
        rows = np.concatenate([np.arange(o[f], o[f] + d["counts"][f]) for f in range(n)]).astype(np.int64)
        out.append({k: v if k == "counts" else v[rows] for k, v in d.items()})
    return out


@pytest.mark.parametrize("channels,with_maps", [(3, True), (4, True), (3, False), (4, False)])
def test_colour_sessions_read_lbd_on_rgb2gray(channels, with_maps):
    e = Engine(0)
    cam, maps = rig("kitti")   # a rig whose remapped scenes keep stereo lines
    mc, sc, tc, oc = configs(500, 4)
    rect = e.rectifier_create_color(cam.width, cam.height, channels, *(maps if with_maps else ()))
    ss = e.stereo_session_create(cam, tc, mc, sc, oc, T.default_lsd_config(), rect, 2)
    ss.use_fld_lines(True)
    ss.retain(True)
    st = [colour(d, s) for s, d in enumerate(scenes(2, 2, 77, cam.width, cam.height))]
    if channels == 4:
        for d in st:
            for k in ("img_l", "img_r"):
                d[k] = np.concatenate([d[k], np.full(d[k].shape[:-1] + (1,), 99, np.uint8)], -1)
    ids = np.array([1, 0])
    for f in range(2):
        fr = frames_of(st, ids, {0: f, 1: f})
        fr["fast_th"] = None
        bgr_l, bgr_r = e.rectify_batch(rect, fr["img_l"], fr["img_r"])   # lines on the BGR grey copy: any lines will do
        lines = line_fields(e, T.default_lsd_config(), bgr_l, bgr_r)
        if f == 0:
            ss.initialize(ids, dict(fr, **lines))
        else:
            ss.insert(ids, dict(fr, **lines))
        got = ss.read()
        want = colour_chain(e, cam, tc, mc, sc, oc, maps if with_maps else None, fr, lines)
        assert_frames(got[0], got[1], want)
        assert got[1]["counts"].sum() > 0
    e.close()


# ---- errors ----
def test_errors_leave_the_session_usable():
    e = Engine(0)
    tw = Twins(e, 2)
    st = scenes(2, 3, 55)
    ids = np.arange(2)
    good = tw.fld(frames_of(st, ids, {0: 0, 1: 0}), ids)

    def bad(code, **kw):
        f = dict(good, **kw)
        with pytest.raises(PlstvoError) as ex:
            tw.B.initialize(ids, f)
        assert ex.value.code == code

    bad(-1, ll_off=None)                                       # missing
    bad(-1, seg_r=None)
    off = good["ll_off"].copy()
    off[1], off[2] = off[2], off[1]
    if off[1] != off[2]:
        bad(-1, ll_off=off)                                    # decreasing
    npix = good["npix_l"].copy()
    npix[0] = 0
    bad(-1, npix_l=npix)                                       # numOfPixels 0
    tw.B.initialize(ids, good)                                 # still usable
    with pytest.raises(PlstvoError):
        tw.B.use_fld_lines(False)                              # a stream holds a frame
    with pytest.raises(PlstvoError):
        tw.B.run(e.handler_config(), ids, 1, step_major(st, ids, 1, 1))   # a run without its lines
    nxt = tw.fld(frames_of(st, ids, {0: 1, 1: 1}), ids)
    tw.B.insert(ids, nxt)
    # line fields where the session has no lines
    mc, sc, tc, oc = configs(500, 4)
    tc.has_lines = 0
    s2 = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, None, None, 2)
    s2.use_fld_lines(True)
    with pytest.raises(PlstvoError):
        s2.initialize(ids, good)
    s2.initialize(ids, frames_of(st, ids, {0: 0, 1: 0}))
    s2.insert(ids, frames_of(st, ids, {0: 1, 1: 1}))
    e.close()


def cat_reads(parts):
    return [{k: np.concatenate([p[j][k] for p in parts]) for k in parts[0][j]} for j in range(2)]


def add_alpha(st):
    for d in st:
        for k in ("img_l", "img_r"):
            d[k] = np.concatenate([d[k], np.full(d[k].shape[:-1] + (1,), 99, np.uint8)], -1)
    return st


@pytest.mark.parametrize("channels", [3, 4])
def test_colour_cams_session_with_a_mapless_entry(channels):
    """per-stream colour rectifiers (the table instantiations), one of them without maps: each stream's rows equal the chain
    under its own camera and maps"""
    e = Engine(0)
    cam, maps = rig("kitti")
    mc, sc, tc, oc = configs(500, 4)
    m2 = [m.copy() for m in maps]
    m2[0][..., 0] = np.clip(m2[0][..., 0].astype(np.int32) + 1, -32768, 32767).astype(np.int16)   # another unit's maps
    m2[2][..., 0] = m2[0][..., 0]
    rects = [e.rectifier_create_color(cam.width, cam.height, channels, *maps),
             e.rectifier_create_color(cam.width, cam.height, channels),
             e.rectifier_create_color(cam.width, cam.height, channels, *m2)]
    rect_maps = [maps, None, m2]
    cams = three_cams(cam)
    ss = e.stereo_session_create_cams(cams, tc, mc, sc, oc, T.default_lsd_config(), rects, 3)
    ss.use_fld_lines(True)
    ss.retain(True)
    st = [colour(d, s) for s, d in enumerate(scenes(3, 2, 91, cam.width, cam.height))]
    if channels == 4:
        st = add_alpha(st)
    ids = np.array([2, 0, 1])
    for f in range(2):
        fr = frames_of(st, ids, {0: f, 1: f, 2: f})
        fr["fast_th"] = None
        per, lines_all = [], []
        for k, i in enumerate(ids):
            one = {key: fr[key][k:k + 1] for key in ("img_l", "img_r")}
            gl, gr = e.rectify_batch(rects[i], one["img_l"], one["img_r"])
            lines_all.append(line_fields(e, T.default_lsd_config(), gl, gr))
            per.append(colour_chain(e, cams[i], tc, mc, sc, oc, rect_maps[i], one, lines_all[-1]))
        lines = {}
        for side in ("l", "r"):
            cnt = [int(x[f"l{side}_off"][-1]) for x in lines_all]
            lines[f"l{side}_off"] = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
            for key in ("seg", "angle", "npix"):
                lines[f"{key}_{side}"] = np.concatenate([x[f"{key}_{side}"] for x in lines_all])
        (ss.initialize if f == 0 else ss.insert)(ids, dict(fr, **lines))
        got = ss.read()
        assert_frames(got[0], got[1], cat_reads(per))
        assert got[1]["counts"].sum() > 0
    e.close()


def test_colour_run_equals_inserts_and_the_chain():
    """a colour FLD run (LBD on the run's RGB2GRAY plane) equals T inserts with the host's threshold and prior updates on a
    twin session, and its last step's frames equal the host chain at that step's thresholds"""
    e = Engine(0)
    cam, maps = rig("kitti")
    mc, sc, tc, oc = configs(500, 4)
    oc.fast_threshold = 0
    rect = e.rectifier_create_color(cam.width, cam.height, 3, *maps)
    A, B = (e.stereo_session_create(cam, tc, mc, sc, oc, T.default_lsd_config(), rect, 3) for _ in range(2))
    for s in (A, B):
        s.use_fld_lines(True)
        s.retain(True)
    S, T_ = 3, 3
    st = [colour(d, s) for s, d in enumerate(scenes(S, T_ + 1, 313, cam.width, cam.height))]
    ids = np.array([1, 2, 0])

    def lines_of(fr):
        gl, gr = e.rectify_batch(rect, fr["img_l"], fr["img_r"])
        return line_fields(e, T.default_lsd_config(), gl, gr)

    f0 = frames_of(st, ids, {i: 0 for i in ids})
    f0["fast_th"] = np.full(S, 20, np.int32)
    for s in (A, B):
        s.initialize(ids, dict(f0, **lines_of(f0)))
    h = HandlerConfig(fast_min_th=7, fast_max_th=30, fast_feat_th=20)
    fr = step_major(st, ids, 1, T_)
    th0 = np.full(S, 20, np.int32)
    res, th_rows, ns = A.run(h, ids, T_, dict(fr, **lines_of(fr)), th0)
    th, pri = th0.copy(), None
    for t in range(T_):
        one = {k: fr[k][t * S:(t + 1) * S] for k in ("img_l", "img_r")}
        np.testing.assert_array_equal(th, th_rows[t])
        r, n = B.insert(ids, dict(one, fast_th=th, **lines_of(one)), pri)
        assert r.tobytes() == res[t].tobytes()
        np.testing.assert_array_equal(n, ns[t])
        th = np.int32([update_fast_threshold(h, int(th[k]), r[k]["DT"], float(r[k]["err_norm"]), int(r[k]["n_inliers_pt"]))
                       for k in range(S)])
        pri = priors_of(r)
    np.testing.assert_array_equal(th, th_rows[T_])
    a, b = A.read(), B.read()
    assert_frames(a[0], a[1], b[:2])
    last = {k: fr[k][(T_ - 1) * S:] for k in ("img_l", "img_r")}
    want = colour_chain(e, cam, tc, mc, sc, oc, maps, last, lines_of(last), th_rows[T_ - 1])
    assert_frames(a[0], a[1], want)
    assert a[1]["counts"].sum() > 0
    e.close()


def test_handler_example_fld_equals_lsd(tmp_path):
    """examples/fld_cpp.cpp: the FLD session and the FLD StereoStreamsHandler (per-frame inserts and both
    insertStereoSequences) fed LSD's segments equal their LSD twins byte for byte"""
    exe = str(tmp_path / "fld_cpp")
    subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-I", ROOT + "/include", ROOT + "/examples/fld_cpp.cpp", "-L", LIBDIR,
                    "-lplstvo_b200", f"-Wl,-rpath,{LIBDIR}", "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "the FLD session equals the LSD session" in out.stdout
    assert "the FLD handler equals the LSD handler" in out.stdout
    assert int(out.stdout.split("handler key frames ")[1].split()[0]) > 0   # the key-frame overload saw a key frame
