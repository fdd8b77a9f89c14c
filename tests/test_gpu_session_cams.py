"""A camera (and a rectifier) per stream on the GPU: plstvo_track_batch_cams and plstvo_stereo_session_create_cams.
1. track_batch_cams row p equals track_batch with cam = cams[p], byte for byte, under K2 and under the streamed solver (each
   pinned in a subprocess: PLSTVO_STREAM_SOLVE is read once per process), GN and solver_mode 1, C5-size lists; all cameras
   equal: byte-equal to track_batch.
2. A cams session without rectifiers equals, stream by stream, plain sessions with that stream's camera driven through the
   same calls (results, n_stereo and every array read() returns), with uneven arrival, per-stream FAST thresholds, a stream
   re-initialised mid-run and retention on.
3. With rectifiers (grey rigs with their own maps and a NULL entry; BGR with and without maps) it equals the same session
   without them fed each stream's plstvo_rectify_batch output.
4. All cameras equal (no rectifier, one shared rectifier): byte-equal to the plain session.
5. Errors.  6. examples/cams_cpp.cpp against a Python loop of the handler rules per stream."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_track_images import CAM_SMALL, assert_same, configs, moving_views, sm_count
from test_gpu_track_images_lsd import images_only
from test_gpu_rectify import case_args, rig
from test_gpu_stereo_session import frames_of, stream_frames
from stvo_pl_b200 import synth
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError, init_undistort_rectify_map
from stvo_pl_b200.handler import HandlerConfig, KeyframeTest, update_fast_threshold

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def three_cams(cam):
    """cam and two units of its model with their own calibrations: fx, fy +-3 %, cx +-10 px, baseline +-10 %."""
    mk = lambda f, dx, b: T.PlCamera(fx=cam.fx * f, fy=cam.fy * f, cx=cam.cx + dx, cy=cam.cy, b=cam.b * b,  # noqa: E731
                                     width=cam.width, height=cam.height)
    return [mk(1.0, 0.0, 1.0), mk(1.03, 10.0, 1.1), mk(0.97, -10.0, 0.9)]


# ---- 1. track_batch_cams against track_batch per camera, each solver pinned ----
TRACK_JOB = r'''
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests")
from test_gpu_session_cams import track_cams_check
track_cams_check(int(sys.argv[2]))
print("OK")
'''


def track_cams_check(B):
    """Contract 3 at B pairs of C5-size lists, GN and solver_mode 1, in the calling process's solver setting."""
    e = Engine()
    prev, curr, _, cam = synth.make_batch("hd", B)
    cams = three_cams(cam)
    rng = np.random.default_rng(B)
    which = rng.choice(3, B, p=[0.6, 0.3, 0.1])
    which[:3] = [0, 1, 2]
    po, lo = prev.pt_off, prev.ls_off
    for mode in (0, 1):
        cfg = T.kitti_config()
        cfg.solver_mode = mode
        got = e.track_batch_cams([cams[k] for k in which], cfg, prev, curr)
        want = [e.track_batch(c, cfg, prev, curr) for c in cams]
        for p in range(B):
            w = want[which[p]]
            assert got["results"][p].tobytes() == w["results"][p].tobytes(), (mode, p, which[p])
            for key, off in (("m12_pt", po), ("inlier_pt", po), ("m12_ls", lo), ("inlier_ls", lo)):
                assert got[key][off[p]:off[p + 1]].tobytes() == w[key][off[p]:off[p + 1]].tobytes(), (mode, p, key)
        # the cameras are told apart: the anchors differ on some rows
        for k in (1, 2):
            assert (want[0]["results"]["DT"] != want[k]["results"]["DT"]).any(axis=(1, 2)).sum() > B // 2, (mode, k)
        # all cameras equal: the new instantiations against the old ones on identical values
        eq = e.track_batch_cams([cam] * B, cfg, prev, curr)
        for key in want[0]:
            assert eq[key].tobytes() == want[0][key].tobytes(), (mode, key)
    e.close()


@pytest.mark.parametrize("solver", ["k2", "streamed"])
@pytest.mark.parametrize("size", ["37", "sms+5"])
def test_track_batch_cams_equals_track_batch_per_camera(solver, size):
    B = 37 if size == "37" else sm_count() + 5
    env = {k: v for k, v in os.environ.items() if k != "PLSTVO_STREAM_SOLVE"}
    env["PLSTVO_STREAM_SOLVE"] = "0" if solver == "k2" else "1"
    r = subprocess.run([sys.executable, "-c", TRACK_JOB, ROOT, str(B)], capture_output=True, text=True, env=env, timeout=1200)
    assert r.returncode == 0 and "OK" in r.stdout, r.stderr[-3000:]


# ---- 2. sessions: the cams session against shadow plain sessions driven through the same calls ----
def frame_rows(read_out, ns, insert):
    """Per frame of the call: (point rows, line rows, m12 / inlier rows of its kept frame) of a read(), sliced by n_stereo."""
    pt, ls, m12p, inp, m12l, inl = read_out
    c = 2 if insert else 0
    out = []
    o = [0, 0, 0, 0]
    for k in range(len(ns)):
        n_p, n_l = int(ns[k, c]), int(ns[k, c + 1])
        row = {f"pt_{key}": v[o[0]:o[0] + n_p] for key, v in pt.items() if key != "counts"}
        row.update({f"ls_{key}": v[o[1]:o[1] + n_l] for key, v in ls.items() if key != "counts"})
        o[0] += n_p
        o[1] += n_l
        if insert:
            kp, kl = int(ns[k, 0]), int(ns[k, 1])
            row.update(m12_pt=m12p[o[2]:o[2] + kp], inlier_pt=inp[o[2]:o[2] + kp], m12_ls=m12l[o[3]:o[3] + kl],
                       inlier_ls=inl[o[3]:o[3] + kl])
            o[2] += kp
            o[3] += kl
        out.append(row)
    return out


class Shadows:
    """The cams session and one plain session per distinct camera, every call made on all of them; stream i's rows are
    checked against the plain session of its camera."""

    def __init__(self, e, cams, which, cfgs, rects=None, retain=True):
        self.e, self.which = e, which
        tc, mc, sc, oc, lc = cfgs
        S = len(which)
        self.ss = e.stereo_session_create_cams([cams[k] for k in which], tc, mc, sc, oc, lc, rects, S)
        self.plain = [e.stereo_session_create(c, tc, mc, sc, oc, lc, None, S) for c in cams]
        self.retain = retain
        if retain:
            for s in [self.ss] + self.plain:
                s.retain(True)

    def call(self, insert, ids, frames, shadow_frames=None, priors=None):
        ids = np.int32(ids)
        sf = frames if shadow_frames is None else shadow_frames
        if insert:
            got = self.ss.insert(ids, frames, priors)
            want = [p.insert(ids, sf, priors) for p in self.plain]
        else:
            got = (None, self.ss.initialize(ids, frames))
            want = [(None, p.initialize(ids, sf)) for p in self.plain]
        for k, i in enumerate(ids):
            w = want[self.which[i]]
            np.testing.assert_array_equal(got[1][k], w[1][k])
            if insert:
                assert got[0][k].tobytes() == w[0][k].tobytes(), (k, i)
        if self.retain:
            g = frame_rows(self.ss.read(), got[1], insert)
            ws = [frame_rows(p.read(), w[1], insert) for p, w in zip(self.plain, want)]
            for k, i in enumerate(ids):
                w = ws[self.which[i]][k]
                assert g[k].keys() == w.keys()
                for key in g[k]:
                    assert g[k][key].tobytes() == w[key].tobytes(), (k, i, key)
        return got, want

    def close(self):
        for s in [self.ss] + self.plain:
            s.close()


def drive(sh, st, S, NF, rng, shadow_of=None):
    """Uneven arrival over S streams of NF frames: two initialize calls, rounds of inserts of varying size, one stream
    re-initialised mid-run; shadow_of(frames, ids) gives the shadows' frames (default: the same)."""
    conv = shadow_of or (lambda f, ids: f)
    pos = {i: 0 for i in range(S)}
    order = rng.permutation(S)
    for ids in (order[:S // 3], order[S // 3:]):
        fr = frames_of(st, ids, pos)
        sh.call(False, ids, fr, conv(fr, ids))
    sizes = [S, 5, S // 2, S, 9, S - 2]
    cams_seen = set()
    for rnd, n in enumerate(sizes):
        pool = [i for i in range(S) if pos[i] + 1 < NF]
        ids = np.int32(rng.permutation(pool)[:max(1, min(n, len(pool)))])
        if rnd == 2 and len(ids) > 1:   # one stream starts over while the others continue
            again = np.int32([ids[-1]])
            ids = ids[:-1]
            pos[int(again[0])] += 1
            fr = frames_of(st, again, pos)
            sh.call(False, again, fr, conv(fr, again))
        for i in ids:
            pos[int(i)] += 1
        fr = frames_of(st, ids, pos)
        pri = None
        if rnd % 2:
            pri = np.zeros(len(ids), T.PRIOR_DTYPE)
            pri["Tfw"] = pri["DT"] = np.eye(4)
            pri["Tfw_cov"] = np.eye(6)
        got, _ = sh.call(True, ids, fr, conv(fr, ids), pri)
        cams_seen |= {int(sh.which[i]) for i in ids}
    return cams_seen


@pytest.mark.parametrize("size", ["37", "sms+5"])
def test_session_equals_plain_sessions_per_camera(size):
    S = 37 if size == "37" else sm_count() + 5
    st = stream_frames(S, 8, 5100 + S)
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    cams = three_cams(CAM_SMALL)
    rng = np.random.default_rng(S)
    which = rng.choice(3, S, p=[0.5, 0.3, 0.2])
    which[:3] = [0, 1, 2]
    e = Engine()
    sh = Shadows(e, cams, which, (tc, mc, sc, oc, lc))
    assert drive(sh, st, S, 8, rng) == {0, 1, 2}
    assert sh.ss.device_bytes > sh.plain[0].device_bytes - 4096   # the camera table is counted
    sh.close()
    e.close()


# ---- 3. rectifiers per stream ----
def perturbed_maps(seed):
    """The EuRoC rig with its K and D perturbed, maps from plstvo_init_undistort_rectify_map (left, right)."""
    rng = np.random.default_rng(seed)
    out = []
    for side in ("euroc_l", "euroc_r"):
        model, K, D, R, P, w, h = case_args(side)
        K = np.array(K, np.float64).copy()
        D = np.array(D, np.float64).copy()
        K.flat[0] *= 1 + rng.uniform(-0.02, 0.02)
        K.flat[4] *= 1 + rng.uniform(-0.02, 0.02)
        K.flat[2] += rng.uniform(-4, 4)
        K.flat[5] += rng.uniform(-4, 4)
        D[:2] *= 1 + rng.uniform(-0.1, 0.1, 2)
        out += list(init_undistort_rectify_map(model, K, D, R, P, w, h))
    return out


def colour(frames, seed):
    """BGR frames whose channels differ, from grey frames."""
    rng = np.random.default_rng(seed)
    out = dict(frames)
    for k in ("img_l", "img_r"):
        g = frames[k].astype(np.int16)
        off = rng.integers(-25, 26, 3)
        out[k] = np.clip(np.stack([g + off[0], 255 - g // 2 + off[1], g + off[2]], -1), 0, 255).astype(np.uint8)
    return out


def rectified(e, rects, which_rect, frames, ids):
    """What the session without rectifiers is fed: each stream's frames through plstvo_rectify_batch with its rectifier."""
    out = dict(frames)
    il, ir = [], []
    for k, i in enumerate(ids):
        r = rects[which_rect[i]]
        if r is None:
            il.append(frames["img_l"][k])
            ir.append(frames["img_r"][k])
        else:
            a, b = e.rectify_batch(r, frames["img_l"][k:k + 1], frames["img_r"][k:k + 1])
            il.append(a[0])
            ir.append(b[0])
    out["img_l"], out["img_r"] = np.stack(il), np.stack(ir)
    return out


@pytest.mark.parametrize("kind", ["grey", "bgr"])
def test_session_with_rectifiers_equals_rectify_then_session(kind):
    S, NF = 7, 6
    cam, maps = rig("euroc")
    W, H = cam.width, cam.height
    st = [images_only(moving_views(NF, W, H, 6100 + 13 * s, 0)) for s in range(S)]
    rng = np.random.default_rng(61)
    for s, d in enumerate(st):
        d["fast_th"] = rng.choice([0, 10, 20], NF).astype(np.int32)
        if kind == "bgr":
            st[s] = colour(d, s)
    mc, sc, tc, oc = configs(500, 2)
    lc = T.default_lsd_config()
    e = Engine()
    if kind == "grey":
        rects = [e.rectifier_create(*maps), e.rectifier_create(*perturbed_maps(1)), e.rectifier_create(*perturbed_maps(2)), None]
    else:
        rects = [e.rectifier_create_color(W, H, 3, *maps), e.rectifier_create_color(W, H, 3),
                 e.rectifier_create_color(W, H, 3, *perturbed_maps(3))]
    which_rect = np.arange(S) % len(rects)
    cams = three_cams(cam)
    which = np.arange(S) % 3
    tcfg = (tc, mc, sc, oc, lc)
    # the cams session with rectifiers, against the same session without them fed the rectified frames
    with_r = e.stereo_session_create_cams([cams[k] for k in which], tc, mc, sc, oc, lc, [rects[k] for k in which_rect], S)
    without = e.stereo_session_create_cams([cams[k] for k in which], tc, mc, sc, oc, lc, None, S)
    for s in (with_r, without):
        s.retain(True)
    pos = {i: 0 for i in range(S)}
    rounds = [(False, [3, 0, 5]), (False, [1, 6, 2, 4]), (True, [0, 3]), (True, [6, 5, 4, 2, 1]), (False, [2]),
              (True, [0, 1, 2, 3, 4, 5, 6]), (True, [4, 0]), (True, [6, 3, 1, 5])]
    for r, (insert, ids) in enumerate(rounds):
        ids = np.int32(ids)
        if insert or r > 1:
            for i in ids:
                pos[int(i)] += 1
        fr = frames_of(st, ids, pos)
        plain = rectified(e, rects, which_rect, fr, ids)
        if insert:
            a, b = with_r.insert(ids, fr), without.insert(ids, plain)
            assert_same(a, b)
        else:
            a, b = with_r.initialize(ids, fr), without.initialize(ids, plain)
            np.testing.assert_array_equal(a, b)
        ra, rb = with_r.read(), without.read()
        for x, y in zip(ra, rb):
            if isinstance(x, dict):
                for key in x:
                    assert x[key].tobytes() == y[key].tobytes(), (r, key)
            else:
                assert (x is None and y is None) or x.tobytes() == y.tobytes(), r
    assert e.rectify_kernel_times() > 0
    # and stream by stream, the shadows with each stream's camera fed the rectified frames
    sh = Shadows(e, cams, which, tcfg, [rects[k] for k in which_rect])
    assert drive(sh, st, S, NF, np.random.default_rng(7), lambda f, ids: rectified(e, rects, which_rect, f, ids)) == {0, 1, 2}
    sh.close()
    e.close()


# ---- 4. equal cameras: the per-pair instantiations against the uniform ones ----
@pytest.mark.parametrize("rect", ["none", "shared"])
def test_equal_cameras_equal_the_plain_session(rect):
    S, NF = 9, 6
    if rect == "none":
        cam = CAM_SMALL
        st = stream_frames(S, NF, 8100)
    else:
        cam, maps = rig("euroc")
        st = [images_only(moving_views(NF, cam.width, cam.height, 8200 + 5 * s, 0)) for s in range(S)]
        for d in st:
            d["fast_th"] = np.zeros(NF, np.int32)
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e = Engine()
    r = None if rect == "none" else e.rectifier_create(*maps)
    a = e.stereo_session_create_cams([cam] * S, tc, mc, sc, oc, lc, None if r is None else [r] * S, S)
    b = e.stereo_session_create(cam, tc, mc, sc, oc, lc, r, S)
    for s in (a, b):
        s.retain(True)
    pos = {i: 0 for i in range(S)}
    ids = np.arange(S, dtype=np.int32)
    np.testing.assert_array_equal(a.initialize(ids, frames_of(st, ids, pos)), b.initialize(ids, frames_of(st, ids, pos)))
    for rnd, ids in enumerate([np.int32([4, 0, 8, 2]), ids, np.int32([7, 1]), np.int32([3, 5, 6, 0, 8])]):
        for i in ids:
            pos[int(i)] += 1
        fr = frames_of(st, ids, pos)
        assert_same(a.insert(ids, fr), b.insert(ids, fr))
        for x, y in zip(a.read(), b.read()):
            if isinstance(x, dict):
                for key in x:
                    assert x[key].tobytes() == y[key].tobytes(), (rnd, key)
            else:
                assert x.tobytes() == y.tobytes(), rnd
    e.close()


# ---- 5. errors ----
def test_errors():
    import ctypes as C
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e, other = Engine(), Engine()
    cams = three_cams(CAM_SMALL)

    def create(cs, rects, n):
        arr = (T.PlCamera * max(len(cs), 1))(*cs) if cs is not None else None
        ra = None if rects is None else (C.c_void_p * len(rects))(*[None if x is None else x.handle for x in rects])
        h = e.lib.plstvo_stereo_session_create_cams(e.ctx, arr, C.byref(tc), C.byref(mc), C.byref(sc), C.byref(oc),
                                                    C.byref(lc), ra, n)
        msg = (e.lib.plstvo_last_error(e.ctx) or b"").decode()
        if h:
            e.lib.plstvo_stereo_session_destroy(h)
        return h, msg

    assert create(None, None, 3) == (None, "null cameras")
    assert create(cams, None, 0) == (None, "n_streams must be at least 1")
    wide = T.PlCamera(fx=300.0, fy=300.0, cx=160.0, cy=120.0, b=0.2, width=321, height=240)
    assert create(cams[:2] + [wide], None, 3) == (None, "the cameras differ in image size")
    cam, maps = rig("euroc")
    ecams = three_cams(cam)
    r_other = other.rectifier_create(*maps)
    assert create(ecams, [None, r_other, None], 3) == (None, "a rectifier belongs to another context")
    r_small = e.rectifier_create(*(np.ascontiguousarray(m[:240, :320]) for m in maps))
    assert create(ecams, [r_small, None, None], 3) == (None, "rectifier size differs from the cameras'")
    r_grey = e.rectifier_create(*maps)
    r_bgr = e.rectifier_create_color(cam.width, cam.height, 3)
    assert create(ecams, [r_grey, r_bgr, r_grey], 3) == (None, "the rectifiers differ in channel count")
    h, msg = create(ecams, [r_bgr, None, r_bgr], 3)
    assert h is None and msg.startswith("a colour session needs a colour rectifier for every stream"), msg
    with pytest.raises(PlstvoError, match="n_streams must be at least 1"):
        e.stereo_session_create_cams([], tc, mc, sc, oc, lc, None, 0)
    # the plain calls' errors: a failed insert leaves every stream as it was
    S = 4
    st = stream_frames(S, 6, 9100)
    which = np.int32([0, 1, 2, 1])
    sh = Shadows(e, cams, which, (tc, mc, sc, oc, lc))
    pos = {i: 0 for i in range(S)}
    ids = np.arange(S, dtype=np.int32)
    sh.call(False, ids, frames_of(st, ids, pos))
    for i in (0, 2):
        pos[i] += 1
    bad = frames_of(st, [0, 2], pos)
    with pytest.raises(PlstvoError, match="image size differs from the camera's"):
        sh.ss.insert([0, 2], dict(img_l=np.zeros((2, 240, 330), np.uint8), img_r=np.zeros((2, 240, 330), np.uint8)))
    with pytest.raises(PlstvoError, match="duplicate stream id"):
        sh.ss.insert([2, 2], bad)
    sh.call(True, [0, 2], bad)
    for i in (3, 1, 0):
        pos[i] += 1
    sh.call(True, [3, 1, 0], frames_of(st, [3, 1, 0], pos))
    # track_batch_cams: a null camera array
    prev, curr, _, kcam = synth.make_batch("kitti", 2)
    pc, cc = prev.as_c(), curr.as_c()
    res = np.zeros(2, T.POSE_RESULT_DTYPE)
    assert e.lib.plstvo_track_batch_cams(e.ctx, None, C.byref(tc), C.byref(pc), C.byref(cc), None, res.ctypes.data,
                                         None, None, None, None) == -1
    with pytest.raises(ValueError, match="one camera per pair"):
        e.track_batch_cams([kcam], tc, prev, curr)
    sh.close()
    other.close()
    e.close()


# ---- 6. StereoStreamsHandler with a camera per stream (examples/cams_cpp.cpp) against a Python loop ----
def test_cams_example_equals_python_loop(tmp_path):
    W, H, S = 640, 376, 3
    NF = 7
    scenes = [images_only(moving_views(NF, W, H, 1900 + 31 * s, 0)) for s in range(S)]
    rounds = [[2, 0, 1], [0, 1], [1, 0, 2], [2], [2, 0], [2, 1], [0, 2, 1], [2, 0], [1, 0, 2], [2, 1], [1], [0, 1]]
    pos = {s: 0 for s in range(S)}
    path = tmp_path / "cams.bin"
    events = []
    with open(path, "wb") as f:
        f.write(struct.pack("<iiii", W, H, S, len(rounds)))
        for rnd in rounds:
            rnd = [s for s in rnd if pos[s] < NF]
            f.write(struct.pack("<i", len(rnd)))
            for s in rnd:
                f.write(struct.pack("<i", s))
                f.write(np.ascontiguousarray(scenes[s]["img_l"][pos[s]]).tobytes())
                f.write(np.ascontiguousarray(scenes[s]["img_r"][pos[s]]).tobytes())
                events.append((s, pos[s]))
                pos[s] += 1
    from test_session_cams_host import build_cams_example
    out = subprocess.run([build_cams_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout
    rows = [line.split() for line in out.strip().splitlines()]
    mc, sc, tc, oc = configs(1200, 4)
    oc.fast_threshold = 0
    lc, hc, k = T.default_lsd_config(), HandlerConfig(), T.kitti_camera()
    fs, dx, bs = (1.0, 1.03, 0.97), (0.0, 10.0, -10.0), (1.0, 1.1, 0.9)
    cams = [T.PlCamera(fx=718.856 * fs[i], fy=718.856 * fs[i], cx=607.1928 + dx[i], cy=185.2157, b=0.537165719 * bs[i],
                       width=W, height=H) for i in range(S)]
    assert k.fx == 718.856 and k.b == 0.537165719
    e = Engine()
    state, th, prev_th, kft = {}, {}, {}, {}
    r = 0
    for s, kk in events:
        if kk == 0:
            th[s] = prev_th[s] = hc.orb_fast_th
            state[s] = dict(Tfw=np.eye(4), Tfw_cov=np.eye(6), DT=np.eye(4), DT_cov=np.zeros((6, 6)), err_norm=-1.0)
            kft[s] = KeyframeTest()
            continue
        pri = np.zeros(1, T.PRIOR_DTYPE)
        for key, v in state[s].items():
            pri[key][0] = v
        sc_ = scenes[s]
        prev = dict(img_l=sc_["img_l"][kk - 1:kk], img_r=sc_["img_r"][kk - 1:kk], fast_th=[prev_th[s]])
        curr = dict(img_l=sc_["img_l"][kk:kk + 1], img_r=sc_["img_r"][kk:kk + 1], fast_th=[th[s]])
        res, ns = e.track_stereo_images_lsd_batch(cams[s], tc, mc, sc, oc, lc, prev, curr, pri)
        x, row = res[0], rows[r]
        r += 1
        assert row[:6] == ["stream", str(s), "frame", str(kk), "th", str(th[s])], (row[:6], s, kk, th[s])
        assert [int(v) for v in row[7:11]] == list(ns[0]), (row[7:11], ns[0])
        assert int(row[12]) == x["good"]
        np.testing.assert_array_equal(np.float64(row[14:30]).reshape(4, 4), x["DT"])
        np.testing.assert_array_equal(np.float64(row[31:47]).reshape(4, 4), x["Tfw"])
        kf = kft[s].needNewKF(hc, x["Tfw"], x["DT"], x["DT_cov"])
        assert int(row[48]) == int(kf), (s, kk, row[48], kf)
        Tfw, Tfw_cov = (np.eye(4), np.eye(6)) if kf else (x["Tfw"], x["Tfw_cov"])
        if kf:
            kft[s].T_prevKF, kft[s].cov_prevKF_currF = np.eye(4), np.zeros((6, 6))
            kft[s].prev_f_iskf, kft[s].N_prevKF_currF = True, 0
        state[s] = dict(Tfw=Tfw, Tfw_cov=Tfw_cov, DT=x["DT"], DT_cov=x["DT_cov"], err_norm=float(x["err_norm"]))
        prev_th[s], th[s] = th[s], update_fast_threshold(hc, th[s], x["DT"], float(x["err_norm"]), int(x["n_inliers_pt"]))
    assert r == len(rows)
    e.close()
