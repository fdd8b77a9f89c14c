"""plstvo_stereo_session_retain / _read on the GPU: a session call's new frames (stereo points and lines) and an insert's
matches and inlier flags, read back.  Retention changes no result, launch count or device memory of a session that is not
retaining; every frame read equals match_stereo_points / _lines fed by that frame's own feature-level chain; the matches and
inliers equal plstvo_track_batch fed the two reads; many streams with uneven arrival; every error rule; reuse beside other
calls; and examples/frames_out_cpp.cpp (StereoImageHandler::keepFeatures feeding a features-in StereoFrameHandler).
Needs neither cv2 nor the reference sources."""
import ctypes as C
import struct
import subprocess

import numpy as np
import pytest

from test_gpu_color import colorize_frames
from test_gpu_rectify import rig
from test_gpu_stereo_session import frames_of, stream_frames
from test_gpu_track_images import CAM_SMALL, configs, frames_slice, moving_views, sm_count
from test_gpu_track_images_lsd import images_only, same
from stvo_pl_b200 import synth
from stvo_pl_b200 import types as T
from stvo_pl_b200.engine import Engine, PlstvoError

pytestmark = pytest.mark.gpu


def frame_chain(e, rect, cam, tc, mc, sc, oc, lc, frames):
    """The feature-level chain of frames (n stereo pairs): rectify_batch where there is a rectifier, ORB at each frame's
    threshold (0: oc's), LSD, LBD, then match_stereo_points / _lines on all n frames.  Returns the (pt, ls) dicts a read
    returns: the records of the survivors, and per-frame counts."""
    il, ir = frames["img_l"], frames["img_r"]
    if rect is not None:
        il, ir = e.rectify_batch(rect, il, ir)
    n = len(il)
    images = np.concatenate([il, ir])
    t = np.zeros(n, np.int32) if frames.get("fast_th") is None else np.int32(frames["fast_th"])
    t = np.where(t == 0, oc.fast_threshold, t).astype(np.int32)
    out = []
    for lines, on in ((False, tc.has_points), (True, tc.has_lines)):
        if not on:
            d = e.stereo_outputs(0, n, lines)
            del d["m12"]
            out.append(d)
            continue
        if lines:
            _, kl = e.lsd_detect_batch(lc, images)
            off = kl["off"]
            desc = e.lbd_compute_batch(images, off, kl["seg"], kl["angle"], kl["npix"])
            a, b = int(off[n]), int(off[2 * n])
            total, d = e.match_stereo_lines(cam, mc, sc, off[:n + 1], kl["seg"][:a], kl["angle"][:a], np.zeros(a, np.int32),
                                            desc[:a], off[n:] - off[n], kl["seg"][a:b], desc[a:b])
        else:
            _, orb = e.orb_detect_and_compute_batch(oc, images, np.concatenate([t, t]))
            off = orb["off"]
            a, b = int(off[n]), int(off[2 * n])
            total, d = e.match_stereo_points(cam, mc, sc, off[:n + 1], orb["xy"][:a], orb["octave"][:a], orb["desc"][:a],
                                             off[n:] - off[n], orb["xy"][a:b], orb["desc"][a:b])
        del d["m12"]
        # match_stereo_* write frame f's survivors from row off[f] on; a read holds them compact, frame after frame
        rows = np.concatenate([np.arange(off[f], off[f] + d["counts"][f]) for f in range(n)]).astype(np.int64)
        assert len(rows) == total
        out.append({k: v if k == "counts" else v[rows] for k, v in d.items()})
    return out


def assert_frames(read_pt, read_ls, want):
    for got, exp in ((read_pt, want[0]), (read_ls, want[1])):
        assert got.keys() == exp.keys()
        for k in got:
            np.testing.assert_array_equal(got[k], exp[k], err_msg=k)
            assert got[k].dtype == exp[k].dtype, k


def frame_batch(pt, ls):
    """A read's frames as a features-in FrameBatch (both roles' fields)."""
    return T.FrameBatch(pt_off=np.concatenate([[0], np.cumsum(pt["counts"])]).astype(np.int32),
                        ls_off=np.concatenate([[0], np.cumsum(ls["counts"])]).astype(np.int32),
                        pdesc=pt["desc"], ldesc=ls["desc"], pt_P=pt["P"], pt_pl=pt["pl"], pt_sigma2=pt["sigma2"],
                        ls_sP=ls["sP"], ls_eP=ls["eP"], ls_le=ls["le"], ls_spl=ls["spl"], ls_epl=ls["epl"],
                        ls_sigma2=ls["sigma2"], ls_level=ls["level"])


def identity_priors(n):
    pri = np.zeros(n, T.PRIOR_DTYPE)
    pri["Tfw"] = pri["DT"] = np.eye(4)
    pri["Tfw_cov"] = np.eye(6)
    return pri


# ---- 1. no behaviour change; 2. frames equal the chain; 3. matches equal the features-in tracker ----
MODES = ["fast", "harris", "no_points", "no_lines", "rectifier", "color"]


@pytest.mark.parametrize("mode", MODES)
def test_one_stream_frames_and_matches(mode):
    rect_rig = mode in ("rectifier", "color")
    W, H = (752, 480) if rect_rig else (1241, 376)
    th = [20, 0, 12, 35, 20, 5, 0, 50, 20]
    fr = images_only(moving_views(9, W, H, 611, 200, fast_th=th))
    mc, sc, tc, oc = configs(1200, 4, T.ORB_HARRIS_SCORE if mode == "harris" else T.ORB_FAST_SCORE)
    lc = T.default_lsd_config()
    if mode == "no_points":
        tc.has_points = 0
    if mode == "no_lines":
        tc.has_lines = 0
        lc = None
    e = Engine()
    rect, cam = None, T.kitti_camera()
    if rect_rig:
        cam, maps = rig("euroc")
        rect = e.rectifier_create(*maps) if mode == "rectifier" else e.rectifier_create_color(W, H, 3, *maps)
        if mode == "color":
            fr = colorize_frames(fr, 3, 77)
    plain, kept, toggled = (e.stereo_session_create(cam, tc, mc, sc, oc, lc, rect, 1) for _ in range(3))
    kept.retain(True)
    toggled.retain(True)
    toggled.retain(False)

    def call(ss, k, pri):
        f = frames_slice(fr, k, k + 1)
        before = e.launches
        got = ss.initialize([0], f) if k == 0 else ss.insert([0], f, pri)
        return got, e.launches - before

    prev = None
    for k in range(9):
        pri = identity_priors(1) if k % 2 else None
        (a, da), (b, db), (c, dc) = (call(ss, k, pri) for ss in (plain, kept, toggled))
        same(a, b)
        same(a, c)
        assert dc == da and db == da + 2, (da, db, dc)
        assert toggled.device_bytes == plain.device_bytes < kept.device_bytes
        pt, ls, m12_pt, inl_pt, m12_ls, inl_ls = kept.read()
        assert_frames(pt, ls, frame_chain(e, rect, cam, tc, mc, sc, oc, lc, frames_slice(fr, k, k + 1)))
        ns = a if k == 0 else a[1]
        np.testing.assert_array_equal(pt["counts"], ns[:, -2])
        np.testing.assert_array_equal(ls["counts"], ns[:, -1])
        if k == 0:
            assert m12_pt is None and inl_ls is None
        else:
            want = e.track_batch(cam, tc, frame_batch(*prev), frame_batch(pt, ls), pri)
            assert want["results"].tobytes() == a[0].tobytes()
            same((m12_pt, inl_pt, m12_ls, inl_ls), (want["m12_pt"], want["inlier_pt"], want["m12_ls"], want["inlier_ls"]))
            assert len(m12_pt) == ns[0, 0] and len(m12_ls) == ns[0, 1]
            assert ((m12_pt >= -1) & (m12_pt < max(ns[0, 2], 1))).all()
        prev = (pt, ls)
    if mode != "no_points":
        assert len(prev[0]["pl"]) > 0
    if mode in ("fast", "harris", "rectifier"):   # the colourised texture keeps few stereo points: no inlier is promised
        assert inl_pt.any()
    if mode != "no_lines":
        assert len(prev[1]["spl"]) > 0
    e.close()


# ---- 4. many streams, uneven arrival ----
@pytest.mark.parametrize("size", ["37", "sms+5"])
def test_many_streams_uneven_arrival(size):
    S = 37 if size == "37" else sm_count() + 5
    NF = 6
    st = stream_frames(S, NF, 5200 + S)
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e = Engine()
    plain = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)
    kept = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)
    kept.retain(True)
    rng = np.random.default_rng(S)
    pos = {i: 0 for i in range(S)}
    order = rng.permutation(S)
    last = {}   # each stream's last frame as read: (pt, ls) of that frame alone
    for ids in (order[:S // 3], order[S // 3:]):
        fr = frames_of(st, ids, pos)
        same(plain.initialize(ids, fr), kept.initialize(ids, fr))
        pt, ls, *_ = kept.read()
        assert_frames(pt, ls, frame_chain(e, None, CAM_SMALL, tc, mc, sc, oc, lc, fr))
        last.update(split(ids, pt, ls))
    sizes = [S, 5, S // 2, S - 2] if size == "37" else [S, 5, S - 2]
    seen_solvers = set()
    for rnd, n in enumerate(sizes):
        pool = [i for i in range(S) if pos[i] + 1 < NF]
        ids = np.int32(rng.permutation(pool)[:n])
        for i in ids:
            pos[int(i)] += 1
        fr = frames_of(st, ids, pos)
        pri = identity_priors(len(ids)) if rnd % 2 else None
        a = plain.insert(ids, fr, pri)
        same(a, kept.insert(ids, fr, pri))
        pt, ls, m12_pt, inl_pt, m12_ls, inl_ls = kept.read()
        assert_frames(pt, ls, frame_chain(e, None, CAM_SMALL, tc, mc, sc, oc, lc, fr))
        prev_pt = cat([last[int(i)][0] for i in ids])
        prev_ls = cat([last[int(i)][1] for i in ids])
        want = e.track_batch(CAM_SMALL, tc, frame_batch(prev_pt, prev_ls), frame_batch(pt, ls), pri)
        assert want["results"].tobytes() == a[0].tobytes()
        same((m12_pt, inl_pt, m12_ls, inl_ls), (want["m12_pt"], want["inlier_pt"], want["m12_ls"], want["inlier_ls"]))
        last.update(split(ids, pt, ls))
        seen_solvers.add(len(ids) > sm_count())
    if size != "37":
        assert seen_solvers == {True, False}, "both sides of the K2 / streamed policy"
    e.close()


def split(ids, pt, ls):
    """{stream id: (pt, ls) of its frame alone} from a read in call order."""
    out = {}
    op, ol = np.concatenate([[0], np.cumsum(pt["counts"])]), np.concatenate([[0], np.cumsum(ls["counts"])])
    for k, i in enumerate(ids):
        out[int(i)] = tuple({key: v[k:k + 1] if key == "counts" else v[o[k]:o[k + 1]] for key, v in d.items()}
                            for d, o in ((pt, op), (ls, ol)))
    return out


def cat(ds):
    return {k: np.concatenate([d[k] for d in ds]) for k in ds[0]}


# ---- 5. errors ----
def raw_read(e, ss, out=True, ctx=None):
    o = T.PlStereoFrameOut()
    rc = e.lib.plstvo_stereo_session_read(ctx or e.ctx, ss.handle, C.byref(o) if out else None)
    return rc, (e.lib.plstvo_last_error(ctx or e.ctx) or b"").decode()


def test_errors():
    S = 4
    st = stream_frames(S, 12, 9100)
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e, other = Engine(), Engine()
    ss = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)
    pos = {i: 0 for i in range(S)}
    ids0 = np.int32([0, 1, 2, 3])
    ss.initialize(ids0, frames_of(st, ids0, pos))
    assert raw_read(e, ss) == (-1, "retention is off: plstvo_stereo_session_retain(ctx, s, 1) first")
    ss.retain(True)
    assert raw_read(e, ss)[0] == -1 and "nothing retained" in raw_read(e, ss)[1]

    def insert_and_check(ids):
        for i in ids:
            pos[int(i)] += 1
        fr = frames_of(st, ids, pos)
        ss.insert(ids, fr)
        pt, ls, m12_pt, *_ = ss.read()
        assert_frames(pt, ls, frame_chain(e, None, CAM_SMALL, tc, mc, sc, oc, lc, fr))
        assert m12_pt is not None

    insert_and_check(np.int32([2, 0]))
    assert raw_read(e, ss, out=False)[0] == -1                       # null output
    assert raw_read(other, ss, ctx=other.ctx)[1] == "the session belongs to another context"
    with pytest.raises(PlstvoError, match="another context"):
        other._ck(other.lib.plstvo_stereo_session_retain(other.ctx, ss.handle, 0))
    assert raw_read(e, ss)[0] == 2                                   # neither touched what was retained
    # a failed call discards what was retained
    for bad in (np.int32([1, 1]), np.int32([0, 7])):
        with pytest.raises(PlstvoError):
            ss.insert(bad, frames_of(st, [0, 1], pos))
        assert raw_read(e, ss)[0] == -1 and "nothing retained" in raw_read(e, ss)[1]
        insert_and_check(np.int32([3, 1, 0]))
    with pytest.raises(PlstvoError):   # a failed initialize, too
        ss.initialize(np.int32([2, 2]), frames_of(st, [2, 2], pos))
    assert raw_read(e, ss)[0] == -1
    # after an initialize the tracker's arrays are left untouched
    pos[1] += 1
    ss.initialize(np.int32([1]), frames_of(st, [1], pos))
    m12 = np.full(4, 77, np.int32)
    inl = np.full(4, 9, np.uint8)
    o = T.PlStereoFrameOut(m12_pt=m12.ctypes.data_as(T.c_int32_p), inlier_pt=inl.ctypes.data_as(T.c_uint8_p))
    assert e.lib.plstvo_stereo_session_read(e.ctx, ss.handle, C.byref(o)) == 1
    assert (m12 == 77).all() and (inl == 9).all()
    # off frees the arena and forgets; on again needs a new call
    b_on = ss.device_bytes
    ss.retain(False)
    assert ss.device_bytes < b_on
    ss.retain(True)
    assert raw_read(e, ss)[0] == -1
    insert_and_check(np.int32([1, 2]))
    ss.retain(True)                                                   # on while on keeps the last call
    assert raw_read(e, ss)[0] == 2
    other.close()
    e.close()


# ---- 6. reuse: other calls between an insert and its read ----
def test_other_calls_do_not_disturb_the_read():
    S = 3
    st = stream_frames(S, 4, 7700)
    mc, sc, tc, oc = configs(500, 4)
    lc = T.default_lsd_config()
    e = Engine()
    ss = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)
    ss2 = e.stereo_session_create(CAM_SMALL, tc, mc, sc, oc, lc, None, S)
    ss.retain(True)
    ss2.retain(True)
    pos = {i: 0 for i in range(S)}
    ids = np.int32([2, 0, 1])
    ss.initialize(ids, frames_of(st, ids, pos))
    ss2.initialize(ids, frames_of(st, ids, pos))
    for i in ids:
        pos[int(i)] += 1
    ss.insert(ids, frames_of(st, ids, pos))
    first = ss.read()
    prev, curr, _, cam = synth.make_batch("kitti", 2)
    kv = moving_views(2, 320, 240, 77, 50)
    imgs = np.concatenate([kv["img_l"], kv["img_r"]])
    e.track_batch(cam, T.kitti_config(), prev, curr)
    e.track_stereo_images_lsd_batch(CAM_SMALL, tc, mc, sc, oc, lc, images_only(frames_slice(kv, 0, 1)),
                                    images_only(frames_slice(kv, 1, 2)))
    e.orb_detect_and_compute_batch(T.default_orb_detect_config(), imgs)
    e.lsd_detect_batch(lc, imgs)
    ss2.insert(np.int32([1]), frames_of(st, [1], {1: 3}))
    ss2.read()
    same(ss.read(), first)
    e.close()


# ---- 7. examples/frames_out_cpp.cpp: both handlers agree, and its frames equal the Python read of the same images ----
def fnv1a(a):
    h = 1469598103934665603
    for byte in np.ascontiguousarray(a).tobytes():
        h = ((h ^ byte) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def test_frames_example(tmp_path):
    W, H, NF = 640, 376, 6
    sc_ = images_only(moving_views(NF, W, H, 4321, 120))
    path = tmp_path / "frames.bin"
    rounds = [[0, 1], [2], [3, 4, 5]]
    with open(path, "wb") as f:
        f.write(struct.pack("<iiii", W, H, 1, len(rounds)))
        for rnd in rounds:
            f.write(struct.pack("<i", len(rnd)))
            for k in rnd:
                f.write(struct.pack("<i", 0))
                f.write(np.ascontiguousarray(sc_["img_l"][k]).tobytes())
                f.write(np.ascontiguousarray(sc_["img_r"][k]).tobytes())
    from test_session_frames_host import build_frames_example
    out = subprocess.run([build_frames_example(tmp_path), str(path)], capture_output=True, text=True, check=True).stdout
    rows = [line.split() for line in out.strip().splitlines()]
    frames = [r for r in rows if r[0] == "frame"]
    assert [int(r[1]) for r in frames] == list(range(NF))
    by = {}
    for r in rows:
        if r[0] != "frame" and r[0] != "kf":
            by.setdefault(r[0], []).append(r)
    for key in ("pose", "m12_pt", "m12_ls", "inlier_pt", "inlier_ls"):
        pairs = by[key]
        assert len(pairs) == 2 * (NF - 1)
        for a, b in zip(pairs[0::2], pairs[1::2]):
            assert (a[1], b[1]) == ("images", "features") and a[2:] == b[2:], key
    assert any(len(r) > 2 and "1" in r[2:] for r in by["inlier_pt"])
    # the Python read of the same images at the thresholds the handler chose
    mc, sc, tc, oc = configs(1200, 4)
    oc.fast_threshold = 0
    cam = T.kitti_camera()
    cam = T.PlCamera(fx=cam.fx, fy=cam.fy, cx=cam.cx, cy=cam.cy, b=cam.b, width=W, height=H)
    e = Engine()
    ss = e.stereo_session_create(cam, tc, mc, sc, oc, T.default_lsd_config(), None, 1)
    ss.retain(True)
    keys = list(T.FRAME_OUT_POINT_KEYS.values()) + list(T.FRAME_OUT_LINE_KEYS.values())
    for k, r in enumerate(frames):
        fr = dict(img_l=sc_["img_l"][k:k + 1], img_r=sc_["img_r"][k:k + 1], fast_th=np.int32([int(r[3])]))
        ss.initialize([0], fr) if k == 0 else ss.insert([0], fr)
        pt, ls, *_ = ss.read()
        assert [int(r[5]), int(r[6])] == [len(pt["pl"]), len(ls["spl"])]
        arrays = [pt[x] for x in keys[:7]] + [ls[x] for x in keys[7:]]
        assert [f"{fnv1a(a):016x}" for a in arrays] == r[8:], k
    e.close()
