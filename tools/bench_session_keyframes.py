"""What the key-frame test costs inside plstvo_stereo_session_run_keyframes: the run with the test against the plain
plstvo_stereo_session_run on twin sessions, and (up to --loop-max-s streams) against the per-frame insert loop with the host
KeyframeTest and currFrameIsKF's prior reset.  The arms alternate rep by rep in one process on one context.  Each rep checks
that the run with the test equals the loop (results, n_stereo, thresholds and decisions) and equals the plain run up to the
first key frame (after it the priors differ by design).  Prints one JSON line per workload: wall ms per frame (median, min,
max over the reps; every arm returns synchronised), stage [4] (tracking and the handler / key-frame update) of both runs,
the key frames found, and a retained run's key-frame chunk bytes against the header's count (96 B per stereo point and 176 B
per stereo line of every step); with the card's name and power limit read in the same process.
  KITTI size (1241x376) moving grey views, shipped ORB (1200 features, 4 levels) and LSD options, KITTI handler config,
  default key-frame config; S in {1, 8, 64} streams, T = 8.

    python tools/bench_session_keyframes.py --gpus 1
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_stereo_session import card  # noqa: E402
from stvo_pl_b200 import types as T  # noqa: E402
from stvo_pl_b200.engine import Engine  # noqa: E402
from stvo_pl_b200.handler import HandlerConfig, KeyframeTest, update_fast_threshold  # noqa: E402


def stats(v):
    return dict(median=float(np.median(v)), min=float(min(v)), max=float(max(v)))


def priors_of(res):
    p = np.zeros(len(res), T.PRIOR_DTYPE)
    for k in ("Tfw", "Tfw_cov", "DT", "DT_cov", "err_norm"):
        p[k] = res[k]
    return p


def views(S, NF, W, H, seed):
    from test_gpu_track_images import moving_views
    out = []
    for s in range(S):
        d = moving_views(NF, W, H, seed + 13 * s, 0)
        out.append(dict(img_l=d["img_l"], img_r=d["img_r"]))
    return out


def colour(st):
    """BGR frames whose channels differ by a few levels, so that the grey image cvtColor gives keeps the texture's contrast
    (grey = d - 2 or so)."""
    out = []
    for d in st:
        out.append({k: np.clip(np.stack([d[k].astype(np.int16) + 12, d[k], d[k].astype(np.int16) - 12], -1), 0, 255)
                    .astype(np.uint8) for k in ("img_l", "img_r")})
    return out


class _Frame:
    pass


def loop(ss, h, th0, ids, frames, T_):
    """The per-frame loop with the host key-frame test: (results, thresholds, n_stereo, decisions [T, n])."""
    n = len(ids)
    kts = [KeyframeTest() for _ in range(n)]
    th, pri, res_all, ns_all, rows, kfs = th0.copy(), None, [], [], [th0.copy()], []
    for t in range(T_):
        fr = dict(img_l=frames["img_l"][t * n:(t + 1) * n], img_r=frames["img_r"][t * n:(t + 1) * n], fast_th=th)
        res, ns = ss.insert(ids, fr, pri)
        th = np.int32([update_fast_threshold(h, int(th[k]), res[k]["DT"], float(res[k]["err_norm"]),
                                             int(res[k]["n_inliers_pt"])) for k in range(n)])
        fire = [kts[k].needNewKF(h, res[k]["Tfw"], res[k]["DT"], res[k]["DT_cov"]) for k in range(n)]
        pri = priors_of(res)
        for k in range(n):
            if fire[k]:
                kts[k].currFrameIsKF(_Frame())
                pri["Tfw"][k], pri["Tfw_cov"][k] = np.eye(4), np.eye(6)
        res_all.append(res.copy())
        ns_all.append(ns.copy())
        rows.append(th.copy())
        kfs.append(fire)
    return np.stack(res_all), np.stack(rows), np.stack(ns_all), np.int32(kfs)


def workload(e, cfgs, cam, st, S, T_, reps, with_loop):
    """Arms on twin sessions, alternated rep by rep: kf (run_keyframes), plain (run) and, with_loop, the per-frame loop with
    the host test.  Then one retained run_keyframes: its device bytes against the header's count."""
    tc, mc, sc, oc, lc = cfgs
    h = HandlerConfig(fast_min_th=7, fast_max_th=30)   # config_kitti.yaml; key-frame thresholds src/config.cpp:40-42
    ids = np.arange(S, dtype=np.int32)
    th0 = np.full(S, 20, np.int32)
    A, B, C = (e.stereo_session_create(cam, tc, mc, sc, oc, lc, None, S) for _ in range(3))
    times = {"kf": [], "plain": [], "loop": []}
    stage = {"kf": [], "plain": []}
    n_kf = 0
    for r in range(reps):
        init = {k: np.stack([st[s % len(st)][k][0] for s in range(S)]) for k in ("img_l", "img_r")}
        for x in (A, B, C):
            x.initialize(ids, init)
        frames = {k: np.concatenate([np.stack([st[s % len(st)][k][t] for s in range(S)]) for t in range(1, T_ + 1)])
                  for k in ("img_l", "img_r")}
        arms = [("kf", lambda: A.run_keyframes(h, h, ids, T_, frames, e.initial_keyframe_state(S), th0)),
                ("plain", lambda: B.run(h, ids, T_, frames, th0))]
        if with_loop:
            arms.append(("loop", lambda: loop(C, h, th0, ids, frames, T_)))
        k = r % len(arms)
        arms = arms[k:] + arms[:k]
        out = {}
        for name, fn in arms:
            t0 = time.perf_counter()
            out[name] = fn()
            times[name].append((time.perf_counter() - t0) * 1e3 / (S * T_))
            if name in stage:
                stage[name].append(e.track_stereo_images_stage_times().tolist())
        kr, kk, kt, kn = out["kf"]
        n_kf += int(kk["new_kf"].sum())
        if with_loop:
            lr, lt, ln, lk = out["loop"]
            if not (kr.tobytes() == lr.tobytes() and np.array_equal(kt, lt) and np.array_equal(kn, ln)
                    and np.array_equal(kk["new_kf"], lk)):
                raise SystemExit(f"S={S} T={T_} rep {r}: the run with the test and the per-frame loop differ")
        # with no key frame the two runs take the same priors: compare the steps up to the first key frame
        pr, pt, pn = out["plain"]
        first = int(np.argmax(kk["new_kf"].any(1))) + 1 if kk["new_kf"].any() else T_
        if not (kr[:first].tobytes() == pr[:first].tobytes() and np.array_equal(kn[:first], pn[:first])):
            raise SystemExit(f"S={S} T={T_} rep {r}: the run with the test and the plain run differ before the first key frame")
    # one retained run: the key-frame chunks' bytes against the header's 96 B per point and 176 B per line of every step
    A.retain(True)
    A.initialize(ids, init)
    kr, kk, kt, kn = A.run_keyframes(h, h, ids, T_, frames, e.initial_keyframe_state(S), th0)
    rows, _, _ = A.read_keyframes()
    after = A.device_bytes
    A.initialize(ids, init)   # discards the key frames and frees their chunks
    chunk_bytes = after - A.device_bytes
    stated = int(kn[:, :, 2].sum()) * 96 + int(kn[:, :, 3].sum()) * 176
    res = dict(S=S, T=T_, width=cam.width, height=cam.height, key_frames=n_kf, per_frame_loop_checked=with_loop,
               kf_ms_per_frame=stats(times["kf"]), plain_ms_per_frame=stats(times["plain"]),
               kf_stage4_ms_median=float(np.median([s[4] for s in stage["kf"]])),
               plain_stage4_ms_median=float(np.median([s[4] for s in stage["plain"]])),
               retained_key_frames=int(len(rows)), retained_stated_bytes=stated, retained_chunk_bytes=int(chunk_bytes),
               reps=reps)
    if with_loop:
        res["loop_ms_per_frame"] = stats(times["loop"])
    for x in (A, B, C):
        x.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1,8,64")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--loop-max-s", type=int, default=8, help="largest S at which the per-frame loop arm runs too")
    a = ap.parse_args()
    if a.gpus != 1:
        raise SystemExit("--gpus 1 only")
    if a.reps < 3:
        raise SystemExit("--reps must be at least 3")
    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    oc, lc = T.default_orb_detect_config(1200, 4), T.default_lsd_config()
    oc.fast_threshold = 0   # as the handlers set it: every frame at the handler's threshold
    cfgs = (tc, mc, sc, oc, lc)
    name, power = card()
    head = dict(card=name, power_limit=power)
    e = Engine()
    cam = T.kitti_camera()
    st = views(8, a.steps + 1, cam.width, cam.height, 5100)   # stream s views scene s % 8
    workload(e, cfgs, cam, st, 2, 2, 3, True)   # warm-up, not reported
    for S in [int(x) for x in a.sizes.split(",")]:
        print(json.dumps(dict(head, **workload(e, cfgs, cam, st, S, a.steps, a.reps, S <= a.loop_max_s))), flush=True)
    e.close()


if __name__ == "__main__":
    main()
