"""What one plstvo_stereo_session_run saves against the per-frame loop it equals: T inserts of a session, the FAST threshold and
the prior carried on the host between calls (handler.update_fast_threshold, priorOf).  Both arms run in one process on one
context, alternating rep by rep on twin sessions initialised from the same frames; each rep checks that the two arms'
results, n_stereo and threshold rows are byte-identical.  Prints one JSON line per workload: wall ms per frame (T S frames;
median, min, max over the reps; both arms return synchronised), the run's stage times (plstvo_track_stereo_images_stage_times),
the run session's device memory, and the card's name and power limit read in the same process.
  KITTI size (1241x376) moving grey views, shipped ORB (1200 features, 4 levels) and LSD options, KITTI handler config;
  S in {1, 8, 64} streams, T in {8, 32} frames.  A workload whose images would need more device memory than --max-gb
  (LSD's 35 bytes or so per scaled pixel, as the header states) is reported as not run.
  One colour row: EuRoC size (752x480) BGR frames (channels d + 12, d, d - 12 of a grey view d) through a colour rectifier
  with maps, S = 8, T = 8.

    python tools/bench_session_run.py --gpus 1
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
from stvo_pl_b200.handler import HandlerConfig, update_fast_threshold  # noqa: E402


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


def loop(ss, h, th0, ids, frames, T_):
    n = len(ids)
    th, pri, res_all, ns_all, rows = th0.copy(), None, [], [], [th0.copy()]
    for t in range(T_):
        fr = dict(img_l=frames["img_l"][t * n:(t + 1) * n], img_r=frames["img_r"][t * n:(t + 1) * n], fast_th=th)
        res, ns = ss.insert(ids, fr, pri)
        th = np.int32([update_fast_threshold(h, int(th[k]), res[k]["DT"], float(res[k]["err_norm"]),
                                             int(res[k]["n_inliers_pt"])) for k in range(n)])
        pri = priors_of(res)
        res_all.append(res.copy())
        ns_all.append(ns.copy())
        rows.append(th.copy())
    return np.stack(res_all), np.stack(rows), np.stack(ns_all)


def workload(e, cfgs, cam, rect, st, S, T_, reps):
    tc, mc, sc, oc, lc = cfgs
    h = HandlerConfig(fast_min_th=7, fast_max_th=30)   # config_kitti.yaml
    ids = np.arange(S, dtype=np.int32)
    th0 = np.full(S, 20, np.int32)
    A = e.stereo_session_create(cam, tc, mc, sc, oc, lc, rect, S)
    B = e.stereo_session_create(cam, tc, mc, sc, oc, lc, rect, S)
    t_run, t_loop, stage = [], [], []
    for r in range(reps):
        init = {k: np.stack([st[s % len(st)][k][0] for s in range(S)]) for k in ("img_l", "img_r")}
        A.initialize(ids, init)
        B.initialize(ids, init)
        frames = {k: np.concatenate([np.stack([st[s % len(st)][k][t] for s in range(S)]) for t in range(1, T_ + 1)])
                  for k in ("img_l", "img_r")}
        arms = [("run", lambda: A.run(h, ids, T_, frames, th0)), ("loop", lambda: loop(B, h, th0, ids, frames, T_))]
        if r % 2:
            arms.reverse()
        out = {}
        for name, fn in arms:
            t0 = time.perf_counter()
            out[name] = fn()
            ms = (time.perf_counter() - t0) * 1e3 / (S * T_)
            (t_run if name == "run" else t_loop).append(ms)
            if name == "run":
                stage.append(e.track_stereo_images_stage_times().tolist())
        (r1, th1, n1), (r2, th2, n2) = out["run"], out["loop"]
        if not (r1.tobytes() == r2.tobytes() and np.array_equal(th1, th2) and np.array_equal(n1, n2)):
            raise SystemExit(f"S={S} T={T_} rep {r}: the run and the per-frame loop differ")
    res = dict(S=S, T=T_, width=cam.width, height=cam.height, colour=rect is not None, byte_identical=True,
               run_ms_per_frame=stats(t_run), loop_ms_per_frame=stats(t_loop),
               run_stage_ms_median=[float(np.median([s[k] for s in stage])) for k in range(5)],
               session_device_bytes=A.device_bytes, reps=reps)
    A.close()
    B.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1,8,64")
    ap.add_argument("--steps", default="8,32")
    ap.add_argument("--max-gb", type=float, default=60.0, help="largest estimated image residency a workload may take")
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
    sizes, steps = [int(x) for x in a.sizes.split(",")], [int(x) for x in a.steps.split(",")]
    st = views(8, max(steps) + 1, cam.width, cam.height, 5100)   # stream s views scene s % 8
    workload(e, cfgs, cam, None, st, 2, 2, 1)   # warm-up, not reported
    scaled_px = round(cam.width * lc.scale) * round(cam.height * lc.scale)
    for S in sizes:
        for T_ in steps:
            gb = 2 * S * T_ * scaled_px * 35 / 1e9
            if gb > a.max_gb:
                print(json.dumps(dict(head, S=S, T=T_, not_run=f"about {gb:.0f} GB of images resident, over --max-gb")), flush=True)
                continue
            print(json.dumps(dict(head, **workload(e, cfgs, cam, None, st, S, T_, a.reps))), flush=True)
    from test_gpu_rectify import rig
    ecam, maps = rig("euroc")
    rect = e.rectifier_create_color(ecam.width, ecam.height, 3, *maps)
    est = colour(views(8, 9, ecam.width, ecam.height, 5300))
    print(json.dumps(dict(head, **workload(e, cfgs, ecam, rect, est, 8, 8, a.reps))), flush=True)
    e.close()


if __name__ == "__main__":
    main()
