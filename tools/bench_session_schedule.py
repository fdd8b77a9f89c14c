"""What one plstvo_stereo_session_run_schedule saves against the per-frame insert chain it equals, on streams that drop
frames: per step, one plstvo_stereo_session_insert of the streams that have a frame, the FAST threshold and the prior
carried on the host (handler.ScheduleStreams).  Both arms run in one process on one context, alternating rep by rep on twin
sessions initialised from the same frames, on the same frames and drop pattern; each rep checks that the two arms' results,
n_stereo and threshold rows are byte-identical.  Prints one JSON line per workload: wall ms per present frame (median, min,
max over the reps; both arms return synchronised), the scheduled run's stage times (plstvo_track_stereo_images_stage_times),
and the card's name and power limit read in the same process.
  KITTI size (1241x376) moving grey views, shipped ORB (1200 features, 4 levels) and LSD options, KITTI handler config, as
  tools/bench_session_run.py; S in {1, 8} streams, T in {8, 32} steps, each entry dropped with probability 0 %, 5 % or 20 %
  (seeded; a drop rate of 0 is the dense run's workload).

    python tools/bench_session_schedule.py --gpus 1
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

from bench_session_run import stats, views  # noqa: E402
from bench_stereo_session import card  # noqa: E402
from stvo_pl_b200 import types as T  # noqa: E402
from stvo_pl_b200.engine import Engine  # noqa: E402
from stvo_pl_b200.handler import HandlerConfig, ScheduleStreams, schedule_frames  # noqa: E402


def chain(ss, h, th0, ids, sched, frames):
    """Per step, one insert of the streams with a frame: (results [T, n], thresholds [T + 1, n], n_stereo [T, n, 4])"""
    T_, n = sched.shape
    m = ScheduleStreams(h, th0)
    res_all = np.zeros((T_, n), T.POSE_RESULT_DTYPE)
    rows = np.zeros((T_ + 1, n), np.int32)
    ns_all = np.zeros((T_, n, 4), np.int32)
    b = 0
    for t in range(T_):
        rows[t] = m.th
        ins = np.nonzero(sched[t])[0]
        if not len(ins):
            continue
        fr = dict(img_l=frames["img_l"][b:b + len(ins)], img_r=frames["img_r"][b:b + len(ins)], fast_th=m.th[ins].copy())
        b += len(ins)
        res, ns = ss.insert(ids[ins], fr, m.prior[ins].copy())
        res_all[t, ins] = res
        ns_all[t, ins] = ns
        for k, r in zip(ins, res):
            m.inserted(k, r)
    rows[T_] = m.th
    return res_all, rows, ns_all


def workload(e, cfgs, cam, st, S, T_, rate, reps):
    tc, mc, sc, oc, lc = cfgs
    h = HandlerConfig(fast_min_th=7, fast_max_th=30)   # config_kitti.yaml
    ids = np.arange(S, dtype=np.int32)
    th0 = np.full(S, 20, np.int32)
    rng = np.random.default_rng(1000 * S + T_ + int(rate * 100))
    sched = (rng.random((T_, S)) >= rate).astype(np.uint8)
    present = int(sched.sum())
    frames = schedule_frames(sched, lambda t, k: {key: st[k % len(st)][key][t + 1][None] for key in ("img_l", "img_r")})
    A = e.stereo_session_create(cam, tc, mc, sc, oc, lc, None, S)
    B = e.stereo_session_create(cam, tc, mc, sc, oc, lc, None, S)
    t_sched, t_chain, stage = [], [], []
    for r in range(reps):
        init = {k: np.stack([st[s % len(st)][k][0] for s in range(S)]) for k in ("img_l", "img_r")}
        A.initialize(ids, init)
        B.initialize(ids, init)
        arms = [("schedule", lambda: A.run_schedule(h, ids, sched, frames, th0)),
                ("chain", lambda: chain(B, h, th0, ids, sched, frames))]
        if r % 2:
            arms.reverse()
        out = {}
        for name, fn in arms:
            t0 = time.perf_counter()
            out[name] = fn()
            ms = (time.perf_counter() - t0) * 1e3 / max(present, 1)
            (t_sched if name == "schedule" else t_chain).append(ms)
            if name == "schedule":
                stage.append(e.track_stereo_images_stage_times().tolist())
        (r1, th1, n1), (r2, th2, n2) = out["schedule"], out["chain"]
        if not (r1.tobytes() == r2.tobytes() and np.array_equal(th1, th2) and np.array_equal(n1, n2)):
            raise SystemExit(f"S={S} T={T_} rate={rate} rep {r}: the scheduled run and the insert chain differ")
    res = dict(S=S, T=T_, drop_rate=rate, present_frames=present, width=cam.width, height=cam.height, byte_identical=True,
               schedule_ms_per_frame=stats(t_sched), chain_ms_per_frame=stats(t_chain),
               schedule_stage_ms_median=[float(np.median([s[k] for s in stage])) for k in range(5)], reps=reps)
    A.close()
    B.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1,8")
    ap.add_argument("--steps", default="8,32")
    ap.add_argument("--rates", default="0,0.05,0.2")
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
    steps = [int(x) for x in a.steps.split(",")]
    st = views(8, max(steps) + 1, cam.width, cam.height, 5100)   # stream s views scene s % 8
    workload(e, cfgs, cam, st, 2, 2, 0.2, 1)   # warm-up, not reported
    for S in (int(x) for x in a.sizes.split(",")):
        for T_ in steps:
            for rate in (float(x) for x in a.rates.split(",")):
                print(json.dumps(dict(head, **workload(e, cfgs, cam, st, S, T_, rate, a.reps))), flush=True)
    e.close()


if __name__ == "__main__":
    main()
