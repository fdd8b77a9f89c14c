"""What a camera per stream costs and saves: plstvo_stereo_session_create_cams against plain sessions, in one process on one
context, the arms alternating round by round (the order rotates).  Every arm's results and n_stereo are compared stream by
stream, byte for byte.  Prints one JSON line per workload with each arm's wall time per round (median, min, max; session
calls return synchronised) and the card's name and power limit read in the same run.  Where the arms' batches fall on
different sides of the K2 / streamed policy (more pairs than SMs in one arm only), their results are not the same
computation: n_stereo is still compared, results are not ("results_compared": false).
  (a) KITTI size (1241x376), shipped ORB (1200 features, 4 levels) and LSD options: one insert of a cams session over S
      streams on K cameras (stream s on camera s % K), against K plain sessions of S / K streams each, inserted back to back.
  (b) The same size: a cams session whose S cameras are all equal against the plain session (the per-pair path's cost,
      the same bytes out).
  (c) EuRoC size (752x480): a cams session with S distinct per-stream rectifiers against one with a single shared rectifier,
      with the remap kernel's time (plstvo_rectify_kernel_times).  The maps differ, so the outputs are not compared.

    python tools/bench_session_cams.py --gpus 1
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

from bench_stereo_session import card, frames, scenes  # noqa: E402
from stvo_pl_b200 import types as T  # noqa: E402
from stvo_pl_b200.engine import Engine, init_undistort_rectify_map  # noqa: E402


def stats(v):
    return dict(median=float(np.median(v)), min=float(min(v)), max=float(max(v)))


def calibrations(cam, K):
    """K units of one camera model: fx, fy within +-3 %, cx within +-10 px, the baseline within +-10 %."""
    out = []
    for k in range(K):
        t = 0.0 if K == 1 else 2.0 * k / (K - 1) - 1.0
        out.append(T.PlCamera(fx=cam.fx * (1 + 0.03 * t), fy=cam.fy * (1 + 0.03 * t), cx=cam.cx + 10 * t, cy=cam.cy,
                              b=cam.b * (1 - 0.1 * t), width=cam.width, height=cam.height))
    return out


def timed(fn):
    t0 = time.perf_counter()
    r = fn()
    return r, (time.perf_counter() - t0) * 1e3


def split_vs_cams(e, cfgs, sc, S, K, reps, sms):
    """(a): the cams session against K plain sessions, one per camera."""
    tc, mc, scfg, oc, lc = cfgs
    cams = calibrations(T.kitti_camera(), K)
    which = np.arange(S) % K
    ids = np.arange(S, dtype=np.int32)
    groups = [ids[which == k] for k in range(K)]
    same_solver = all((len(g) > sms) == (S > sms) for g in groups)   # plan_solve's batch-size rule (GN, lists in shared memory)
    one = e.stereo_session_create_cams([cams[k] for k in which], tc, mc, scfg, oc, lc, None, S)
    many = [e.stereo_session_create(cams[k], tc, mc, scfg, oc, lc, None, len(g)) for k, g in enumerate(groups)]
    f0 = frames(sc, S, 0, 20)
    one.initialize(ids, f0)
    for ss, g in zip(many, groups):
        ss.initialize(np.arange(len(g), dtype=np.int32), {k: v[g] for k, v in f0.items()})
    t = {"cams": [], "split": []}
    for r in range(1, reps + 1):
        f = frames(sc, S, r, 20)
        arms = ["cams", "split"] if r % 2 else ["split", "cams"]
        for arm in arms:
            if arm == "cams":
                got, ms = timed(lambda: one.insert(ids, f))
            else:
                def run_split():
                    return [ss.insert(np.arange(len(g), dtype=np.int32), {k: v[g] for k, v in f.items()})
                            for ss, g in zip(many, groups)]
                parts, ms = timed(run_split)
            t[arm].append(ms)
        for (res, ns), g in zip(parts, groups):
            if got[1][g].tobytes() != ns.tobytes() or (same_solver and got[0][g].tobytes() != res.tobytes()):
                raise SystemExit(f"S={S} K={K} round {r}: the cams session differs from the plain sessions")
    for ss in [one] + many:
        e.stereo_session_destroy(ss)
    return dict(workload="a", streams=S, cameras=K, rounds=reps, identical=True, results_compared=same_solver,
                insert_ms={k: stats(v) for k, v in t.items()}, speedup_median=float(np.median(t["split"]) / np.median(t["cams"])))


def equal_cams(e, cfgs, sc, S, reps):
    """(b): all cameras equal against the plain session."""
    tc, mc, scfg, oc, lc = cfgs
    cam = T.kitti_camera()
    ids = np.arange(S, dtype=np.int32)
    arms = dict(cams=e.stereo_session_create_cams([cam] * S, tc, mc, scfg, oc, lc, None, S),
                plain=e.stereo_session_create(cam, tc, mc, scfg, oc, lc, None, S))
    for ss in arms.values():
        ss.initialize(ids, frames(sc, S, 0, 20))
    t = {k: [] for k in arms}
    for r in range(1, reps + 1):
        f = frames(sc, S, r, 20)
        got = {}
        for name in (list(arms) if r % 2 else list(arms)[::-1]):
            got[name], ms = timed(lambda: arms[name].insert(ids, f))
            t[name].append(ms)
        if any(x.tobytes() != y.tobytes() for x, y in zip(got["cams"], got["plain"])):
            raise SystemExit(f"S={S} round {r}: equal cameras differ from the plain session")
    for ss in arms.values():
        e.stereo_session_destroy(ss)
    return dict(workload="b", streams=S, rounds=reps, identical=True, insert_ms={k: stats(v) for k, v in t.items()})


def euroc_maps(n, seed=11):
    """n EuRoC-size map pairs of one pinhole model with perturbed intrinsics and distortion."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy = 458.654, 457.296, 367.215, 248.375
    D = np.array([-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05])
    P = np.array([[435.2, 0, 367.4, 0], [0, 435.2, 252.2, 0], [0, 0, 1, 0]], np.float64)
    out = []
    for _ in range(n):
        sides = []
        for _side in range(2):
            K = np.array([[fx * (1 + rng.uniform(-0.02, 0.02)), 0, cx + rng.uniform(-4, 4)],
                          [0, fy * (1 + rng.uniform(-0.02, 0.02)), cy + rng.uniform(-4, 4)], [0, 0, 1]])
            sides += list(init_undistort_rectify_map(T.RECTIFY_PINHOLE, K, D * (1 + rng.uniform(-0.1, 0.1)), np.eye(3), P,
                                                     752, 480))
        out.append(sides)
    return out


def rectifiers(e, cfgs, S, reps):
    """(c): S distinct per-stream rectifiers against one shared rectifier, EuRoC size."""
    from test_gpu_track_images import moving_views
    tc, mc, scfg, oc, lc = cfgs
    cam = T.PlCamera(fx=435.2, fy=435.2, cx=367.4, cy=252.2, b=0.11, width=752, height=480)
    maps = euroc_maps(S)
    own = [e.rectifier_create(*m) for m in maps]
    shared = own[0]
    sc = []
    for s in range(min(S, 16)):
        d = moving_views(reps + 1, 752, 480, 4100 + 7 * s, 0)
        sc.append(dict(img_l=d["img_l"], img_r=d["img_r"]))
    ids = np.arange(S, dtype=np.int32)
    arms = dict(own=e.stereo_session_create_cams([cam] * S, tc, mc, scfg, oc, lc, own, S),
                shared=e.stereo_session_create_cams([cam] * S, tc, mc, scfg, oc, lc, [shared] * S, S))
    for ss in arms.values():
        ss.initialize(ids, frames(sc, S, 0, 20))
    t = {k: [] for k in arms}
    k_ms = {k: [] for k in arms}
    for r in range(1, reps + 1):
        f = frames(sc, S, r, 20)
        for name in (list(arms) if r % 2 else list(arms)[::-1]):
            _, ms = timed(lambda: arms[name].insert(ids, f))
            t[name].append(ms)
            k_ms[name].append(e.rectify_kernel_times())
    for ss in arms.values():
        e.stereo_session_destroy(ss)
    for r in own:
        e.rectifier_destroy(r)
    return dict(workload="c", streams=S, rounds=reps, width=752, height=480, insert_ms={k: stats(v) for k, v in t.items()},
                remap_kernel_ms={k: stats(v) for k, v in k_ms.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1: a session lives on one device")
    ap.add_argument("--reps", type=int, default=5, help="timed rounds per workload (at least 3)")
    ap.add_argument("--scenes", type=int, default=16)
    ap.add_argument("--only", default="abc", help="which workloads to run")
    ap.add_argument("--sizes", default="8,64,sms+5", help="stream counts of (a) and (b)")
    a = ap.parse_args()
    if a.gpus != 1:
        raise SystemExit("--gpus 1 only")
    if a.reps < 3:
        raise SystemExit("--reps must be at least 3")
    mc, scfg, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    oc, lc = T.default_orb_detect_config(1200, 4), T.default_lsd_config()
    cfgs = (tc, mc, scfg, oc, lc)
    name, power = card()
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    e = Engine()
    sc = scenes(a.scenes, a.reps + 1)
    head = dict(card=name, power_limit=power)
    split_vs_cams(e, cfgs, sc, 8, 2, 1, sms)   # warm-up, not reported
    sizes = [sms + 5 if x == "sms+5" else int(x) for x in a.sizes.split(",")]
    if "a" in a.only:
        for S in sizes:
            for K in (2, 8):
                print(json.dumps(dict(head, **split_vs_cams(e, cfgs, sc, S, K, a.reps, sms))), flush=True)
    if "b" in a.only:
        for S in sizes:
            print(json.dumps(dict(head, **equal_cams(e, cfgs, sc, S, a.reps))), flush=True)
    if "c" in a.only:
        for S in (8, 64):
            print(json.dumps(dict(head, **rectifiers(e, cfgs, S, a.reps))), flush=True)
    e.close()


if __name__ == "__main__":
    main()
