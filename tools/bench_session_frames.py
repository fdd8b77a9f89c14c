"""What reading a session call's frames back costs: plstvo_stereo_session_insert timed three ways on the same frames, in one
process on one context, the arms alternating frame by frame: retention off, retention on without a read, and retention on
followed by plstvo_stereo_session_read of every array.  KITTI-size moving views (1241x376), the shipped ORB (1200 features,
4 levels) and LSD options, two workloads: 1 stream x 50 frames, and sm_count + 5 streams x 8 rounds (every stream in every
round, so the streamed solver is taken).  The three arms' results and n_stereo are compared byte for byte.  Prints one JSON
line per workload: each arm's insert wall time (median, min, max; a session call returns synchronised), the read's time and
bytes, the retained device bytes, and the card's name and power limit read in the same run.

    python tools/bench_session_frames.py --gpus 1
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

from bench_stereo_session import W, H, card, frames, scenes  # noqa: E402
from stvo_pl_b200 import types as T  # noqa: E402
from stvo_pl_b200.engine import Engine  # noqa: E402


def stats(v):
    return dict(median=float(np.median(v)), min=float(min(v)), max=float(max(v)))


def run(e, cam, cfgs, sc_frames, S, steps):
    """One workload: S streams, `steps` inserts after one initialize; returns its JSON record."""
    tc, mc, sc, oc, lc = cfgs
    ids = np.arange(S, dtype=np.int32)
    arms = {name: e.stereo_session_create(cam, tc, mc, sc, oc, lc, None, S) for name in ("off", "on", "on_read")}
    arms["on"].retain(True)
    arms["on_read"].retain(True)
    for ss in arms.values():
        ss.initialize(ids, frames(sc_frames, S, 0, 20))
    t = {name: [] for name in arms}
    t_read, read_bytes = [], 0
    for k in range(1, steps + 1):
        curr = frames(sc_frames, S, k, 20)
        names = list(arms)
        names = names[k % 3:] + names[:k % 3]   # rotate the order: no arm always runs first
        got = {}
        for name in names:
            t0 = time.perf_counter()
            got[name] = arms[name].insert(ids, curr)
            t1 = time.perf_counter()
            if name == "on_read":
                out = arms[name].read()
                t2 = time.perf_counter()
                t_read.append((t2 - t1) * 1e3)
                read_bytes = sum(a.nbytes for d in out[:2] for a in d.values()) + sum(a.nbytes for a in out[2:])
                t[name].append((t2 - t0) * 1e3)
            else:
                t[name].append((t1 - t0) * 1e3)
        for name in ("on", "on_read"):
            if any(x.tobytes() != y.tobytes() for x, y in zip(got[name], got["off"])):
                raise SystemExit(f"S={S} step {k}: retention arm {name} differs from retention off")
    rec = dict(streams=S, inserts=steps, identical=True,
               insert_ms={name: stats(v) for name, v in t.items()},
               read_ms=stats(t_read), read_bytes_last=int(read_bytes),
               read_GB_s_last=float(read_bytes / (t_read[-1] * 1e-3) / 1e9),
               device_bytes=dict(off=arms["off"].device_bytes, on=arms["on"].device_bytes))
    for ss in arms.values():
        e.stereo_session_destroy(ss)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="only 1: a session lives on one device")
    ap.add_argument("--frames", type=int, default=50, help="inserts of the one-stream workload")
    ap.add_argument("--rounds", type=int, default=8, help="inserts of the many-stream workload")
    ap.add_argument("--scenes", type=int, default=16)
    a = ap.parse_args()
    if a.gpus != 1:
        raise SystemExit("--gpus 1 only")
    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    oc, lc = T.default_orb_detect_config(1200, 4), T.default_lsd_config()
    cfgs = (tc, mc, sc, oc, lc)
    cam = T.kitti_camera()
    name, power = card()
    e = Engine()
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # warm-up (not timed): every arena of a 1-stream and an S-stream call
    warm = scenes(2, 2)
    run(e, cam, cfgs, warm, 1, 1)
    run(e, cam, cfgs, warm, sms + 5, 1)
    for S, steps, n_scenes in ((1, a.frames, 1), (sms + 5, a.rounds, a.scenes)):
        rec = run(e, cam, cfgs, scenes(n_scenes, steps + 1), S, steps)
        print(json.dumps(dict(card=name, power_limit=power, width=W, height=H, **rec)), flush=True)
    e.close()


if __name__ == "__main__":
    main()
