"""One plstvo_stereo_session_insert over S streams against the only way to track S live streams without a session:
plstvo_track_stereo_raw_images_batch over the same S (previous, new) pairs, which detects and describes the previous frames
again.  KITTI-size frames (1241x376), the shipped ORB (1200 features, 4 levels) and LSD options, S in {1, 8, 64, 256}.  The
two arms alternate in one process on one context and their outputs are compared byte for byte; the card's name and power
limit are read in the same run.  Prints one JSON line per S: call time (median, min, max over the reps), the images' PCIe bytes
per call, and the session's device memory.

    python tools/bench_stereo_session.py [--sizes 1,8,64,256] [--reps 5] [--scenes 16]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from stvo_pl_b200 import types as T  # noqa: E402
from stvo_pl_b200.engine import Engine  # noqa: E402

W, H = 1241, 376


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def scenes(n, NF, seed=3100):
    from test_gpu_track_images import moving_views
    out = []
    for s in range(n):
        d = moving_views(NF, W, H, seed + 13 * s, 0)
        out.append(dict(img_l=d["img_l"], img_r=d["img_r"]))
    return out


def frames(sc, S, k, th):
    return dict(img_l=np.stack([sc[s % len(sc)]["img_l"][k] for s in range(S)]),
                img_r=np.stack([sc[s % len(sc)]["img_r"][k] for s in range(S)]),
                fast_th=np.full(S, th, np.int32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,256")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--scenes", type=int, default=16)
    a = ap.parse_args()
    sizes = [int(x) for x in a.sizes.split(",")]
    sc_frames = scenes(a.scenes, a.reps + 1)
    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    oc, lc = T.default_orb_detect_config(1200, 4), T.default_lsd_config()
    cam = T.kitti_camera()
    name, power = card()
    e = Engine()
    for S in sizes:
        ids = np.arange(S, dtype=np.int32)
        ss = e.stereo_session_create(cam, tc, mc, sc, oc, lc, None, S)
        ss.initialize(ids, frames(sc_frames, S, 0, 20))
        # warm-up of both arms' arenas (not timed): the batch call on frames (0, 1)
        e.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, None, frames(sc_frames, S, 0, 20), frames(sc_frames, S, 1, 20))
        t_sess, t_batch = [], []
        for k in range(1, a.reps + 1):
            prev, curr = frames(sc_frames, S, k - 1, 20), frames(sc_frames, S, k, 20)
            t0 = time.perf_counter()
            got = ss.insert(ids, curr)
            t1 = time.perf_counter()
            want = e.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, None, prev, curr)
            t2 = time.perf_counter()
            if got[0].tobytes() != want[0].tobytes() or got[1].tobytes() != want[1].tobytes():
                raise SystemExit(f"S={S} rep {k}: the session's insert differs from the batch call")
            t_sess.append((t1 - t0) * 1e3)
            t_batch.append((t2 - t1) * 1e3)
        img = W * H
        print(json.dumps(dict(
            S=S, card=name, power_limit=power, reps=a.reps, identical=True,
            session_ms=dict(median=float(np.median(t_sess)), min=float(min(t_sess)), max=float(max(t_sess))),
            batch_ms=dict(median=float(np.median(t_batch)), min=float(min(t_batch)), max=float(max(t_batch))),
            speedup=float(np.median(t_batch) / np.median(t_sess)),
            session_h2d_image_bytes=2 * S * img, batch_h2d_image_bytes=4 * S * img,
            session_device_bytes=ss.device_bytes)), flush=True)
        e.stereo_session_destroy(ss)
    e.close()


if __name__ == "__main__":
    main()
