"""Rectification speed on the GPU against cv2.remap on the host (tools/make_rectify_golden.py's EuRoC rig, 752 x 480).

  1. the remap: plstvo_rectify_batch at 1 and 256 pairs, as the remap kernel's device time (CUDA events) and as the call's
     wall time (host images in and out); cv2.remap on one host thread and on all of them, over the same images.
  2. raw images to pose: plstvo_track_stereo_raw_images_batch against cv2.remap on the host (all threads) followed by
     plstvo_track_stereo_images_lsd_batch, at 1 and 64 pairs.
Prints one JSON line per measurement, with the card and its power limit.  cv2 is optional: its rows say "not measured"
without it.

    python tools/bench_rectify.py [--reps 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def timed(fn, reps: int) -> float:
    """median wall seconds of fn() over reps runs (after one warm-up run)"""
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    from stvo_pl_b200 import types as T
    from stvo_pl_b200.engine import Engine
    from test_gpu_track_images import configs, moving_views
    import make_rectify_golden as M
    try:
        import cv2
    except ImportError:
        cv2 = None
    gpu = card()
    z = np.load(os.path.join(ROOT, "tests", "golden", "rectify.npz"))
    from stvo_pl_b200.engine import init_undistort_rectify_map

    def maps(c):
        w, h = (int(v) for v in z[f"{c}_size"])
        return init_undistort_rectify_map(int(z[f"{c}_model"]), z[f"{c}_K"], z[f"{c}_D"], z[f"{c}_R"], z[f"{c}_P"], w, h)

    (m1l, m2l), (m1r, m2r) = maps("euroc_l"), maps("euroc_r")
    W, H = 752, 480
    e = Engine()
    rect = e.rectifier_create(m1l, m2l, m1r, m2r)
    out = []
    for B in (1, 256):
        il = np.stack([M.image(100 + b, W, H) for b in range(B)])
        ir = np.stack([M.image(900 + b, W, H) for b in range(B)])
        wall = timed(lambda: e.rectify_batch(rect, il, ir), a.reps)
        kms = []
        for _ in range(a.reps):
            e.rectify_batch(rect, il, ir)
            kms.append(e.rectify_kernel_times())
        k = float(np.median(kms)) * 1e-3
        px = 2 * B * W * H
        # bytes the kernel must move per pixel: 4 (map1) + 2 (map2) + 1 (write) + at least 1 read of the source
        out.append(dict(what="remap_gpu", pairs=B, kernel_ms=k * 1e3, kernel_images_per_s=2 * B / k,
                        kernel_gb_per_s=px * 8 / k / 1e9, call_ms=wall * 1e3, call_images_per_s=2 * B / wall, card=gpu))
        for threads in (1, os.cpu_count()):
            if cv2 is None:
                out.append(dict(what="remap_cv2", pairs=B, threads=threads, result="not measured: cv2 missing"))
                continue
            cv2.setNumThreads(threads)

            def host():
                for b in range(B):
                    cv2.remap(il[b], m1l, m2l, cv2.INTER_LINEAR)
                    cv2.remap(ir[b], m1r, m2r, cv2.INTER_LINEAR)
            t = timed(host, max(3, a.reps // 4))
            out.append(dict(what="remap_cv2", pairs=B, threads=threads, ms=t * 1e3, images_per_s=2 * B / t))
    # raw images to pose
    fx, fy, cx, cy, b = z["euroc_l_cam"]
    cam = T.PlCamera(fx=fx, fy=fy, cx=cx, cy=cy, b=b, width=W, height=H)
    mc, sc, tc, oc = configs(1200, 4)
    lc = T.default_lsd_config()
    for B in (1, 64):
        fr = moving_views(B + 1, W, H, 811, 200)
        prev = dict(img_l=fr["img_l"][:B], img_r=fr["img_r"][:B], fast_th=None)
        curr = dict(img_l=fr["img_l"][1:], img_r=fr["img_r"][1:], fast_th=None)
        t_gpu = timed(lambda: e.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, rect, prev, curr), max(3, a.reps // 4))
        row = dict(what="raw_images_call", pairs=B, ms=t_gpu * 1e3, pairs_per_s=B / t_gpu, card=gpu)
        if cv2 is not None:
            cv2.setNumThreads(os.cpu_count())

            def host_then_lsd():
                rec = [dict(img_l=np.stack([cv2.remap(i, m1l, m2l, cv2.INTER_LINEAR) for i in s["img_l"]]),
                            img_r=np.stack([cv2.remap(i, m1r, m2r, cv2.INTER_LINEAR) for i in s["img_r"]]), fast_th=None)
                       for s in (prev, curr)]
                return e.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, rec[0], rec[1])
            t_host = timed(host_then_lsd, max(3, a.reps // 4))
            row.update(host_remap_then_lsd_ms=t_host * 1e3, speedup=t_host / t_gpu)
        else:
            row.update(host_remap_then_lsd_ms="not measured: cv2 missing")
        out.append(row)
    e.close()
    for r in out:
        print(json.dumps(r))


if __name__ == "__main__":
    main()
