"""Benchmark of LSD line detection (plstvo_lsd_detect_batch); prints one JSON line.

Batches of KITTI-size images (1241x376, seeded integer-only images from tests/orb_images.py) with the shipped options
(lsd_nfeatures 300).  value = images/s through the whole call (upload, kernels, the host's KeyLine step, download); the
line also carries the device time per stage (CUDA events), the card and its power limit, and two CPU arms measured in the
same run: cv2's LineSegmentDetector (4.13) plus the same KeyLine step on one host thread and on every host thread (one
image per thread, cv2's own threading off).  The CPU arms are null without cv2.  Writes nothing to the tree.

    python tools/bench_lsd.py --gpus 1 --steps 5 --warmup 1 [--images 256] [--no-cpu]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import cpu_model, host_threads  # noqa: E402
import orb_images as OI  # noqa: E402

W, H = 1241, 376
METRIC = "LSD key lines, KITTI-size images (shipped options, 300 lines each)"
UNIT = "images/s"


def make_images(n_img):
    base = np.stack([OI.make_image(W, H, 5000 + k) for k in range(16)])
    return np.ascontiguousarray(base[np.arange(n_img) % 16])


def cpu_arm(images, threads, reps=1):
    """cv2 LSD plus the reference's KeyLine step (the restatement's), one image per host thread; images/s."""
    try:
        import cv2
    except ImportError:
        return None
    from oracle import lsd
    cv2.setNumThreads(1)
    o = lsd.LsdOracle()

    def one(img):
        d = cv2.createLineSegmentDetector(0, 1.2, 0.6, 2.0, 22.5, 0, 0.7, 1024)
        seg = d.detect(img)[0]
        seg = np.zeros((0, 4), np.float32) if seg is None else seg.reshape(-1, 4)
        return len(o.keylines_from_segments(W, H, seg, 0.025, 300)["angle"])

    n = len(images)
    t0 = time.perf_counter()
    for _ in range(reps):
        if threads == 1:
            for img in images:
                one(img)
        else:
            with ThreadPoolExecutor(threads) as ex:
                list(ex.map(one, images))
    return n * reps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--images", type=int, default=256)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    from stvo_pl_b200 import types as T
    from stvo_pl_b200.engine import Engine
    eng = Engine(0)
    cfg = T.default_lsd_config()
    images = make_images(a.images)
    for _ in range(a.warmup):
        eng.lsd_detect_batch(cfg, images)
    times = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        total, _ = eng.lsd_detect_batch(cfg, images)
        times.append(time.perf_counter() - t0)
    stage_ms = [round(float(v), 3) for v in eng.lsd_kernel_times()]
    # small batches: the rate the images call would see per stereo pair
    small = {}
    for b in (2, 16):
        eng.lsd_detect_batch(cfg, images[:b])
        t0 = time.perf_counter()
        for _ in range(3):
            eng.lsd_detect_batch(cfg, images[:b])
        small[str(b)] = round(3 * b / (time.perf_counter() - t0), 1)
    eng.close()
    line = {"impl": "gpu", "metric": METRIC, "value": round(a.images / float(np.median(times)), 1), "unit": UNIT,
            "n_gpus": 1, "images": a.images, "lines": int(total), "median_s": round(float(np.median(times)), 4),
            "stage_ms": dict(zip(["blur_resize", "grad_seeds", "grow", "host_angles", "rect"], stage_ms)),
            "small_batch_images_per_s": small}
    if not a.no_cpu:
        n_cpu = min(len(images), 64)
        threads = host_threads()
        line["cpu_1_thread"] = cpu_arm(images[:8], 1)
        line["cpu_all_threads"] = cpu_arm(images[:n_cpu], threads, reps=2)
        line["cpu_threads"] = threads
        line["cpu"] = cpu_model()
        for k in ("cpu_1_thread", "cpu_all_threads"):
            line[k] = None if line[k] is None else round(line[k], 1)
    try:
        line["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        line["gpu"] = None
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
