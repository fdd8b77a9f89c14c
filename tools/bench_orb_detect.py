"""Benchmark of ORB detection + description (plstvo_orb_detect_and_compute_batch); prints one JSON line.

The left and right images of B KITTI-size stereo frames (1241x376), seeded integer-only images (tests/orb_images.py).
--config default: 1200 features over 4 levels (src/config.cpp); kitti: 2000 features on 1 level (config_kitti.yaml); FAST
score, threshold 20.  value = images/s through the whole call (upload, kernels, download); the line also carries the device
time per stage (CUDA events), the key points per image, the GPU with its power limit, and a CPU arm (the reference selection
plus the C description oracle on every host thread, and cv2.ORB.detectAndCompute on one thread when cv2 is importable, else
null).  Writes nothing to the tree.

    python tools/bench_orb_detect.py --gpus 1 --steps 20 --warmup 3 [--pairs 128] [--config default|kitti] [--no-cpu]
                                     [--impl reference]
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

from bench import cpu_model, host_threads  # noqa: E402
from stvo_pl_b200 import types as T  # noqa: E402
import orb_images as OI  # noqa: E402

W, H = 1241, 376
CONFIGS = {"default": dict(n_features=1200, n_levels=4), "kitti": dict(n_features=2000, n_levels=1)}
UNIT = "images/s"


def make_images(n_img):
    base = np.stack([OI.make_image(W, H, 1000 + k) for k in range(8)])
    return np.ascontiguousarray(base[np.arange(n_img) % 8])


def cpu_arm(images, p, threads):
    import ref_orb_detect as R
    n = min(len(images), max(16, 2 * threads))
    ref = R.OrbDetectRef()
    ref.detect_batch(images[:2], threads=threads, **p)
    t0 = time.perf_counter()
    ref.detect_batch(images[:n], threads=threads, **p)
    out = {"value": n / (time.perf_counter() - t0), "unit": UNIT, "cores": threads, "kind": "port", "cpu": cpu_model(),
           "sample": f"{n} images, NumPy selection + C description oracle, one image per host thread"}
    try:
        import cv2
    except ImportError:
        out["cv2"] = None
        return out
    cv2.setNumThreads(1)
    orb = cv2.ORB_create(p["n_features"], 1.2, p["n_levels"], 19, 0, 2, cv2.ORB_FAST_SCORE, 31, 20)
    t0 = time.perf_counter()
    for k in range(n):
        orb.detectAndCompute(images[k], None)
    out["cv2"] = {"value": n / (time.perf_counter() - t0), "unit": UNIT, "version": cv2.__version__,
                  "sample": f"{n} images, cv2.ORB.detectAndCompute, one thread"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="one GPU: the call is per context")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=128, help="stereo pairs per step (2 images each)")
    ap.add_argument("--config", default="default", choices=sorted(CONFIGS))
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu", action="store_true", help="skip the CPU arm")
    args = ap.parse_args()
    p = CONFIGS[args.config]
    metric = (f"ORB detectAndCompute, KITTI-size stereo images ({p['n_features']} features, {p['n_levels']} level"
              f"{'s' if p['n_levels'] > 1 else ''}, FAST score)")
    threads = host_threads()
    n_img = 2 * args.pairs
    images = make_images(n_img)
    if args.impl == "reference":
        c = cpu_arm(images, p, threads)
        print(json.dumps({"impl": "reference", "metric": metric, "value": c["value"], "unit": UNIT, "n_gpus": 0, "steps": 1,
                          "warmup": 1, "higher_is_better": True, "config": {"workload": "orb_detect", "orb": args.config},
                          "cpu_baseline": c}), flush=True)
        return 0
    import torch
    from stvo_pl_b200.engine import Engine
    eng = Engine(int(os.environ.get("LOCAL_RANK", "0")))
    cfg = T.default_orb_detect_config(p["n_features"], p["n_levels"])
    for _ in range(max(args.warmup, 1)):
        n, out = eng.orb_detect_and_compute_batch(cfg, images)
    torch.cuda.synchronize()
    stage = np.zeros(4)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        n, out = eng.orb_detect_and_compute_batch(cfg, images)
        stage += eng.orb_detect_kernel_times()
    dt = time.perf_counter() - t0
    stage /= args.steps
    dev_ms = float(stage.sum())
    line = {"metric": metric, "value": n_img * args.steps / dt, "unit": UNIT, "n_gpus": 1, "steps": args.steps,
            "warmup": max(args.warmup, 1), "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True,
            "dtype": "u8/f32", "data": "synthetic",
            "config": {"workload": "orb_detect", "orb": args.config, "pairs_per_step": args.pairs, "images_per_step": n_img,
                       "image": [W, H], "n_features": p["n_features"],
                       "levels": [OI.level_size(W, H, 1.2, l) for l in range(p["n_levels"])],
                       "keypoints_per_step": int(n), "keypoints_per_image": n / n_img},
            "kernel_ms_per_step": {"pyramid_and_blur": float(stage[0]), "fast_and_nms": float(stage[1]),
                                   "selection": float(stage[2]), "angle_and_describe": float(stage[3])},
            "device_images_per_s": n_img / (dev_ms * 1e-3),
            "e2e": {"value": n_img * args.steps / dt, "unit": UNIT, "h2d_bytes_per_step": int(images.nbytes),
                    "d2h_bytes_per_step": int(n * 48 + (n_img + 1) * 4)}}
    try:
        line["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        line["gpu"] = torch.cuda.get_device_name(0)
    if not args.no_cpu:
        line["cpu_baseline"] = cpu_arm(images, p, threads)
    print(json.dumps(line), flush=True)
    eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
