"""Benchmark of ORB description (plstvo_orb_compute_batch); prints one JSON line.

The left and right images of B KITTI-size stereo frames (1241x376), seeded integer-only images (tests/orb_images.py),
1200 seeded key points per image spread over 4 levels the way ORB spreads its budget, angles computed (the
detectAndCompute half after selection).  value = images/s through the whole call (upload, kernels, download); the line also
carries the device time per stage (CUDA events), the algorithmic HBM bytes and a CPU arm (the C oracle on every host
thread, and cv2.ORB.compute when cv2 is importable, else null).  Writes nothing to the tree.

    python tools/bench_orb.py --gpus 1 --steps 20 --warmup 3 [--pairs 128] [--no-cpu] [--impl reference]
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

W, H, NKP = 1241, 376, 1200
METRIC = "ORB angles + descriptors of given key points, KITTI-size stereo images (4 levels, 1200 key points each)"
UNIT = "images/s"


def make_inputs(n_img):
    base = np.stack([OI.make_image(W, H, 1000 + k) for k in range(8)])
    images = np.ascontiguousarray(base[np.arange(n_img) % 8])
    kps = [OI.make_keypoints(W, H, NKP, 4, 1.2, 2000 + k) for k in range(8)]
    xy = np.concatenate([kps[k % 8][0] for k in range(n_img)])
    oc = np.concatenate([kps[k % 8][1] for k in range(n_img)])
    off = (np.arange(n_img + 1) * NKP).astype(np.int32)
    return images, off, xy, oc


def cpu_arm(images, off, xy, oc, threads):
    from oracle.orb import OrbOracle
    n = min(len(images), max(16, 2 * threads))
    orc = OrbOracle()
    orc.compute_batch(images[:2], off[:3], xy[:2 * NKP], oc[:2 * NKP], None, threads=threads)
    t0 = time.perf_counter()
    orc.compute_batch(images[:n], off[:n + 1], xy[:n * NKP], oc[:n * NKP], None, threads=threads)
    out = {"value": n / (time.perf_counter() - t0), "unit": UNIT, "cores": threads, "kind": "port", "cpu": cpu_model(),
           "sample": f"{n} images, C oracle, one image per host thread"}
    try:
        import cv2
    except ImportError:
        out["cv2"] = None
        return out
    orb = cv2.ORB_create(1200, 1.2, 4, 19, 0, 2, cv2.ORB_FAST_SCORE, 31, 20)
    ck = [[cv2.KeyPoint(float(x), float(y), 31, 0.0, 0, int(o), -1)
           for (x, y), o in zip(xy[k * NKP:(k + 1) * NKP], oc[k * NKP:(k + 1) * NKP])] for k in range(8)]
    t0 = time.perf_counter()
    for k in range(n):
        orb.compute(images[k], ck[k % 8])
    out["cv2"] = {"value": n / (time.perf_counter() - t0), "unit": UNIT, "version": cv2.__version__,
                  "sample": f"{n} images, cv2.ORB.compute (given angles), one thread calling"}
    return out


def hbm_bytes_per_image():
    """Algorithmic HBM bytes per image: the image read once; each resized level written once and read twice (its blur, the
    next resize); each blurred level written once; per key point 16 B in and 40 B out, plus its two 31x31 patches."""
    lvl = [w * h for w, h in (OI.level_size(W, H, 1.2, l) for l in range(4))]
    return W * H + sum(3 * v for v in lvl[1:]) + sum(lvl) + NKP * (16 + 40 + 2 * 961)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="one GPU: the call is per context")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, default=128, help="stereo pairs per step (2 images each)")
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu", action="store_true", help="skip the CPU arm")
    args = ap.parse_args()
    threads = host_threads()
    n_img = 2 * args.pairs
    images, off, xy, oc = make_inputs(n_img)
    if args.impl == "reference":
        c = cpu_arm(images, off, xy, oc, threads)
        print(json.dumps({"impl": "reference", "metric": METRIC, "value": c["value"], "unit": UNIT, "n_gpus": 0, "steps": 1,
                          "warmup": 1, "higher_is_better": True, "config": {"workload": "orb"}, "cpu_baseline": c}), flush=True)
        return 0
    import torch
    from stvo_pl_b200.engine import Engine
    eng = Engine(int(os.environ.get("LOCAL_RANK", "0")))
    cfg = T.default_orb_config()
    for _ in range(max(args.warmup, 1)):
        n, out = eng.orb_compute_batch(cfg, images, off, xy, oc, None)
    torch.cuda.synchronize()
    stage = np.zeros(3)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        n, out = eng.orb_compute_batch(cfg, images, off, xy, oc, None)
        stage += eng.orb_kernel_times()
    dt = time.perf_counter() - t0
    stage /= args.steps
    dev_ms = float(stage.sum())
    bytes_img = hbm_bytes_per_image()
    line = {"metric": METRIC, "value": n_img * args.steps / dt, "unit": UNIT, "n_gpus": 1, "steps": args.steps,
            "warmup": max(args.warmup, 1), "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True,
            "dtype": "u8/f32", "data": "synthetic",
            "config": {"workload": "orb", "pairs_per_step": args.pairs, "images_per_step": n_img, "image": [W, H],
                       "keypoints_per_image": NKP, "levels": [OI.level_size(W, H, 1.2, l) for l in range(4)],
                       "survivors_per_step": int(n)},
            "kernel_ms_per_step": {"pyramid_and_blur": float(stage[0]), "border_filter": float(stage[1]),
                                   "angle_and_describe": float(stage[2])},
            "device_images_per_s": n_img / (dev_ms * 1e-3),
            "hbm": {"algorithmic_bytes_per_step": int(bytes_img * n_img),
                    "achieved_GBps_over_device_time": bytes_img * n_img / (dev_ms * 1e-3) / 1e9},
            "e2e": {"value": n_img * args.steps / dt, "unit": UNIT,
                    "h2d_bytes_per_step": int(images.nbytes + xy.nbytes + oc.nbytes + off.nbytes),
                    "d2h_bytes_per_step": int(n_img * NKP * 40 + n_img * 4)}}
    try:
        line["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        line["gpu"] = torch.cuda.get_device_name(0)
    if not args.no_cpu:
        line["cpu_baseline"] = cpu_arm(images, off, xy, oc, threads)
    print(json.dumps(line), flush=True)
    eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
