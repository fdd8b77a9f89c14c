"""Benchmark of LBD line description (plstvo_lbd_compute_batch); prints one JSON line.

B KITTI-size images (1241x376, seeded integer-only images from tests/orb_images.py) with seeded key lines of LSD-like
lengths (a NumPy generator: no cv2 needed), 300 per image (default config, lsd_nfeatures 300) and 100 per image (KITTI
config).  value = images/s through the whole call (upload, kernels, download) at 300 lines; the line also carries the
100-line figure, the device time per stage (CUDA events), the algorithmic HBM bytes and a CPU arm (the reference's own
BinaryDescriptor::compute from oracle/_ref, one image per host thread; null when that library is not built).  Writes
nothing to the tree.

    python tools/bench_lbd.py --gpus 1 --steps 20 --warmup 3 [--images 256] [--no-cpu] [--impl reference]
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
import orb_images as OI  # noqa: E402

W, H = 1241, 376
CONFIGS = {"default": 300, "kitti": 100}
METRIC = "LBD descriptors of given key lines, KITTI-size images (300 lines each)"
UNIT = "images/s"


def make_lines(n, seed):
    """n key lines with LSD-like lengths: mostly 10-60 px, a tail of long ones up to the image width; numOfPixels is the
    8-connected pixel count of the rounded end points."""
    rng = np.random.default_rng(seed)
    length = np.minimum(float(W), 10.0 + rng.exponential(30.0, n) * rng.choice([1.0, 8.0], n, p=[0.9, 0.1]))
    th = rng.uniform(-np.pi, np.pi, n)
    cx, cy = rng.uniform(0, W - 1, n), rng.uniform(0, H - 1, n)
    seg = np.stack([cx - 0.5 * length * np.cos(th), cy - 0.5 * length * np.sin(th),
                    cx + 0.5 * length * np.cos(th), cy + 0.5 * length * np.sin(th)], 1)
    seg[:, 0::2] = np.clip(seg[:, 0::2], 0, W - 1)
    seg[:, 1::2] = np.clip(seg[:, 1::2], 0, H - 1)
    seg = seg.astype(np.float32)
    ang = np.arctan2(seg[:, 3].astype(np.float64) - seg[:, 1], seg[:, 2].astype(np.float64) - seg[:, 0]).astype(np.float32)
    r = np.rint(seg.astype(np.float64)).astype(np.int64)
    npix = (np.maximum(np.abs(r[:, 2] - r[:, 0]), np.abs(r[:, 3] - r[:, 1])) + 1).astype(np.int32)
    return seg, ang, npix


def make_inputs(n_img, n_lines):
    base = np.stack([OI.make_image(W, H, 3000 + k) for k in range(8)])
    images = np.ascontiguousarray(base[np.arange(n_img) % 8])
    parts = [make_lines(n_lines, 4000 + k) for k in range(8)]
    seg = np.concatenate([parts[k % 8][0] for k in range(n_img)])
    ang = np.concatenate([parts[k % 8][1] for k in range(n_img)])
    npix = np.concatenate([parts[k % 8][2] for k in range(n_img)])
    off = (np.arange(n_img + 1) * n_lines).astype(np.int32)
    return images, off, seg, ang, npix


def cpu_arm(images, off, seg, ang, npix, threads):
    from concurrent.futures import ThreadPoolExecutor
    from oracle import lbd
    if not lbd.available():
        return None
    n = min(len(images), max(16, 2 * threads))

    def one(k):
        a, b = off[k], off[k + 1]
        return lbd.compute(images[k], seg[a:b], ang[a:b], npix[a:b])

    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(one, range(min(n, threads))))
        t0 = time.perf_counter()
        list(ex.map(one, range(n)))
        dt = time.perf_counter() - t0
    return {"value": n / dt, "unit": UNIT, "cores": threads, "kind": "reference", "cpu": cpu_model(),
            "sample": f"{n} images, the reference's BinaryDescriptor::compute (oracle/_ref), one image per host thread"}


def hbm_bytes_per_step(n_img, npix):
    """Algorithmic HBM bytes of one call: each image read once, its (dx, dy) map written once (4 B a pixel), per line
    63 x numOfPixels 4-byte gathers, 28 B of inputs and 32 B of output."""
    return n_img * 5 * W * H + 63 * 4 * int(npix.sum()) + len(npix) * (28 + 32)


def run_gpu(eng, images, off, seg, ang, npix, steps, warmup):
    for _ in range(max(warmup, 1)):
        eng.lbd_compute_batch(images, off, seg, ang, npix)
    stage = np.zeros(2)
    t0 = time.perf_counter()
    for _ in range(steps):
        eng.lbd_compute_batch(images, off, seg, ang, npix)
        stage += eng.lbd_kernel_times()
    dt = time.perf_counter() - t0
    return len(images) * steps / dt, dt / steps * 1e3, stage / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="one GPU: the call is per context")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--images", type=int, default=256, help="images per call")
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu", action="store_true", help="skip the CPU arm")
    ap.add_argument("--longest-first", action="store_true",
                    help="order each image's lines by numOfPixels, longest first (the descriptor kernel runs one block per line "
                         "in grid order; this measures whether that order matters)")
    args = ap.parse_args()
    threads = host_threads()
    inputs = {k: make_inputs(args.images, n) for k, n in CONFIGS.items()}
    if args.longest_first:
        for k, (images, off, seg, ang, npix) in inputs.items():
            idx = np.concatenate([off[i] + np.argsort(-npix[off[i]:off[i + 1]], kind="stable") for i in range(len(images))])
            inputs[k] = (images, off, seg[idx], ang[idx], npix[idx])
    if args.impl == "reference":
        c = cpu_arm(*inputs["default"], threads)
        print(json.dumps({"impl": "reference", "metric": METRIC, "value": c["value"] if c else None, "unit": UNIT, "n_gpus": 0,
                          "steps": 1, "warmup": 1, "higher_is_better": True, "config": {"workload": "lbd"},
                          "cpu_baseline": c}), flush=True)
        return 0
    import torch
    from stvo_pl_b200.engine import Engine
    eng = Engine(int(os.environ.get("LOCAL_RANK", "0")))
    res = {k: run_gpu(eng, *inputs[k], args.steps, args.warmup) for k in CONFIGS}
    v, ms, stage = res["default"]
    npix = inputs["default"][4]
    bytes_step = hbm_bytes_per_step(args.images, npix)
    dev_ms = float(stage.sum())
    line = {"metric": METRIC, "value": v, "unit": UNIT, "n_gpus": 1, "steps": args.steps, "warmup": max(args.warmup, 1),
            "ms_per_step": ms, "higher_is_better": True, "dtype": "u8/i16/f32", "data": "synthetic",
            "config": {"workload": "lbd", "images_per_step": args.images, "image": [W, H],
                       "lines_per_image": CONFIGS["default"], "mean_num_of_pixels": float(npix.mean()),
                       "max_num_of_pixels": int(npix.max()), "line_order": "longest first" if args.longest_first else "as generated"},
            "kernel_ms_per_step": {"blur_and_sobel": float(stage[0]), "describe": float(stage[1])},
            "device_images_per_s": args.images / (dev_ms * 1e-3),
            "hbm": {"algorithmic_bytes_per_step": int(bytes_step),
                    "achieved_GBps_over_device_time": bytes_step / (dev_ms * 1e-3) / 1e9},
            "kitti_config": {"lines_per_image": CONFIGS["kitti"], "value": res["kitti"][0], "unit": UNIT,
                             "ms_per_step": res["kitti"][1],
                             "kernel_ms_per_step": {"blur_and_sobel": float(res["kitti"][2][0]),
                                                    "describe": float(res["kitti"][2][1])}}}
    try:
        line["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        line["gpu"] = torch.cuda.get_device_name(0)
    if not args.no_cpu:
        line["cpu_baseline"] = cpu_arm(*inputs["default"], threads)
    print(json.dumps(line), flush=True)
    eng.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
