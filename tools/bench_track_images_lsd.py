"""Benchmark of stereo images alone -> pose (plstvo_track_stereo_images_lsd_sequence / _batch) against the two-call chain it
composes (plstvo_lsd_detect_batch, then plstvo_track_stereo_images_sequence / _batch fed its key lines); prints one JSON line.

A KITTI-size (1241x376) sequence of --frames stereo frames from tests/test_gpu_track_images.moving_views (a seeded textured
plane at constant disparity, the camera moving a few pixels per frame), ORB 1200 features on 4 levels, the shipped LSD
options (300 lines per image, scale 1.2).  Two shapes, each through both arms, the arms alternating in this invocation:
  sequence  the whole sequence in one call;
  pair      one pair per call (B = 1, the shape of plstvo::StereoImageHandler), over the first --pairs pairs.
value = pairs/s of the sequence through the images-only call, host images in, host results out, synchronised.  The outputs
of the two arms must be byte-identical.  Also printed: medians of --steps timed runs per arm, the device time per stage, the
bytes each arm moves over PCIe (from the shapes), and the card with its power limit, read in the same run.  Writes nothing to
the tree.

    python tools/bench_track_images_lsd.py --gpus 1 [--steps 5] [--warmup 1] [--frames 257] [--pairs 8]
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

from stvo_pl_b200 import types as T  # noqa: E402
from test_gpu_track_images import moving_views  # noqa: E402

W, H = 1241, 376
METRIC = "stereo images alone -> pose, KITTI-size sequence (LSD 300 lines, ORB 1200 x 4 levels)"
UNIT = "pairs/s"
RESULT_BYTES = 8 * 147 + 4 * 10
KL_DOWN = 16 + 4 + 4 + 4 + 4   # a key line as plstvo_lsd_detect_batch returns it: segment, angle, npix, response, length


def chain(eng, cam, tc, mc, sc, oc, lc, sets, sequence, priors=None):
    """plstvo_lsd_detect_batch on every image in the images call's block order, then the images call fed its key lines."""
    NF = len(sets[0]["img_l"])
    _, kl = eng.lsd_detect_batch(lc, np.concatenate([im for s in sets for im in (s["img_l"], s["img_r"])]))
    fed = []
    for j, s in enumerate(sets):
        d = dict(img_l=s["img_l"], img_r=s["img_r"], fast_th=s.get("fast_th"))
        for side, b in (("l", 2 * j), ("r", 2 * j + 1)):
            off = kl["off"][b * NF:(b + 1) * NF + 1]
            d[f"l{side}_off"] = off - off[0]
            for k in ("seg", "angle", "npix"):
                d[f"{k}_{side}"] = kl[k][off[0]:off[-1]]
        fed.append(d)
    if sequence:
        return eng.track_stereo_images_sequence(cam, tc, mc, sc, oc, fed[0], priors), kl
    return eng.track_stereo_images_batch(cam, tc, mc, sc, oc, fed[0], fed[1], priors), kl


def pcie_bytes(n_img, img_bytes, n_lines, n_left_lines):
    """Host <-> device bytes in which the arms differ, from the shapes: the images (once, or twice) and the key lines (the
    chain brings LSD's rows down to the host and feeds them back; the images-only call sends the kept key lines up once, as
    the chain's second call also does).  LSD's region hops, ORB's offsets, the stereo step's counts and the results are the
    same in both arms and left out."""
    lines_up = n_lines * (16 + 8 + 4) + n_left_lines * 4    # segments, (cos, sin), numOfPixels; left angles for the stereo step
    images_only = img_bytes + lines_up
    chain_ = 2 * img_bytes + n_lines * KL_DOWN + (n_img + 1) * 4 + lines_up
    return {"images_only_call": int(images_only), "chain": int(chain_), "saved": int(chain_ - images_only)}


def timed(fn, steps):
    t = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="one GPU: the call is per context")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--frames", type=int, default=257)
    ap.add_argument("--pairs", type=int, default=8)
    args = ap.parse_args()
    import torch
    from stvo_pl_b200.engine import Engine
    eng = Engine(int(os.environ.get("LOCAL_RANK", "0")))
    cam = T.kitti_camera()
    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    oc, lc = T.default_orb_detect_config(1200, 4), T.default_lsd_config()
    fr = moving_views(args.frames, W, H, 7004, 0)
    fr = dict(img_l=fr["img_l"], img_r=fr["img_r"], fast_th=None)
    NF, pairs = args.frames, args.frames - 1
    out = {}

    # the sequence in one call
    new = lambda: eng.track_stereo_images_lsd_sequence(cam, tc, mc, sc, oc, lc, fr)   # noqa: E731
    old = lambda: chain(eng, cam, tc, mc, sc, oc, lc, [fr], True)                      # noqa: E731
    a, (b, kl) = new(), old()
    identical = a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1])
    for _ in range(max(args.warmup - 1, 0)):
        new(), old()
    t_new, t_old, stage, lsd_ms = [], [], np.zeros(5), np.zeros(5)
    for _ in range(args.steps):       # the two arms alternate
        t_new += timed(new, 1)
        stage += eng.track_stereo_images_stage_times()
        lsd_ms += eng.lsd_kernel_times()
        t_old += timed(old, 1)
    tn, to = float(np.median(t_new)), float(np.median(t_old))
    nl, nll = int(kl["off"][-1]), int(kl["off"][NF])
    out["sequence"] = {"pairs": pairs, "pairs_per_s": pairs / tn, "ms_per_call": tn * 1e3, "chain_pairs_per_s": pairs / to,
                       "chain_ms_per_call": to * 1e3, "speedup": to / tn,
                       "spread_ms": {"images_only": [min(t_new) * 1e3, max(t_new) * 1e3], "chain": [min(t_old) * 1e3, max(t_old) * 1e3]},
                       "identical_outputs": bool(identical), "good_pairs": int(a[0]["good"].sum()),
                       "mean_stereo_points": float(a[1][:, 0].mean()), "mean_stereo_lines": float(a[1][:, 1].mean()),
                       "stage_ms": dict(zip(("upload", "orb", "lines", "stereo_step", "tracking"), (stage / args.steps).round(3).tolist())),
                       "lsd_kernel_ms": dict(zip(("blur_resize", "gradient_seeds", "grow", "host_angles", "rectangles"),
                                                 (lsd_ms / args.steps).round(3).tolist())),
                       "pcie_bytes": pcie_bytes(2 * NF, 2 * fr["img_l"].size, nl, nll)}

    # one pair per call, as the handler calls it
    P = min(args.pairs, pairs)
    sl = lambda a_, b_: dict(img_l=fr["img_l"][a_:b_], img_r=fr["img_r"][a_:b_], fast_th=None)   # noqa: E731
    sets = [(sl(p, p + 1), sl(p + 1, p + 2)) for p in range(P)]
    new1 = lambda: [eng.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, x, y) for x, y in sets]   # noqa: E731
    old1 = lambda: [chain(eng, cam, tc, mc, sc, oc, lc, [x, y], False) for x, y in sets]                  # noqa: E731
    a1, b1 = new1(), old1()
    identical1 = all(x[0].tobytes() == y[0][0].tobytes() and np.array_equal(x[1], y[0][1]) for x, y in zip(a1, b1))
    for _ in range(max(args.warmup - 1, 0)):
        new1(), old1()
    t_new, t_old = [], []
    kms = {"images_only": np.zeros(5), "chain": np.zeros(5)}   # LSD's device stages per call, each arm
    sms = {"images_only": np.zeros(5), "chain": np.zeros(5)}   # the images call's stages per call, each arm
    for _ in range(args.steps):   # the two arms alternate; after each call its LSD and stage times are read
        for arm, one, t in (("images_only", lambda x, y: eng.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, x, y), t_new),
                            ("chain", lambda x, y: chain(eng, cam, tc, mc, sc, oc, lc, [x, y], False), t_old)):
            t0 = time.perf_counter()
            for x, y in sets:
                one(x, y)
                kms[arm] += eng.lsd_kernel_times()
                sms[arm] += eng.track_stereo_images_stage_times()
            t.append(time.perf_counter() - t0)
    tn, to = float(np.median(t_new)) / P, float(np.median(t_old)) / P
    nl1 = sum(int(y[1]["off"][-1]) for y in b1)
    nll1 = sum(int(y[1]["off"][1] + y[1]["off"][3] - y[1]["off"][2]) for y in b1)
    out["pair"] = {"pairs": P, "pairs_per_s": 1 / tn, "ms_per_call": tn * 1e3, "chain_pairs_per_s": 1 / to,
                   "chain_ms_per_call": to * 1e3, "speedup": to / tn,
                   "spread_ms_per_call": {"images_only": [min(t_new) / P * 1e3, max(t_new) / P * 1e3],
                                          "chain": [min(t_old) / P * 1e3, max(t_old) / P * 1e3]},
                   "identical_outputs": bool(identical1),
                   "lsd_kernel_ms": {arm: dict(zip(("blur_resize", "gradient_seeds", "grow", "host_angles", "rectangles"),
                                                   (v / (args.steps * P)).round(3).tolist())) for arm, v in kms.items()},
                   "stage_ms": {arm: dict(zip(("upload", "orb", "lines" if arm == "images_only" else "lbd", "stereo_step",
                                               "tracking"), (v / (args.steps * P)).round(3).tolist())) for arm, v in sms.items()},
                   "pcie_bytes_per_call": {k: v // P for k, v in pcie_bytes(4, 4 * W * H, nl1, nll1).items()}}

    s = out["sequence"]
    line = {"metric": METRIC, "value": s["pairs_per_s"], "unit": UNIT, "n_gpus": 1, "steps": args.steps,
            "warmup": max(args.warmup, 1), "higher_is_better": True, "data": "synthetic",
            "config": {"workload": "track_images_lsd", "frames": args.frames, "image": [W, H]}, "shapes": out}
    try:
        line["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                     capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        line["gpu"] = torch.cuda.get_device_name(0)
    print(json.dumps(line), flush=True)
    eng.close()
    return 0 if all(v["identical_outputs"] for v in out.values()) else 1


if __name__ == "__main__":
    sys.exit(main())
