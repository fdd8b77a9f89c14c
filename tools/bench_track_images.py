"""Benchmark of stereo images -> pose (plstvo_track_stereo_images_sequence) against the three calls it composes
(plstvo_orb_detect_and_compute_batch, plstvo_lbd_compute_batch, plstvo_track_stereo_sequence); prints one JSON line.

A KITTI-size (1241x376) sequence of --frames stereo frames from tests/test_gpu_track_images.moving_views (a seeded textured
plane at constant disparity, the camera moving a few pixels per frame, key lines drawn on the texture and mapped into every
view).  Two configs: `default` (ORB 1200 features on 4 levels, 300 lines per image) and `kitti` (2000 features on 1 level,
100 lines).  value = pairs/s through the images call, host images and key lines in, host results out, synchronised; the
composition arm runs on the same inputs, alternating with it in this invocation, and the two must give identical bytes.
Also printed: the device time per stage, the bytes each arm moves over PCIe (from the shapes), and the card with its power
limit, read in the same run.  Writes nothing to the tree.

    python tools/bench_track_images.py --gpus 1 [--steps 5] [--warmup 1] [--frames 257]
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
from test_gpu_track_images import compose, moving_views  # noqa: E402

W, H = 1241, 376
CONFIGS = {"default": (1200, 4, 300), "kitti": (2000, 1, 100)}   # ORB features, levels, lines per image
METRIC = "stereo images -> pose, KITTI-size sequence (ORB 1200 x 4 levels, 300 lines per image)"
UNIT = "pairs/s"
RESULT_BYTES = 8 * 147 + 4 * 10


def pcie_bytes(frames, orb_off, harris=False):
    """Host <-> device bytes of one sequence through either arm, from the shapes (small control traffic of the stereo step,
    which both arms share, left out)."""
    NF = len(frames["img_l"])
    n_img, img = 2 * NF, 2 * frames["img_l"].size
    nl = int(frames["ll_off"][-1] + frames["lr_off"][-1])
    nll, nkp = int(frames["ll_off"][-1]), int(orb_off[-1])
    nkl = int(orb_off[NF])                        # left key points
    lines_up = nl * (16 + 8 + 4)                  # segments, (cos, sin), numOfPixels
    off_rb = (n_img + 1) * 4 * (2 if harris else 1)
    results = (NF - 1) * RESULT_BYTES + NF * 8
    images_arm = img + 4 * NF + lines_up + nll * 4 + off_rb + results          # + left angles for the stereo step
    orb_down = nkp * (8 + 4 + 4 + 4 + 32) + off_rb
    stereo_up = nkp * (8 + 32) + nkl * 4 + nl * (16 + 32) + nll * (4 + 4)    # key points, octaves, lines, angles, octaves
    composition = img + 4 * n_img + orb_down + img + lines_up + nl * 32 + stereo_up + results
    return {"images_call": int(images_arm), "composition": int(composition)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1, help="one GPU: the call is per context")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--frames", type=int, default=257)
    args = ap.parse_args()
    import torch
    from stvo_pl_b200.engine import Engine
    eng = Engine(int(os.environ.get("LOCAL_RANK", "0")))
    cam = T.kitti_camera()
    mc, sc, tc = T.default_stereo_match_config(), T.default_stereo_config(), T.kitti_config()
    mc.min_ratio_12_p = 0.75
    out = {}
    for name, (nfeat, nlev, nlines) in CONFIGS.items():
        oc = T.default_orb_detect_config(nfeat, nlev)
        fr = moving_views(args.frames, W, H, 7000 + nlev, nlines)
        pairs = args.frames - 1
        a = eng.track_stereo_images_sequence(cam, tc, mc, sc, oc, fr)
        b = compose(eng, cam, tc, mc, sc, oc, [fr], True)
        identical = a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1])
        _, orb = eng.orb_detect_and_compute_batch(oc, np.concatenate([fr["img_l"], fr["img_r"]]))
        for _ in range(max(args.warmup - 1, 0)):
            eng.track_stereo_images_sequence(cam, tc, mc, sc, oc, fr)
            compose(eng, cam, tc, mc, sc, oc, [fr], True)
        t_img, t_cmp, stage = [], [], np.zeros(5)
        for _ in range(args.steps):       # the two arms alternate
            t0 = time.perf_counter()
            eng.track_stereo_images_sequence(cam, tc, mc, sc, oc, fr)
            t_img.append(time.perf_counter() - t0)
            stage += eng.track_stereo_images_stage_times()
            t0 = time.perf_counter()
            compose(eng, cam, tc, mc, sc, oc, [fr], True)
            t_cmp.append(time.perf_counter() - t0)
        ti, tcmp = float(np.median(t_img)), float(np.median(t_cmp))
        out[name] = {"pairs_per_s": pairs / ti, "ms_per_sequence": ti * 1e3, "composition_pairs_per_s": pairs / tcmp,
                     "composition_ms_per_sequence": tcmp * 1e3, "speedup": tcmp / ti, "identical_outputs": bool(identical),
                     "good_pairs": int(a[0]["good"].sum()), "mean_stereo_points": float(a[1][:, 0].mean()),
                     "mean_stereo_lines": float(a[1][:, 1].mean()),
                     "stage_ms": dict(zip(("upload", "orb", "lbd", "stereo_step", "tracking"),
                                          (stage / args.steps).round(3).tolist())),
                     "pcie_bytes": pcie_bytes(fr, orb["off"]),
                     "orb": {"n_features": nfeat, "n_levels": nlev}, "lines_per_image": nlines}
    d = out["default"]
    line = {"metric": METRIC, "value": d["pairs_per_s"], "unit": UNIT, "n_gpus": 1, "steps": args.steps,
            "warmup": max(args.warmup, 1), "higher_is_better": True, "data": "synthetic",
            "config": {"workload": "track_images", "frames": args.frames, "image": [W, H]}, "configs": out}
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
