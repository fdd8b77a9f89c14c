"""Colour input on the GPU against host conversion (cv2.cvtColor, plus cv2.remap on colour for a distorted rig).

  1. the preparation kernel: plstvo_rectify_batch with a colour rectifier at 2, 64 and 512 images, for KITTI 1241 x 376 BGR
     without maps and EuRoC 752 x 480 BGR with maps (tools/make_rectify_golden.py's rig), as the kernel's device time (CUDA
     events) and its algorithmic bytes over that time: C + 1 bytes per pixel (read C, write 1), plus 6 of map with maps.
  2. colour images to pose: plstvo_track_stereo_raw_images_batch with the colour rectifier against cv2.cvtColor (after
     cv2.remap on the colour image for the EuRoC rig) on the host, on one thread and on all of them, followed by
     plstvo_track_stereo_images_lsd_batch on the grey images, at 1 and 64 pairs; with the bytes each uploads.
Prints one JSON line per measurement, with the card and its power limit.  cv2 is optional: its rows say "not measured"
without it.

    python tools/bench_color.py [--reps 10]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_rectify import card, timed  # noqa: E402

HBM_TB_S = 3.35   # H100 SXM data sheet


def colorize(g, seed):
    """BGR images with the grey texture of g: B = 255 - g (+-3 of noise), G = g, R = g^2 / 255"""
    rng = np.random.default_rng(seed)
    g = np.asarray(g).astype(np.int32)
    return np.stack([np.clip(255 - g + rng.integers(-3, 4, g.shape), 0, 255), g, g * g // 255], -1).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    from stvo_pl_b200 import types as T
    from stvo_pl_b200.engine import Engine, init_undistort_rectify_map
    from test_gpu_track_images import configs, moving_views
    try:
        import cv2
    except ImportError:
        cv2 = None
    gpu = card()
    z = np.load(os.path.join(ROOT, "tests", "golden", "rectify.npz"))

    def maps(c):
        w, h = (int(v) for v in z[f"{c}_size"])
        return init_undistort_rectify_map(int(z[f"{c}_model"]), z[f"{c}_K"], z[f"{c}_D"], z[f"{c}_R"], z[f"{c}_P"], w, h)

    (m1l, m2l), (m1r, m2r) = maps("euroc_l"), maps("euroc_r")
    fx, fy, cx, cy, b = z["euroc_l_cam"]
    setups = {"kitti_bgr_no_maps": (T.kitti_camera(), None), "euroc_bgr_maps": (
        T.PlCamera(fx=fx, fy=fy, cx=cx, cy=cy, b=b, width=752, height=480), (m1l, m2l, m1r, m2r))}
    e = Engine()
    out = []
    # 1. the preparation kernel
    for name, (cam, mp) in setups.items():
        W, H = cam.width, cam.height
        rect = e.rectifier_create_color(W, H, 3, *(mp or ()))
        rng = np.random.default_rng(1)
        for n_img in (2, 64, 512):
            B = n_img // 2
            il = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
            ir = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
            e.rectify_batch(rect, il, ir)
            kms = []
            for _ in range(a.reps):
                e.rectify_batch(rect, il, ir)
                kms.append(e.rectify_kernel_times())
            k = float(np.median(kms)) * 1e-3
            px = n_img * W * H
            per_px = 3 + 1 + (6 if mp else 0)
            gbs = px * per_px / k / 1e9
            out.append(dict(what="color_prepare_kernel", setup=name, images=n_img, kernel_ms=k * 1e3,
                            bytes_per_pixel=per_px, gb_per_s=gbs, share_of_hbm_datasheet=gbs / (HBM_TB_S * 1e3), card=gpu))
        e.rectifier_destroy(rect)
    # 2. colour images to pose
    mc, sc, tc, oc = configs(1200, 4)
    lc = T.default_lsd_config()
    for name, (cam, mp) in setups.items():
        W, H = cam.width, cam.height
        rect = e.rectifier_create_color(W, H, 3, *(mp or ()))
        for B in (1, 64):
            fr = moving_views(B + 1, W, H, 811, 200)
            col = dict(img_l=colorize(fr["img_l"], 2), img_r=colorize(fr["img_r"], 3))
            prev = dict(img_l=col["img_l"][:B], img_r=col["img_r"][:B], fast_th=None)
            curr = dict(img_l=col["img_l"][1:], img_r=col["img_r"][1:], fast_th=None)
            t_gpu = timed(lambda: e.track_stereo_raw_images_batch(cam, tc, mc, sc, oc, lc, rect, prev, curr), max(3, a.reps // 2))
            px = 4 * B * W * H
            row = dict(what="color_images_call", setup=name, pairs=B, ms=t_gpu * 1e3, pairs_per_s=B / t_gpu,
                       upload_bytes=px * 3, card=gpu)
            if cv2 is None:
                row.update(host="not measured: cv2 missing")
                out.append(row)
                continue

            def host_then_grey():
                def grey(img, m1, m2):
                    src = img if mp is None else cv2.remap(img, m1, m2, cv2.INTER_LINEAR)
                    return cv2.cvtColor(src, cv2.COLOR_BGR2GRAY)
                fed = [dict(img_l=np.stack([grey(i, m1l, m2l) for i in s["img_l"]]),
                            img_r=np.stack([grey(i, m1r, m2r) for i in s["img_r"]]), fast_th=None) for s in (prev, curr)]
                return e.track_stereo_images_lsd_batch(cam, tc, mc, sc, oc, lc, fed[0], fed[1])
            for threads in (1, os.cpu_count()):
                cv2.setNumThreads(threads)
                t_host = timed(host_then_grey, max(3, a.reps // 2))
                row[f"host_{threads}_threads_then_grey_ms"] = t_host * 1e3
                row[f"speedup_vs_host_{threads}_threads"] = t_host / t_gpu
            row["host_upload_bytes"] = px
            out.append(row)
        e.rectifier_destroy(rect)
    e.close()
    for r in out:
        print(json.dumps(r))


if __name__ == "__main__":
    main()
