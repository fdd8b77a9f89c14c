"""Writes tests/golden/orb_default.npz and tests/golden/orb_kitti.npz from cv2's ORB (needs cv2).

Images come from tests/orb_images.py (seeded, integer-only); the files keep their SHA-256, not their pixels.
  orb_default: 4 levels, scale 1.2, two 640x480 images.
  orb_kitti:   1 level (config_kitti.yaml), the left and right images of two 1241x376 stereo frames of a textured plane
               moving parallel to the image plane; used by the end-to-end tracking test too.
Each holds, per image: detectAndCompute's key points (pt, octave, angle as float32 bits) and descriptors, and ORB::compute
on seeded key points with given angles (including key points on both sides of the border filter) with its survivors'
source indices and descriptors.

    python tools/make_orb_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import orb_images as I  # noqa: E402

KITTI_W, KITTI_H, SHIFT = 1241, 376, (14, 3)   # frame 2 = frame 1 moved by (14, 3) px; right = left moved by DISP px
DISP = 24


def kitti_views(seed: int = 11):
    """Left / right images of two frames cropped from one larger seeded texture: a plane parallel to the image plane at
    constant disparity, the camera moving by SHIFT pixels between the frames."""
    big = I.make_image(KITTI_W + 64, KITTI_H + 16, seed)
    out = []
    for f in range(2):
        x0, y0 = 8 + f * SHIFT[0], 4 + f * SHIFT[1]
        out.append(big[y0:y0 + KITTI_H, x0:x0 + KITTI_W])                  # left
        out.append(big[y0:y0 + KITTI_H, x0 + DISP:x0 + DISP + KITTI_W])    # right: scene point at x appears at x - DISP
    return np.stack(out)


def border_keypoints(W, H, edge=19):
    """Key points on both sides of runByImageBorder's cvRound(pt) test, all at level 0."""
    xs = [edge - 1.0, edge - 0.5, edge - 0.49, edge + 0.0, W - edge - 1.0, W - edge - 0.5, W - edge - 0.51, W - edge + 0.0]
    pts = [(x, H / 2) for x in xs] + [(W / 2, edge - 0.5), (W / 2, edge + 0.0), (W / 2, H - edge - 0.5), (W / 2, H - edge - 1.0)]
    return np.array(pts, np.float32)


def golden(images, n_levels, scale, n_given, seed):
    import cv2
    orb = cv2.ORB_create(1200, scale, n_levels, 19, 0, 2, cv2.ORB_FAST_SCORE, 31, 20)
    n, H, W = images.shape
    rec = dict(n_levels=np.int32(n_levels), scale=np.float64(scale), width=np.int32(W), height=np.int32(H),
               sha256=np.array([I.sha256(im) for im in images]), cv2_version=np.array(cv2.__version__))
    det_off, det_xy, det_oct, det_ang, det_desc = [0], [], [], [], []
    g_off, g_xy, g_oct, g_ang, g_src, g_desc, g_cnt = [0], [], [], [], [], [], []
    for i, img in enumerate(images):
        kps, des = orb.detectAndCompute(img, None)
        det_xy.append(np.array([k.pt for k in kps], np.float32).reshape(-1, 2))
        det_oct.append(np.array([k.octave for k in kps], np.int32))
        det_ang.append(np.array([k.angle for k in kps], np.float32))
        det_desc.append(np.asarray(des, np.uint8).reshape(-1, 32))
        det_off.append(det_off[-1] + len(kps))
        xy, oct_, ang = I.make_keypoints(W, H, n_given, n_levels, scale, seed + 101 * i)
        bxy = border_keypoints(W, H)
        bang = np.float32([0, 45, 90, 135, 180, 225, 270, 359.99, 44.99, 45.01, 315, 0])[:len(bxy)]
        xy, oct_ = np.concatenate([bxy, xy]), np.concatenate([np.zeros(len(bxy), np.int32), oct_])
        ang = np.concatenate([bang, ang]).astype(np.float32)
        order = np.argsort(oct_, kind="stable")     # ORB::compute regroups unsorted input by octave: give it sorted
        xy, oct_, ang = xy[order], oct_[order], ang[order]
        ckp = [cv2.KeyPoint(float(x), float(y), 31, float(a), 0, int(o), -1) for (x, y), a, o in zip(xy, ang, oct_)]
        out, d = orb.compute(img, ckp)
        src, j = [], 0
        for k in out:                                # survivors keep input order: walk the input
            while not (np.float32(k.pt[0]) == xy[j, 0] and np.float32(k.pt[1]) == xy[j, 1] and k.octave == oct_[j]):
                j += 1
            src.append(j)
            j += 1
        g_xy.append(xy); g_oct.append(oct_); g_ang.append(ang)
        g_src.append(np.array(src, np.int32)); g_desc.append(np.asarray(d, np.uint8).reshape(-1, 32)); g_cnt.append(len(out))
        g_off.append(g_off[-1] + len(xy))
    rec.update(det_off=np.int32(det_off), det_xy=np.concatenate(det_xy), det_oct=np.concatenate(det_oct),
               det_angle_bits=np.concatenate(det_ang).view(np.uint32), det_desc=np.concatenate(det_desc),
               given_off=np.int32(g_off), given_xy=np.concatenate(g_xy), given_oct=np.concatenate(g_oct),
               given_angle_bits=np.concatenate(g_ang).view(np.uint32), given_counts=np.int32(g_cnt),
               given_src_idx=np.concatenate(g_src), given_desc=np.concatenate(g_desc))
    return rec


def default_images():
    return np.stack([I.make_image(640, 480, s) for s in (1, 2)])


if __name__ == "__main__":
    out = os.path.join(ROOT, "tests", "golden")
    np.savez_compressed(os.path.join(out, "orb_default.npz"), **golden(default_images(), 4, 1.2, 1500, 5))
    np.savez_compressed(os.path.join(out, "orb_kitti.npz"), **golden(kitti_views(), 1, 1.2, 800, 9))
    for f in ("orb_default.npz", "orb_kitti.npz"):
        print(f, os.path.getsize(os.path.join(out, f)), "bytes")
