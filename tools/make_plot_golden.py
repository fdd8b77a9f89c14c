"""Writes tests/golden/plot.npz: what cv2 4.13 draws for StereoFrame::plotStereoFrame, so that oracle/plot.py is held to
OpenCV where cv2 is not installed.

  kitti_seed, kitti_pl, kitti_spl, kitti_epl   a 1241 x 376 BGR frame (make_color_golden.color_image(seed)) with 2000
                                               points and 300 lines, many within 3 px of the border or leaving it
  kitti_mask                                   np.packbits of the pixels cv2.circle / cv2.line set to (0, 200, 0)
  grid_sha                                     SHA-256 of cv2's masks of every segment between end points on
                                               [-4, W + 3] x [-4, H + 3] of the GRID canvases, both orders, row-major
  circle_sha                                   SHA-256 of cv2's masks of every radius-3 circle centre on [-3, W + 2] x [-3, H + 2]
                                               of a 9 x 7 canvas
  remap<C>_seed, remap<C>_map1, remap<C>_map2  a 64 x 48 C-channel image (C = 3, 4) and cv2.convertMaps maps whose taps leave
  remap<C>_out                                 the image; cv2.cvtColor(cv2.remap(img), COLOR_BGR(A)2BGR)

    python tools/make_plot_golden.py            # needs cv2; rewrites tests/golden/plot.npz
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_color_golden as MC  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "plot.npz")
COLOUR = (0, 200, 0)
GRID = [(9, 7), (5, 4), (1, 1), (3, 8), (2, 1)]
KITTI = (1241, 376)


def grid_points(w: int, h: int, margin: int):
    return [(x, y) for y in range(-margin, h + margin) for x in range(-margin, w + margin)]


def kitti_inputs(seed: int = 2024):
    """the KITTI-size case's frame and rows: points anywhere (a third within 3 px of a border), lines of every length,
    a third with an end outside the image, float end points whose int() truncates toward zero"""
    W, H = KITTI
    rng = np.random.default_rng(seed)
    base = MC.color_image(seed, W, H, 3)
    pl = np.stack([rng.uniform(0, W, 2000), rng.uniform(0, H, 2000)], 1)
    edge = rng.random(2000) < 1 / 3
    pl[edge, 0] = np.where(rng.random(edge.sum()) < 0.5, rng.uniform(0, 3.5, edge.sum()), rng.uniform(W - 3.5, W, edge.sum()))
    spl = np.stack([rng.uniform(-0.9, W, 300), rng.uniform(-0.9, H, 300)], 1)
    length, ang = rng.exponential(80, 300), rng.uniform(-np.pi, np.pi, 300)
    epl = spl + np.stack([length * np.cos(ang), length * np.sin(ang)], 1)
    out = rng.random(300) < 1 / 3
    epl[out] += np.stack([rng.uniform(-60, 60, out.sum()), rng.uniform(-60, 60, out.sum())], 1) * 10
    return base, pl, spl, epl


def cv2_plot(base, pl, spl, epl):
    """plotStereoFrame's drawing with cv2 on a copy of base"""
    import cv2
    img = base.copy()
    for x, y in pl:
        cv2.circle(img, (int(x), int(y)), 3, COLOUR, 1)
    for s, e in zip(spl, epl):
        cv2.line(img, (int(s[0]), int(s[1])), (int(e[0]), int(e[1])), COLOUR, 1)
    return img


def cv2_grid_sha() -> str:
    import cv2
    h = hashlib.sha256()
    for w, hh in GRID:
        pts = grid_points(w, hh, 4)
        for p in pts:
            for q in pts:
                img = np.zeros((hh, w, 3), np.uint8)
                cv2.line(img, p, q, COLOUR, 1)
                h.update(np.packbits(img[..., 1] == 200).tobytes())
    return h.hexdigest()


def cv2_circle_sha() -> str:
    import cv2
    h = hashlib.sha256()
    for c in grid_points(9, 7, 3):
        img = np.zeros((7, 9, 3), np.uint8)
        cv2.circle(img, c, 3, COLOUR, 1)
        h.update(np.packbits(img[..., 1] == 200).tobytes())
    return h.hexdigest()


def build() -> dict:
    import cv2
    g = {}
    base, pl, spl, epl = kitti_inputs()
    img = cv2_plot(base, pl, spl, epl)
    g.update(kitti_seed=np.int64(2024), kitti_pl=pl, kitti_spl=spl, kitti_epl=epl,
             kitti_mask=np.packbits(np.any(img != base, -1) | np.all(img == COLOUR, -1)))
    g["grid_sha"] = np.str_(cv2_grid_sha())
    g["circle_sha"] = np.str_(cv2_circle_sha())
    for c in (3, 4):
        seed = 70 + c
        src = MC.color_image(seed, 64, 48, c)
        m1, m2 = MC.own_maps(64, 48, seed)
        out = cv2.remap(src, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        out = out if c == 3 else cv2.cvtColor(out, cv2.COLOR_BGRA2BGR)
        g.update({f"remap{c}_seed": np.int64(seed), f"remap{c}_map1": m1, f"remap{c}_map2": m2, f"remap{c}_out": out})
    return g


if __name__ == "__main__":
    import cv2
    assert cv2.__version__.startswith("4.13"), cv2.__version__
    np.savez_compressed(OUT, **build())
    print("wrote", OUT)
