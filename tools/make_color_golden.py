"""Writes tests/golden/color.npz: cv2 4.13's cvtColor(remap(img), COLOR_BGR2GRAY), and cvtColor alone, of seeded 3- and
4-channel images: what Dataset::nextFrame and the reference's detectors make of a colour frame.

Maps come from tests/golden/rectify.npz's cases where they fit (the EuRoC rig's two sides, the fisheye rig, the KITTI-size
cam_d0 map, the tiny pinhole and fisheye rigs, and its random remap maps whose taps leave the image on every side), or are
cv2.convertMaps maps drawn here (sizes 1x1 to 17x1 and others whose 3 W is not a multiple of 4 or 16, taps beyond every
edge).  Per case c:
  c_channels, c_size (w, h), c_seed            color_image(seed, w, h, channels) is the input
  c_rig                                         the rectify.npz case whose maps are used, "" for c_map1 / c_map2, "-" for none
  c_map1, c_map2                                the maps drawn here
  c_out / c_out_sha                             the grey result, in full up to 64 x 64 pixels, else its SHA-256

    python tools/make_color_golden.py            # needs cv2; rewrites tests/golden/color.npz
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_rectify_golden as M  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "color.npz")
FULL = 64 * 64

RIGS = ["euroc_l", "euroc_r", "fisheye", "kitti_d0", "pin_1x1", "pin_2x3", "pin_5x7", "pin_13x11", "pin_17x1", "fish_8x8",
        "fish_13x11", "remap_1x1", "remap_3x2", "remap_8x8", "remap_37x53", "remap_64x48"]
OWN = [(w, 1) for w in range(1, 18)] + [(5, 3), (7, 9), (21, 4), (45, 2)]
PLAIN = [(w, 1) for w in range(1, 18)] + [(5, 7), (13, 11), (37, 53), (1241, 376), (752, 480)]


def color_image(seed: int, w: int, h: int, channels: int) -> np.ndarray:
    """A seeded colour test image, uint8[h, w, channels] (B, G, R[, A]): a different smooth texture plus noise per colour
    channel, so the grey value differs from each channel, and random alpha."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    planes = []
    for _ in range(3):
        base = 127 + 60 * np.sin(x / rng.uniform(4, 9) + rng.uniform(0, 6)) * np.cos(y / rng.uniform(4, 9) + rng.uniform(0, 6))
        planes.append(np.clip(base + rng.normal(0, 40, (h, w)), 0, 255))
    if channels == 4:
        planes.append(rng.integers(0, 256, (h, w)).astype(np.float64))
    return np.stack(planes, -1).astype(np.uint8)


def own_maps(w: int, h: int, seed: int):
    """cv2.convertMaps of random float maps: taps up to 3 pixels beyond every edge, a tenth of them far out"""
    import cv2
    rng = np.random.default_rng(seed)
    mx = rng.uniform(-3, w + 2, (h, w)).astype(np.float32)
    my = rng.uniform(-3, h + 2, (h, w)).astype(np.float32)
    far = rng.random((h, w)) < 0.1
    mx[far] = rng.uniform(-32000, 32000, far.sum())
    return cv2.convertMaps(mx, my, cv2.CV_16SC2)


def rectify_maps(name: str):
    """the CV_16SC2 maps of rectify.npz's case `name`, as cv2 builds them"""
    import cv2
    for c, model, K, D, R, P, (w, h), _ in M.map_cases():
        if c == name:
            build = cv2.fisheye.initUndistortRectifyMap if model == 1 else cv2.initUndistortRectifyMap
            return build(K, np.asarray(D), R, P, (w, h), cv2.CV_16SC2)
    for c, _, m1, m2 in M.remap_cases():
        if c == name:
            return m1, m2
    raise KeyError(name)


def main():
    import cv2
    assert cv2.__version__.startswith("4.13"), cv2.__version__
    z, names = {}, []
    seed = 7000

    def add(name, channels, w, h, rig, m1, m2):
        nonlocal seed
        seed += 1
        img = color_image(seed, w, h, channels)
        src = img if m1 is None else cv2.remap(img, m1, m2, cv2.INTER_LINEAR)
        out = cv2.cvtColor(src, cv2.COLOR_BGR2GRAY)   # the detectors' code, on 3 or 4 channels alike
        z[f"{name}_channels"], z[f"{name}_size"], z[f"{name}_seed"] = np.int32(channels), np.int32([w, h]), np.int32(seed)
        z[f"{name}_rig"] = np.array(rig)
        if rig == "":
            z[f"{name}_map1"], z[f"{name}_map2"] = m1, m2
        if w * h <= FULL:
            z[f"{name}_out"] = out
        else:
            z[f"{name}_out_sha"] = M.sha(out)
        names.append(name)

    for channels in (3, 4):
        for rig in RIGS:
            m1, m2 = rectify_maps(rig)
            h, w = m2.shape
            add(f"c{channels}_{rig}", channels, w, h, rig, m1, m2)
        for k, (w, h) in enumerate(OWN):
            m1, m2 = own_maps(w, h, 900 + 10 * k + channels)
            add(f"c{channels}_own_{w}x{h}", channels, w, h, "", m1, m2)
        for w, h in PLAIN:
            add(f"c{channels}_plain_{w}x{h}", channels, w, h, "-", None, None)
    z["cases"] = np.array(names)
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
