"""Writes tests/golden/lbd.npz: LBD descriptors of the reference's BinaryDescriptor::compute (default Params, octave 0),
computed by the library oracle/make_ref_lbd.py builds from the reference's own text.  Needs cv2 (the LSD key lines) and
that library.

Images come from tests/orb_images.make_image (seeded, integer-only) or are constant; the file keeps their SHA-256, not
their pixels (case_images() rebuilds them).  Cases, each a batch of images of one size:
  kitti_300 / kitti_100  two 1241x376 images, cv2 LSD key lines with the reference's options, sorted by response and
                         truncated to 300 (default config) and 100 (KITTI config)
  euroc_300              two 752x480 images, the same recipe
  kitti_stereo           the left / right images of the two stereo frames of tests/golden/orb_kitti.npz, the same recipe
                         (the end-to-end tracking test feeds them to plstvo_track_stereo_batch)
  synthetic              a textured 640x480 image and a flat one, hand-placed lines: horizontal, vertical, 45 degrees,
                         through the corners, clamped to the border, 1-pixel, full-width, angles other than atan2 of the
                         segment; the flat image gives the all-zero descriptor
  tiny_WxH               1..8 pixel images with lines across and outside them
  trig_binding           a textured 640x480 image and lines whose descriptor depends on which cos / sin the reference's
                         unqualified cos(float) binds to: glibc's cosf / sinf (what it binds to, through the <math.h> its
                         translation unit includes) and (float)cos((double)angle) give different bytes on each of them

    python tools/make_lbd_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import orb_images as I  # noqa: E402

TINY = [(1, 1), (1, 6), (6, 1), (2, 3), (3, 8), (5, 5), (8, 8), (7, 4)]
# (name, W, H, image seeds (None: flat 128), LSD truncation (None: synthetic lines))
CASES = [("kitti_300", 1241, 376, (21, 22), 300), ("kitti_100", 1241, 376, (21, 22), 100),
         ("euroc_300", 752, 480, (23, 24), 300), ("kitti_stereo", 1241, 376, "kitti_views", 300), ("synthetic", 640, 480, (25, None), None)] + \
        [(f"tiny_{w}x{h}", w, h, (30 + w, 40 + h), None) for w, h in TINY] + [("trig_binding", 640, 480, (61,), None)]
# lines of trig_lines()'s seeded pool on which the two bindings give different descriptors, found by building the reference
# once more without <math.h> (so that cos(float) took the C double cos) and comparing the two libraries over the pool
TRIG_PICK = [640, 229463, 304007, 366975, 439540, 445214, 467122, 478144, 501678, 559865]


def case_images(W, H, seeds):
    if isinstance(seeds, str) or (len(seeds) == 1 and seeds[0] == -2):   # the stereo frames of tests/golden/orb_kitti.npz
        import make_orb_golden
        return make_orb_golden.kitti_views()
    return np.stack([np.full((H, W), 128, np.uint8) if s is None else I.make_image(W, H, s) for s in seeds])


def line_pixels(x0, y0, x1, y1):
    """cv::LineIterator(img, Point2f(p0), Point2f(p1)).count, 8-connected, for end points inside the image: the points are
    cvRound'ed (half to even) and the count is max(|dx|, |dy|) + 1."""
    a = np.rint(np.float64([x0, y0, x1, y1])).astype(np.int64)
    return int(max(abs(a[2] - a[0]), abs(a[3] - a[1])) + 1)


def lsd_keylines(img, n_keep):
    """LSDDetectorC::detect(img, lines, 1, 1, opts) with the reference's options (src/config.cpp:103-112), min length
    0.025 min(W, H), then the sort-by-response-and-truncate of StereoFrame::detectLineFeatures."""
    import cv2
    H, W = img.shape
    lsd = cv2.createLineSegmentDetector(0, 1.2, 0.6, 2.0, 22.5, 1.0, 0.6, 1024)
    segs = lsd.detect(img)[0]
    segs = np.zeros((0, 4), np.float32) if segs is None else segs.reshape(-1, 4).astype(np.float32)
    segs[:, 0::2] = np.where(segs[:, 0::2] < 0, 0, np.where(segs[:, 0::2] >= W, np.float32(W - 1), segs[:, 0::2]))
    segs[:, 1::2] = np.where(segs[:, 1::2] < 0, 0, np.where(segs[:, 1::2] >= H, np.float32(H - 1), segs[:, 1::2]))
    d = segs[:, :2] - segs[:, 2:]
    length = np.sqrt(d[:, 0].astype(np.float64) ** 2 + d[:, 1].astype(np.float64) ** 2).astype(np.float32)
    keep = length.astype(np.float64) > 0.025 * min(W, H)
    segs, length = segs[keep], length[keep]
    angle = np.arctan2((segs[:, 3] - segs[:, 1]).astype(np.float64), (segs[:, 2] - segs[:, 0]).astype(np.float64)).astype(np.float32)
    npix = np.array([line_pixels(*s) for s in segs], np.int32)
    response = length / np.float32(max(W, H))
    order = np.argsort(-response, kind="stable")[:n_keep]
    return segs[order], angle[order], npix[order]


def synthetic_lines(W, H, seed):
    """Hand-placed lines, then seeded random ones (with angles off the segment's own) to fill up."""
    L = []   # (x0, y0, x1, y1, angle or None (atan2), npix or None (line_pixels))
    L += [(100, 200, 300, 200, None, None), (300, 200, 100, 200, None, None)]           # horizontal, both directions
    L += [(50, 40, 50, 400, None, None), (600.5, 420, 600.5, 30, None, None)]          # vertical
    L += [(10, 10, 300, 300, None, None), (400, 50, 200, 250, None, None)]             # 45 degrees
    L += [(0, 0, W - 1, H - 1, None, None), (W - 1, 0, 0, H - 1, None, None)]          # corner to corner
    L += [(0, 3, 120, 3, None, None), (W - 1, 100, W - 1, 300, None, None), (5, H - 1, 200, H - 2, None, None)]
    L += [(320, 240, 320, 240, 0.0, 1), (10.4, 470.6, 10.4, 470.6, 2.0, 1), (0, 0, 0, 0, -1.0, 1)]   # 1-pixel
    L += [(0, 240, W - 1, 240, None, None), (0, 100.25, W - 1, 101.75, None, None)]     # full width
    L += [(100, 100, 200, 120, 1.0, None), (150, 300, 250, 300, -2.5, None), (400, 400, 500, 350, 3.14159, 77)]
    rng = np.random.default_rng(seed)
    for _ in range(40):
        x0, x1 = rng.uniform(-0.4, W - 0.6, 2)
        y0, y1 = rng.uniform(-0.4, H - 0.6, 2)
        ang = None if rng.random() < 0.5 else float(rng.uniform(-np.pi, np.pi))
        L.append((x0, y0, x1, y1, ang, None))
    return _pack(L)


def trig_lines(W, H):
    """TRIG_PICK out of a seeded pool of 600 000 lines with exponential lengths and uniform float angles."""
    rng = np.random.default_rng(62)
    n = 600000
    length = 8.0 + rng.exponential(40.0, n)
    th = rng.uniform(-np.pi, np.pi, n).astype(np.float32)
    cx, cy = rng.uniform(0, W - 1, n), rng.uniform(0, H - 1, n)
    seg = np.stack([cx - 0.5 * length * np.cos(th), cy - 0.5 * length * np.sin(th),
                    cx + 0.5 * length * np.cos(th), cy + 0.5 * length * np.sin(th)], 1)
    seg[:, 0::2] = np.clip(seg[:, 0::2], 0, W - 1)
    seg[:, 1::2] = np.clip(seg[:, 1::2], 0, H - 1)
    seg = seg.astype(np.float32)[TRIG_PICK]
    return seg, th[TRIG_PICK], np.array([line_pixels(*s) for s in seg], np.int32)


def tiny_lines(W, H):
    L = [(0, 0, W - 1, H - 1, None, None), (W - 1, 0, 0, H - 1, None, None), (0, 0, 0, 0, 0.5, 1),
         (-3, H / 2, W + 3, H / 2, 0.0, W + 7), (W / 2, -2, W / 2, H + 2, 1.5707964, H + 5), (0, 0, W - 1, 0, 2.2, 9),
         (W * 0.5, H * 0.5, W * 0.5 + 0.1, H * 0.5 + 0.1, -0.7, 40)]
    return _pack(L)


def _pack(L):
    seg = np.array([l[:4] for l in L], np.float32)
    ang = np.array([np.arctan2(np.float64(s[3] - s[1]), np.float64(s[2] - s[0])) if l[4] is None else l[4]
                    for s, l in zip(seg, L)]).astype(np.float32)
    npix = np.array([line_pixels(*s) if l[5] is None else l[5] for s, l in zip(seg, L)], np.int32)
    return seg, ang, npix


def case_lines(name, W, H, images, n_keep):
    out = []
    for i, img in enumerate(images):
        if n_keep is not None:
            out.append(lsd_keylines(img, n_keep))
        elif name == "synthetic":
            out.append(synthetic_lines(W, H, 77))
        elif name == "trig_binding":
            out.append(trig_lines(W, H))
        else:
            out.append(tiny_lines(W, H))
    return out


def golden():
    import cv2
    from oracle import lbd
    rec = dict(cv2_version=np.array(cv2.__version__), cases=np.array([c[0] for c in CASES]))
    for name, W, H, seeds, n_keep in CASES:
        images = case_images(W, H, seeds)
        per = case_lines(name, W, H, images, n_keep)
        off = np.cumsum([0] + [len(p[0]) for p in per]).astype(np.int32)
        seg = np.concatenate([p[0] for p in per]).reshape(-1, 4)
        ang = np.concatenate([p[1] for p in per])
        npix = np.concatenate([p[2] for p in per])
        desc = lbd.compute_batch(images, off, seg, ang, npix)
        rec.update({f"{name}/size": np.int32([W, H]),
                    f"{name}/seeds": np.int32([-2] if isinstance(seeds, str) else [-1 if s is None else s for s in seeds]),
                    f"{name}/sha256": np.array([I.sha256(im) for im in images]),
                    f"{name}/kl_off": off, f"{name}/seg": seg, f"{name}/angle_bits": ang.view(np.uint32),
                    f"{name}/npix": npix, f"{name}/desc": desc})
    return rec


def load_case(g, name):
    """(images, kl_off, seg, angle, npix, desc) of one case of a loaded golden file."""
    W, H = (int(v) for v in g[f"{name}/size"])
    seeds = [int(s) for s in g[f"{name}/seeds"]]
    images = case_images(W, H, seeds if seeds == [-2] else [None if s < 0 else s for s in seeds])
    assert [I.sha256(im) for im in images] == list(g[f"{name}/sha256"]), f"{name}: images differ from the recorded SHA-256"
    return (images, g[f"{name}/kl_off"], g[f"{name}/seg"], g[f"{name}/angle_bits"].view(np.float32), g[f"{name}/npix"],
            g[f"{name}/desc"])


if __name__ == "__main__":
    path = os.path.join(ROOT, "tests", "golden", "lbd.npz")
    np.savez_compressed(path, **golden())
    print(path, os.path.getsize(path), "bytes")
