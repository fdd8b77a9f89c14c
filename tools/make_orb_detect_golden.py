"""Writes tests/golden/orb_detect.npz from cv2's ORB::detectAndCompute (needs cv2).

Images come from tests/orb_images.py and tools/make_orb_golden.py (seeded, integer-only); the file keeps their SHA-256, not
their pixels.  Each case stores cv2's key points sorted into canonical order (octave, then y, then x): pt, angle and response
as float32 bits, octave and descriptors, per-image offsets, and the ORB parameters.
  default_fast / default_harris: two 640x480 images, the default config (1200 features, 4 levels, 1.2), FAST / Harris;
                                 image 0 level 0 keeps 388 points for a budget of 386 (FAST score ties)
  kitti:  the four views of make_orb_golden.kitti_views() at config_kitti.yaml (2000 features, 1 level), FAST
  euroc:  two 752x480 images, 800 features, 4 levels, FAST
  th5 / th50: one 640x480 image at FAST thresholds 5 and 50

    python tools/make_orb_detect_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_orb_golden as M  # noqa: E402
import orb_images as I  # noqa: E402
import ref_orb_detect as R  # noqa: E402


def cases():
    """name -> (images, ORB parameters)"""
    one = M.default_images()
    return {
        "default_fast": (one, dict(n_features=1200, n_levels=4, scale=1.2, score_type=R.FAST_SCORE, fast_threshold=20)),
        "default_harris": (one, dict(n_features=1200, n_levels=4, scale=1.2, score_type=R.HARRIS_SCORE, fast_threshold=20)),
        "kitti": (M.kitti_views(), dict(n_features=2000, n_levels=1, scale=1.2, score_type=R.FAST_SCORE, fast_threshold=20)),
        "euroc": (np.stack([I.make_image(752, 480, s) for s in (21, 22)]),
                  dict(n_features=800, n_levels=4, scale=1.2, score_type=R.FAST_SCORE, fast_threshold=20)),
        "th5": (I.make_image(640, 480, 3)[None], dict(n_features=1200, n_levels=4, scale=1.2, score_type=R.FAST_SCORE,
                                                      fast_threshold=5)),
        "th50": (I.make_image(640, 480, 3)[None], dict(n_features=1200, n_levels=4, scale=1.2, score_type=R.FAST_SCORE,
                                                       fast_threshold=50)),
    }


def golden():
    import cv2
    rec = dict(cv2_version=np.array(cv2.__version__), names=np.array(list(cases())))
    for name, (images, p) in cases().items():
        res = [R.cv2_detect(cv2, im, **p) for im in images]
        rec[f"{name}_sha256"] = np.array([I.sha256(im) for im in images])
        rec[f"{name}_params"] = np.array([p["n_features"], p["n_levels"], p["score_type"], p["fast_threshold"]], np.int32)
        rec[f"{name}_scale"] = np.float64(p["scale"])
        rec[f"{name}_off"] = np.cumsum([0] + [len(r["xy"]) for r in res]).astype(np.int32)
        rec[f"{name}_xy_bits"] = np.concatenate([r["xy"] for r in res]).view(np.uint32)
        rec[f"{name}_octave"] = np.concatenate([r["octave"] for r in res])
        rec[f"{name}_angle_bits"] = np.concatenate([r["angle"] for r in res]).view(np.uint32)
        rec[f"{name}_response_bits"] = np.concatenate([r["response"] for r in res]).view(np.uint32)
        rec[f"{name}_desc"] = np.concatenate([r["desc"] for r in res])
    return rec


if __name__ == "__main__":
    out = os.path.join(ROOT, "tests", "golden", "orb_detect.npz")
    np.savez_compressed(out, **golden())
    print(out, os.path.getsize(out), "bytes")
