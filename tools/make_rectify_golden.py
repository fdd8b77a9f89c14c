"""Writes tests/golden/rectify.npz: OpenCV 4.13's CV_16SC2 undistort-rectify maps (cv2.initUndistortRectifyMap,
cv2.fisheye.initUndistortRectifyMap) for the rigs PinholeStereoCamera builds, and cv2.remap(INTER_LINEAR) of seeded images
on them and on random cv2.convertMaps maps whose taps leave the image on every side.

Large maps and remapped images are recorded by SHA-256 (the images are regenerated from their seeds by image()); small ones
in full.  Per case c:
  c_model, c_K, c_D, c_R, c_P, c_size (w, h)      the map builder's inputs (maps cases)
  c_map_sha / c_map1, c_map2                      the maps (map1 bytes then map2 bytes)
  c_seed, c_out_sha / c_out                       cv2.remap of image(seed, w, h) on the maps
  c_cam                                           rectified fx, fy, cx, cy, b where the case is a whole rig side

    python tools/make_rectify_golden.py            # needs cv2; rewrites tests/golden/rectify.npz
"""
from __future__ import annotations

import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "rectify.npz")
FULL = 64 * 64   # pixels up to which maps and outputs are stored in full

# The EuRoC MAV dataset's published calibration of its stereo pair (cam0, cam1): intrinsics fx, fy, cx, cy, radial-tangential
# coefficients, and the rotation / translation between the two cameras, as the dataset's own yaml gives them.
EUROC_SIZE = (752, 480)
EUROC_KL = (458.654, 457.296, 367.215, 248.375)
EUROC_KR = (457.587, 456.134, 379.999, 255.238)
EUROC_DL = (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05)
EUROC_DR = (-0.28368365, 0.07451284, -0.00010473, -3.55590700e-05)
EUROC_R = ((9.99997256e-01, 2.31206719e-03, 3.76008102e-04), (-2.31713572e-03, 9.99898049e-01, 1.40898358e-02),
           (-3.43393121e-04, -1.40906685e-02, 9.99900663e-01))
EUROC_T = (-0.11007381, 0.00039912, -0.0008537)
EUROC_BL = 0.110077842
# KITTI 00-02's rectified left camera, with a radial-tangential distortion put on it (cam_d0 branch)
KITTI_SIZE = (1241, 376)
KITTI_K = (718.856, 718.856, 607.1928, 185.2157)
KITTI_D = (-0.12, 0.04, 0.0006, -0.0004)


def image(seed: int, w: int, h: int) -> np.ndarray:
    """A seeded grey test image: smooth texture plus noise, so every interpolation weight matters."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    base = 127 + 60 * np.sin(x / 7.3 + rng.uniform(0, 6)) * np.cos(y / 5.1 + rng.uniform(0, 6))
    return np.clip(base + rng.normal(0, 40, (h, w)), 0, 255).astype(np.uint8)


def sha(*arrays) -> np.ndarray:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), np.uint8)


def kmat(fx, fy, cx, cy, dtype=np.float64):
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype)


def euroc_rig():
    """What PinholeStereoCamera's Kl branch builds: K in float (Mat_<float>), D double, R / P from stereoRectify with
    CALIB_ZERO_DISPARITY, alpha 0.  Returns (left (K, D, R, P), right (...), rectified (fx, fy, cx, cy, b))."""
    import cv2
    Kl, Kr = kmat(*EUROC_KL, np.float32), kmat(*EUROC_KR, np.float32)
    Dl, Dr = np.array(EUROC_DL), np.array(EUROC_DR)
    Rl, Rr, Pl, Pr, _, _, _ = cv2.stereoRectify(Kl, Dl, Kr, Dr, EUROC_SIZE, np.array(EUROC_R), np.array(EUROC_T),
                                                flags=cv2.CALIB_ZERO_DISPARITY, alpha=0)
    cam = (Pl[0, 0], Pl[1, 1], Pl[0, 2], Pl[1, 2], EUROC_BL)
    return (Kl, Dl, Rl, Pl), (Kr, Dr, Rr, Pr), cam


def d0_rig():
    """The cam_d0 branch: K, D (5 coefficients, the last 0) and P in float, P's fy = fx, R = I."""
    fx, fy, cx, cy = KITTI_K
    K = kmat(fx, fy, cx, cy, np.float32)
    D = np.array(list(KITTI_D) + [0.0], np.float32)
    P = np.array([[fx, 0, cx, 0], [0, fx, cy, 0], [0, 0, 1, 0]], np.float32)
    return K, D, np.eye(3), P


def map_cases():
    """(name, model, K, D, R, P, (w, h), cam or None)"""
    import cv2
    rng = np.random.default_rng(77)
    (Kl, Dl, Rl, Pl), (Kr, Dr, Rr, Pr), cam = euroc_rig()
    out = [("euroc_l", 0, Kl, Dl, Rl, Pl, EUROC_SIZE, cam), ("euroc_r", 0, Kr, Dr, Rr, Pr, EUROC_SIZE, cam)]
    K, D, R, P = d0_rig()
    out.append(("kitti_d0", 0, K, D, R, P, KITTI_SIZE, (KITTI_K[0], KITTI_K[0], KITTI_K[2], KITTI_K[3], 0.537)))
    Kp = kmat(430.3, 428.9, 160.7, 101.2)
    Rs = cv2.Rodrigues(rng.normal(0, 0.03, 3))[0]
    Pp = np.hstack([kmat(400.1, 400.1, 158.3, 99.6), np.zeros((3, 1))])
    out.append(("pin5", 0, Kp, [-0.31, 0.12, 0.001, -0.002, -0.02], Rs, Pp, (321, 203), None))
    out.append(("pin8", 0, Kp, [0.9, -0.3, 0.001, 0.002, 0.05, 1.2, -0.2, 0.03], Rs, Pp, (321, 203), None))
    # the reference's dtype branch: pinhole stereoRectify, then the fisheye maps
    Kf = kmat(*EUROC_KL, np.float32)
    Df = np.array([-0.01, 0.02, -0.003, 0.0004])
    Rf, _, Pf, _, _, _, _ = cv2.stereoRectify(Kf, Df, kmat(*EUROC_KR, np.float32), Df, EUROC_SIZE, np.array(EUROC_R),
                                              np.array(EUROC_T), flags=cv2.CALIB_ZERO_DISPARITY, alpha=0)
    out.append(("fisheye", 1, Kf, Df, Rf, Pf, EUROC_SIZE, None))
    # tiny and odd sizes, both models
    for w, h in ((1, 1), (2, 3), (5, 7), (8, 8), (13, 11), (17, 1)):
        Ks = kmat(0.9 * w + 1.3, 0.8 * h + 1.7, w / 2 - 0.3, h / 2 + 0.2)
        Ps = kmat(0.8 * w + 1.1, 0.8 * w + 1.1, w / 2 + 0.1, h / 2 - 0.1)
        out.append((f"pin_{w}x{h}", 0, Ks, [-0.2, 0.05, 0.001, 0.001], Rs, Ps, (w, h), None))
        out.append((f"fish_{w}x{h}", 1, Ks, [0.05, -0.01, 0.002, 0.0], Rs, Ps, (w, h), None))
    # far outside the image: short and int saturation in the pinhole builder, behind the camera in the fisheye one
    Kx = kmat(400.3, 401.7, 300.2, 200.9)
    Px = np.hstack([kmat(40.37, 40.37, 300.71, 200.33), np.zeros((3, 1))])
    out.append(("pin_saturate", 0, Kx, [0.9, 0.9, 0.0013, 0.0011, 0.9], np.eye(3), Px, (203, 131), None))
    out.append(("pin_saturate8", 0, Kx, [0.5, 0.5, 0.011, 0.013, 0.5, 0.0, 0.0, 0.0], np.eye(3), Px, (203, 131), None))
    Rb = cv2.Rodrigues(np.array([0.0, 1.7, 0.0]))[0]
    out.append(("fish_behind", 1, Kx, [0.1, 0.01, 0.001, 0.0001], Rb, Px * 10, (203, 131), None))
    return out


def remap_cases():
    """(name, (w, h), map1, map2): cv2.convertMaps of random float maps, taps beyond every edge, some far out"""
    import cv2
    out = []
    for k, (w, h) in enumerate(((1, 1), (3, 2), (8, 8), (37, 53), (64, 48))):
        rng = np.random.default_rng(500 + k)
        mx = rng.uniform(-3, w + 2, (h, w)).astype(np.float32)
        my = rng.uniform(-3, h + 2, (h, w)).astype(np.float32)
        far = rng.random((h, w)) < 0.1
        mx[far] = rng.uniform(-32000, 32000, far.sum())
        m1, m2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        out.append((f"remap_{w}x{h}", (w, h), m1, m2))
    return out


def main():
    import cv2
    assert cv2.__version__.startswith("4.13"), cv2.__version__
    z = {}
    names = []
    for seed, (name, model, K, D, R, P, (w, h), cam) in enumerate(map_cases()):
        build = cv2.fisheye.initUndistortRectifyMap if model == 1 else cv2.initUndistortRectifyMap
        m1, m2 = build(K, np.asarray(D), R, P, (w, h), cv2.CV_16SC2)
        img = image(seed, w, h)
        out = cv2.remap(img, m1, m2, cv2.INTER_LINEAR)
        P34 = np.asarray(P, np.float64)
        z[f"{name}_model"] = np.int32(model)
        z[f"{name}_K"] = np.asarray(K, np.float64)
        z[f"{name}_D"] = np.asarray(D, np.float64).ravel()
        z[f"{name}_R"] = np.asarray(R, np.float64)
        z[f"{name}_P"] = P34 if P34.shape == (3, 4) else np.hstack([P34, np.zeros((3, 1))])
        z[f"{name}_size"] = np.int32([w, h])
        z[f"{name}_seed"] = np.int32(seed)
        z[f"{name}_map_sha"] = sha(m1, m2)
        z[f"{name}_out_sha"] = sha(out)
        if w * h <= FULL:
            z[f"{name}_map1"], z[f"{name}_map2"], z[f"{name}_out"] = m1, m2, out
        if cam is not None:
            z[f"{name}_cam"] = np.float64(cam)
        names.append(name)
    remaps = []
    for k, (name, (w, h), m1, m2) in enumerate(remap_cases()):
        img = image(1000 + k, w, h)
        z[f"{name}_size"] = np.int32([w, h])
        z[f"{name}_seed"] = np.int32(1000 + k)
        z[f"{name}_map1"], z[f"{name}_map2"] = m1, m2
        z[f"{name}_out"] = cv2.remap(img, m1, m2, cv2.INTER_LINEAR)
        remaps.append(name)
    z["map_cases"] = np.array(names)
    z["remap_cases"] = np.array(remaps)
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
