"""NumPy restatement of what PinholeStereoCamera::rectifyImagesLR computes: OpenCV 4.13's CV_16SC2 undistort-rectify maps
(cv::initUndistortRectifyMap and cv::fisheye::initUndistortRectifyMap) and cv::remap's INTER_LINEAR on them with
BORDER_CONSTANT 0, for 8-bit grey images.

Every step is a separate IEEE double operation (NumPy ufuncs never fuse), in the order OpenCV evaluates it, so the maps
equal OpenCV's bit for bit; the remap is integer arithmetic.  plstvo_init_undistort_rectify_map and rectify_remap_kernel are
held to this module.
"""
from __future__ import annotations

import numpy as np

PINHOLE, FISHEYE = 0, 1
INTER_BITS, INTER_TAB_SIZE = 5, 32
INT_MIN, INT_MAX = -(2 ** 31), 2 ** 31 - 1
# cv::initUndistortRectifyMap's vector loop in OpenCV's x86-64 build dispatched for AVX2: two 4-lane double vectors per
# step.  cv::fisheye::initUndistortRectifyMap has no vector loop.
PINHOLE_LANES = 8


def inv3(m) -> list:
    """cv::invert(DECOMP_LU) of a 3x3 double matrix: the cofactor form OpenCV takes for n == 3 (row-major list of 9
    Python floats; None when the determinant is 0)."""
    m = [[float(m[i][j]) for j in range(3)] for i in range(3)]
    d = (m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0])
         + m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]))
    if d == 0.0:
        return None
    d = 1.0 / d
    return [(m[1][1] * m[2][2] - m[1][2] * m[2][1]) * d, (m[0][2] * m[2][1] - m[0][1] * m[2][2]) * d,
            (m[0][1] * m[1][2] - m[0][2] * m[1][1]) * d,
            (m[1][2] * m[2][0] - m[1][0] * m[2][2]) * d, (m[0][0] * m[2][2] - m[0][2] * m[2][0]) * d,
            (m[0][2] * m[1][0] - m[0][0] * m[1][2]) * d,
            (m[1][0] * m[2][1] - m[1][1] * m[2][0]) * d, (m[0][1] * m[2][0] - m[0][0] * m[2][1]) * d,
            (m[0][0] * m[1][1] - m[0][1] * m[1][0]) * d]


def mul3(a, b) -> list:
    """The 3x3 product a @ b in double, each entry summed left to right (no BLAS, which may fuse)."""
    return [[float(a[i][0]) * float(b[0][j]) + float(a[i][1]) * float(b[1][j]) + float(a[i][2]) * float(b[2][j])
             for j in range(3)] for i in range(3)]


def _cv_round(v: np.ndarray) -> np.ndarray:
    """saturate_cast<int>(double), which is cvRound: round half to even; on x86-64 (cvtsd2si) a result outside int32, or
    NaN, is INT_MIN."""
    r = np.rint(v)
    out = np.full(v.shape, INT_MIN, dtype=np.int64)
    ok = (r >= INT_MIN) & (r <= INT_MAX)
    out[ok] = r[ok].astype(np.int64)
    return out


def _pack(u: np.ndarray, v: np.ndarray, simd_cols: int):
    """The CV_16SC2 pair.  Columns below simd_cols took OpenCV's vector loop, which packs iu >> 5 to short with
    saturation; the others its scalar loop, which truncates to short."""
    iu = _cv_round(u * float(INTER_TAB_SIZE))
    iv = _cv_round(v * float(INTER_TAB_SIZE))
    su, sv = iu >> INTER_BITS, iv >> INTER_BITS
    vec = np.arange(u.shape[1])[None, :] < simd_cols
    su = np.where(vec, np.clip(su, -32768, 32767), su)
    sv = np.where(vec, np.clip(sv, -32768, 32767), sv)
    m1 = np.stack([su.astype(np.int16), sv.astype(np.int16)], axis=-1)
    m2 = ((iv & (INTER_TAB_SIZE - 1)) * INTER_TAB_SIZE + (iu & (INTER_TAB_SIZE - 1))).astype(np.uint16)
    return m1, m2


def _row_coords(ir, width: int, height: int, lanes: int):
    """Per pixel X, Y, W, and how many leading columns took the vector loop.  Row i starts at i*ir[1] + ir[2] (likewise
    for Y and W).  OpenCV's vector loop (lanes > 0) takes the row in blocks of `lanes` pixels: lane k of a block is
    start + k*ir[0], and the start moves on by lanes*ir[0]; the columns left over, and a loop without lanes, add ir[0]
    once per pixel."""
    i = np.arange(height, dtype=np.float64)
    simd_cols = width - width % lanes if lanes else 0
    out = []
    for c in range(3):
        d = ir[3 * c]
        cur = i * ir[3 * c + 1] + ir[3 * c + 2]
        acc = np.empty((height, width), dtype=np.float64)
        j = 0
        while j < simd_cols:
            for k in range(lanes):
                acc[:, j + k] = cur + float(k) * d
            cur = cur + float(lanes) * d
            j += lanes
        while j < width:
            acc[:, j] = cur
            cur = cur + d
            j += 1
        out.append(acc)
    return out, simd_cols


def init_undistort_rectify_map(model: int, K, D, R, P, width: int, height: int):
    """(map1 int16 [h][w][2], map2 uint16 [h][w]) as OpenCV returns them for m1type CV_16SC2.  K 3x3, D the 4 / 5 / 8
    coefficients (fisheye: 4), R 3x3, P 3x3 or 3x4 (first three columns).  Raises ValueError where the library returns
    PLSTVO_E_INVALID."""
    D = [float(d) for d in np.asarray(D, dtype=np.float64).ravel()]
    if model == PINHOLE and len(D) not in (4, 5, 8):
        raise ValueError("pinhole takes 4, 5 or 8 coefficients")
    if model == FISHEYE and len(D) != 4:
        raise ValueError("fisheye takes 4 coefficients")
    if not (1 <= width <= 32767 and 1 <= height <= 32767):
        raise ValueError("size must be 1..32767")
    K = np.asarray(K, dtype=np.float64)
    Pm = np.asarray(P, dtype=np.float64)[:, :3]
    ir = inv3(mul3(Pm, np.asarray(R, dtype=np.float64)))
    if ir is None:
        raise ValueError("singular P * R")
    fx, fy, u0, v0 = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    (X, Y, W), simd_cols = _row_coords(ir, width, height, PINHOLE_LANES if model == PINHOLE else 0)
    with np.errstate(all="ignore"):
        if model == PINHOLE:
            k = D + [0.0] * (8 - len(D))
            k1, k2, p1, p2, k3, k4, k5, k6 = k
            w = 1.0 / W
            x = X * w
            y = Y * w
            x2 = x * x
            y2 = y * y
            r2 = x2 + y2
            _2xy = 2.0 * x * y
            kr = (1.0 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1.0 + ((k6 * r2 + k5) * r2 + k4) * r2)
            xd = x * kr + p1 * _2xy + p2 * (r2 + 2.0 * x2)
            yd = y * kr + p1 * (r2 + 2.0 * y2) + p2 * _2xy
            u = fx * xd + u0
            v = fy * yd + v0
        else:
            x = X / W
            y = Y / W
            r = np.sqrt(x * x + y * y)
            theta = np.arctan(r)
            t2 = theta * theta
            t4 = t2 * t2
            t6 = t4 * t2
            t8 = t4 * t4
            theta_d = theta * (1.0 + D[0] * t2 + D[1] * t4 + D[2] * t6 + D[3] * t8)
            scale = np.where(r == 0, 1.0, theta_d / r)
            u = fx * x * scale + u0
            v = fy * y * scale + v0
            behind = W <= 0
            u = np.where(behind, np.where(X > 0, -np.inf, np.inf), u)
            v = np.where(behind, np.where(Y > 0, -np.inf, np.inf), v)
    return _pack(u, v, simd_cols)


def remap(img: np.ndarray, map1: np.ndarray, map2: np.ndarray) -> np.ndarray:
    """cv::remap(img, map1, map2, INTER_LINEAR, BORDER_CONSTANT, 0) of an 8-bit grey image on CV_16SC2 + CV_16UC1 maps:
    weights ((32 - ax)(32 - ay), ax (32 - ay), (32 - ax) ay, ax ay) * 32, (sum + 2^14) >> 15, a tap outside the image 0."""
    img = np.asarray(img, dtype=np.uint8)
    H, W = img.shape
    sx = map1[..., 0].astype(np.int64)
    sy = map1[..., 1].astype(np.int64)
    f = map2.astype(np.int64) & (INTER_TAB_SIZE * INTER_TAB_SIZE - 1)
    ax, ay = f & (INTER_TAB_SIZE - 1), f >> INTER_BITS
    acc = np.zeros(sx.shape, dtype=np.int64)
    for dy, dx, w in ((0, 0, (32 - ax) * (32 - ay)), (0, 1, ax * (32 - ay)), (1, 0, (32 - ax) * ay), (1, 1, ax * ay)):
        x, y = sx + dx, sy + dy
        inside = (x >= 0) & (x < W) & (y >= 0) & (y < H)
        tap = np.where(inside, img[np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)].astype(np.int64), 0)
        acc += tap * (w * 32)
    return ((acc + (1 << 14)) >> 15).astype(np.uint8)
