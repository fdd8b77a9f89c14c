"""NumPy restatement of StereoFrame::plotStereoFrame (src/stereoFrame.cpp:618-663) on 8-bit images: the rectified left
image in BGR, then cv::circle of every stereo point and cv::line of every stereo line in (B, G, R) = (0, 200, 0).

- The base image is img_l after rectification in the channels the caller gave: cvtColor(GRAY2BGR) replicates a grey value,
  cvtColor(BGRA2BGR) drops alpha, three channels are taken as they are (convertTo(CV_8UC3) is a no-op on 8-bit data).
- circle(img, Point(int(x), int(y)), 3, colour, 1): thickness is int(1.5) = 1 and the line type LINE_8, so OpenCV draws its
  integer radius-3 circle (CIRCLE_3 below, as cv2 draws it on an empty canvas) and clips it pixel by pixel at the border.
- line(img, Point(int(sx), int(sy)), Point(int(ex), int(ey)), colour, 1): LINE_8, thickness 1 is cv::LineIterator from the
  start to the end point after cv::clipLine.  clipLine moves the first end point before the second and computes the
  second's move from the moved first, so which end comes first changes the pixels of a segment that leaves the image.
- int() truncates toward zero.  Every draw writes the same value, so the order of the draws does not change the image.

No OpenCV here: tests/test_plot_host.py holds these functions to cv2 where it is importable, and the GPU tests use them.
"""
from __future__ import annotations

import numpy as np

from oracle import color as C

COLOUR = (0, 200, 0)   # Scalar(0, 200, 0): B, G, R

# (dx, dy) of every pixel cv::circle sets for radius 3, thickness 1, LINE_8
CIRCLE_3 = ((-3, 0), (-2, -2), (-2, -1), (-2, 1), (-2, 2), (-1, -2), (-1, 2), (0, -3), (0, 3), (1, -2), (1, 2), (2, -2),
            (2, -1), (2, 1), (2, 2), (3, 0))


def trunc(v: float) -> int:
    """C++'s int(double): toward zero"""
    return int(np.trunc(v))


def circle_pixels(cx: int, cy: int, width: int, height: int) -> list:
    """the (x, y) pixels cv::circle(img, Point(cx, cy), 3, c, 1, LINE_8) sets on a width x height image"""
    return [(cx + dx, cy + dy) for dx, dy in CIRCLE_3 if 0 <= cx + dx < width and 0 <= cy + dy < height]


def _to_int(v: float) -> int:
    """(int64)(double): toward zero"""
    return int(v)


def clip_line(width: int, height: int, x1: int, y1: int, x2: int, y2: int):
    """cv::clipLine(Size2l, Point2l&, Point2l&): (inside, x1, y1, x2, y2), the end points moved onto the image in this order"""
    if width <= 0 or height <= 0:
        return False, x1, y1, x2, y2
    right, bottom = width - 1, height - 1
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += _to_int(float(a - y1) * (x2 - x1) / (y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += _to_int(float(a - y2) * (x2 - x1) / (y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += _to_int(float(a - x1) * (y2 - y1) / (x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += _to_int(float(a - x2) * (y2 - y1) / (x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, x1, y1, x2, y2


def line_pixels(x1: int, y1: int, x2: int, y2: int, width: int, height: int) -> list:
    """the (x, y) pixels cv::line(img, Point(x1, y1), Point(x2, y2), c, 1, LINE_8) sets on a width x height image:
    cv::LineIterator(img, pt1, pt2, 8, leftToRight = true), which clips first"""
    if not (0 <= x1 < width and 0 <= y1 < height and 0 <= x2 < width and 0 <= y2 < height):
        inside, x1, y1, x2, y2 = clip_line(width, height, x1, y1, x2, y2)
        if not inside:
            return []
    if x2 < x1:   # leftToRight: the ends swap where the line runs right to left
        x1, y1, x2, y2 = x2, y2, x1, y1
    dx, dy = x2 - x1, y2 - y1
    sx, sy = 1, 1
    if dy < 0:
        dy, sy = -dy, -1
    vert = dy > dx
    if vert:
        dx, dy = dy, dx
    err, plus, minus = dx - 2 * dy, 2 * dx, -2 * dy
    x, y = x1, y1
    out = []
    for _ in range(dx + 1):
        out.append((x, y))
        step_minor = err < 0
        err += minus + (plus if step_minor else 0)
        if vert:   # major axis y, minor x
            y += sy
            x += sx if step_minor else 0
        else:
            x += sx
            y += sy if step_minor else 0
    return out


def gray2bgr(img: np.ndarray) -> np.ndarray:
    """cv::cvtColor(COLOR_GRAY2BGR) of uint8[H, W]"""
    img = np.asarray(img, dtype=np.uint8)
    return np.repeat(img[..., None], 3, axis=-1)


def bgra2bgr(img: np.ndarray) -> np.ndarray:
    """cv::cvtColor(COLOR_BGRA2BGR) of uint8[H, W, 4]"""
    return np.ascontiguousarray(np.asarray(img, dtype=np.uint8)[..., :3])


def base_image(frame: np.ndarray, maps=None) -> np.ndarray:
    """plotStereoFrame's img_l_aux of a left image as the caller gave it (uint8[H, W] grey, uint8[H, W, 3] BGR or
    uint8[H, W, 4] BGRA): rectified with maps = (map1, map2) (None: as given), then in BGR"""
    frame = np.asarray(frame, dtype=np.uint8)
    if frame.ndim == 3:
        frame = frame[..., :3]   # remapping each channel and then dropping alpha is BGRA2BGR(remap(img))
    if maps is not None:
        frame = C.remap(frame, maps[0], maps[1]) if frame.ndim == 3 else C.R.remap(frame, maps[0], maps[1])
    return gray2bgr(frame) if frame.ndim == 2 else np.ascontiguousarray(frame)


def plot_stereo_frame(base: np.ndarray, pt_pl, ls_spl, ls_epl) -> np.ndarray:
    """plotStereoFrame on base (uint8[H, W, 3], not modified): circles at pt_pl [n][2], lines ls_spl [m][2] -> ls_epl [m][2]"""
    img = np.array(base, dtype=np.uint8, copy=True)
    H, W = img.shape[:2]
    xs, ys = [], []
    for x, y in np.asarray(pt_pl, dtype=np.float64).reshape(-1, 2):
        for px, py in circle_pixels(trunc(x), trunc(y), W, H):
            xs.append(px)
            ys.append(py)
    spl = np.asarray(ls_spl, dtype=np.float64).reshape(-1, 2)
    epl = np.asarray(ls_epl, dtype=np.float64).reshape(-1, 2)
    for s, e in zip(spl, epl):
        for px, py in line_pixels(trunc(s[0]), trunc(s[1]), trunc(e[0]), trunc(e[1]), W, H):
            xs.append(px)
            ys.append(py)
    if xs:
        img[np.asarray(ys), np.asarray(xs)] = COLOUR
    return img
