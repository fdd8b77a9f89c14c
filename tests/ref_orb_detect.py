"""NumPy restatement of cv::ORB's key-point selection (computeKeyPoints with an empty mask, OpenCV 4.13): FAST-9/16 with
non-max suppression, the level border filter, the per-level feature budget, retainBest as a set operation, and Harris
responses.  The pyramid, angles and descriptors come from the C description oracle (oracle/orb.py).  Key points come out per
image in canonical order: level ascending, then y, then x on the level.

TEST INFRASTRUCTURE: tests/ and tools/ import it; the product package never does."""
from __future__ import annotations

from concurrent.futures import ThreadPoolExecutor

import numpy as np

F32 = np.float32
HARRIS_SCORE, FAST_SCORE = 0, 1
# the FAST-16 circle of radius 3, contiguous (OpenCV's makeOffsets order)
DX = (0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1)
DY = (3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3)
HARRIS_K = F32(0.04)
_HS = F32(1.0) / F32(28 * 255.0)              # 1.f / ((1 << 2) * blockSize * 255.f), blockSize 7
HARRIS_SCALE4 = ((_HS * _HS) * _HS) * _HS


def float_scale(scale: float) -> float:
    """ORB::create takes the scale factor as a float."""
    return float(F32(scale))


def layer_scale(scale: float, level: int) -> np.float32:
    return F32(float_scale(scale) ** level)


def level_budgets(n_features: int, scale: float, n_levels: int):
    """nfeaturesPerLevel, in float as ORB computes it."""
    factor = F32(1.0 / float_scale(scale))
    with np.errstate(divide="ignore", invalid="ignore"):
        nd = F32(n_features) * (F32(1) - factor) / (F32(1) - F32(float(factor) ** n_levels))
    out, total = [], 0
    for _ in range(n_levels - 1):
        n = int(np.rint(nd))
        out.append(n)
        total += n
        nd = F32(nd * factor)
    out.append(max(n_features - total, 0))
    return out


def fast_scores(level: np.ndarray, threshold: int) -> np.ndarray:
    """int32 [h, w]: the FAST score of every corner (score >= threshold) in [3, w - 3) x [3, h - 3), 0 elsewhere."""
    th = min(max(int(threshold), 0), 255)
    h, w = level.shape
    S = np.zeros((h, w), np.int32)
    if w < 7 or h < 7:
        return S
    img = level.astype(np.int16)
    c = img[3:h - 3, 3:w - 3]
    d = np.stack([img[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx] - c for dx, dy in zip(DX, DY)])
    dd = np.concatenate([d, d[:8]])
    mn, mx = dd[0:16].copy(), dd[0:16].copy()
    for j in range(1, 9):                                  # arcs of 9 contiguous pixels
        np.minimum(mn, dd[j:j + 16], out=mn)
        np.maximum(mx, dd[j:j + 16], out=mx)
    sc = np.maximum(mn.max(0).astype(np.int32), -mx.min(0).astype(np.int32)) - 1
    S[3:h - 3, 3:w - 3] = np.where(sc >= th, sc, 0)
    return S


def fast_nms(level: np.ndarray, threshold: int):
    """FastFeatureDetector(threshold, nonmaxSuppression=true): (y, x, score) in raster order.  A corner survives iff its score
    is strictly greater than each of its 8 neighbours' (non-corners count 0)."""
    S = fast_scores(level, threshold)
    h, w = S.shape
    P = np.pad(S, 1)
    keep = S > 0
    for dy in range(3):
        for dx in range(3):
            if dy != 1 or dx != 1:
                keep &= S > P[dy:dy + h, dx:dx + w]
    ys, xs = np.nonzero(keep)
    return ys, xs, S[ys, xs]


def retain_best(resp: np.ndarray, n: int) -> np.ndarray:
    """KeyPointsFilter::retainBest as a set: boolean mask of the points kept (ties with the n-th largest all kept)."""
    if n == 0:
        return np.zeros(len(resp), bool)
    if len(resp) <= n:
        return np.ones(len(resp), bool)
    return resp >= np.sort(resp)[len(resp) - n]


def harris_responses(level: np.ndarray, xs: np.ndarray, ys: np.ndarray) -> np.ndarray:
    """ORB's HarrisResponses (block 7, k 0.04) at level coordinates: integer gradient sums, then float, unfused."""
    if len(xs) == 0:
        return np.zeros(0, F32)
    P = np.pad(level.astype(np.int32), 5, mode="reflect")   # BORDER_REFLECT_101 (ORB's pyramid border)
    Ix = (P[1:-1, 2:] - P[1:-1, :-2]) * 2 + (P[:-2, 2:] - P[:-2, :-2]) + (P[2:, 2:] - P[2:, :-2])
    Iy = (P[2:, 1:-1] - P[:-2, 1:-1]) * 2 + (P[2:, :-2] - P[:-2, :-2]) + (P[2:, 2:] - P[:-2, 2:])
    r = np.arange(-3, 4)
    ii = ys[:, None, None] + 4 + r[None, :, None]            # level (y, x) is Ix[y + 4, x + 4]
    jj = xs[:, None, None] + 4 + r[None, None, :]
    gx, gy = Ix[ii, jj].astype(np.int64), Iy[ii, jj].astype(np.int64)
    a, b, c = (gx * gx).sum((1, 2)), (gy * gy).sum((1, 2)), (gx * gy).sum((1, 2))
    fa, fb, fc = a.astype(F32), b.astype(F32), c.astype(F32)
    s = fa + fb
    return ((fa * fb - fc * fc) - (HARRIS_K * s) * s) * HARRIS_SCALE4


class OrbDetectRef:
    def __init__(self):
        from oracle.orb import OrbOracle
        self.orb = OrbOracle()

    def select(self, img, n_features=1200, n_levels=4, scale=1.2, score_type=FAST_SCORE, fast_threshold=20, edge=19):
        """computeKeyPoints: (level, y, x, response) arrays in canonical order."""
        pyr = self.orb.pyramid(img, n_levels, float_scale(scale))
        budget = level_budgets(n_features, scale, n_levels)
        out = []
        for lvl, (raw, _) in enumerate(pyr):
            h, w = raw.shape
            ys, xs, sc = fast_nms(raw, fast_threshold)
            m = (xs >= edge) & (xs < w - edge) & (ys >= edge) & (ys < h - edge)
            ys, xs, resp = ys[m], xs[m], sc[m].astype(F32)
            k = retain_best(resp, 2 * budget[lvl] if score_type == HARRIS_SCORE else budget[lvl])
            ys, xs, resp = ys[k], xs[k], resp[k]
            if score_type == HARRIS_SCORE:
                resp = harris_responses(raw, xs, ys)
                k = retain_best(resp, budget[lvl])
                ys, xs, resp = ys[k], xs[k], resp[k]
            out.append((np.full(len(xs), lvl, np.int32), ys.astype(np.int32), xs.astype(np.int32), resp.astype(F32)))
        return tuple(np.concatenate([o[i] for o in out]) for i in range(4))

    def detect(self, img, n_features=1200, n_levels=4, scale=1.2, score_type=FAST_SCORE, fast_threshold=20, edge=19,
               describe=True):
        """detectAndCompute on one image: dict(xy, octave, angle, response, desc) in canonical order."""
        lvl, ys, xs, resp = self.select(img, n_features, n_levels, scale, score_type, fast_threshold, edge)
        ls = np.array([layer_scale(scale, q) for q in range(n_levels)], F32)
        xy = np.stack([xs.astype(F32) * ls[lvl], ys.astype(F32) * ls[lvl]], 1).astype(F32).reshape(-1, 2)
        out = dict(xy=xy, octave=lvl, response=resp)
        if describe:
            n = len(xy)
            ang, desc, _, cnt = self.orb.compute_batch(img[None], [0, n], xy, lvl, None, n_levels=n_levels,
                                                       scale=float_scale(scale), edge=edge)
            assert cnt[0] == n     # detectAndCompute's own points all pass the image border filter
            out.update(angle=ang, desc=desc)
        return out

    def detect_batch(self, images, fast_th=None, threads=8, **cfg):
        """detect on each image (fast_th: per-image thresholds or None for cfg's), on host threads; concatenated, with
        off [n + 1]."""
        images = np.ascontiguousarray(images, np.uint8)
        th = [cfg.pop("fast_threshold", 20)] * len(images) if fast_th is None else [int(t) for t in fast_th]
        with ThreadPoolExecutor(max(1, threads)) as ex:
            res = list(ex.map(lambda a: self.detect(a[0], fast_threshold=a[1], **cfg), zip(images, th)))
        out = {k: np.concatenate([r[k] for r in res]) for k in ("xy", "octave", "angle", "response", "desc")}
        out["xy"] = out["xy"].reshape(-1, 2)
        out["desc"] = out["desc"].reshape(-1, 32)
        out["off"] = np.cumsum([0] + [len(r["xy"]) for r in res]).astype(np.int32)
        return out


def cv2_detect(cv2, img, n_features=1200, n_levels=4, scale=1.2, score_type=FAST_SCORE, fast_threshold=20, edge=19):
    """cv2's detectAndCompute sorted into canonical order (octave, y, x)."""
    o = cv2.ORB_create(n_features, scale, n_levels, edge, 0, 2, score_type, 31, fast_threshold)
    kps, d = o.detectAndCompute(img, None)
    xy = np.array([k.pt for k in kps], F32).reshape(-1, 2)
    oc = np.array([k.octave for k in kps], np.int32)
    order = np.lexsort((xy[:, 0], xy[:, 1], oc))
    return dict(xy=xy[order], octave=oc[order], angle=np.array([k.angle for k in kps], F32)[order],
                response=np.array([k.response for k in kps], F32)[order],
                desc=np.asarray(d if d is not None else np.zeros((0, 32)), np.uint8).reshape(-1, 32)[order])
