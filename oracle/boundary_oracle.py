"""Depth-boundary errors restated in float64 numpy (omnidata_b200/csrc/boundary.cu, DESIGN.md §3 "Depth-boundary
metrics").  Runs on the host.  The detector is written operation by operation in the kernels' order, so every value
matches bit for bit; hysteresis is scipy.ndimage.label with the 3x3 structure and the distances come from
scipy.ndimage.distance_transform_edt (squared exactly from its nearest-edge indices).  Square roots are numpy's
(correctly rounded; torch's CPU square root can land one ulp low)."""
from __future__ import annotations

import math
from typing import List

import numpy as np
from scipy import ndimage

NO_EDGE = -1                  # squared distance of every pixel of a map without edges (UINT64_MAX read as int64)


def _np(t, dtype=np.float64) -> np.ndarray:
    if t is None:
        return None
    if hasattr(t, "detach"):
        t = t.detach().cpu().numpy()
    return np.asarray(t).astype(dtype)


def gaussian_taps(sigma: float):
    """(R, taps k = -R .. R): exp(-k^2 / (2 sigma^2)) normalised to sum 1, summed in k order (boundary.cu
    edge_params; libm exp on both sides)."""
    r = int(math.floor(4.0 * sigma + 0.5))
    w = [math.exp(-float(k * k) / (2.0 * sigma * sigma)) for k in range(-r, r + 1)]
    s = 0.0
    for v in w:
        s += v
    return r, np.array([v / s for v in w], dtype=np.float64)


def valid_set(g, mask=None, min_depth: float = 1e-3, max_depth: float = math.inf) -> np.ndarray:
    """V = {mask != 0, g finite, min_depth < g <= max_depth} of one image [H,W]."""
    g = _np(g).reshape(_np(g).shape[-2:])
    with np.errstate(invalid="ignore"):
        v = np.isfinite(g) & (g > min_depth) & (g <= max_depth)
    if mask is not None:
        v &= _np(mask).reshape(g.shape) != 0
    return v


def weak_strong(f, valid: np.ndarray, sigma: float = math.sqrt(2.0), low: float = 0.1, high: float = 0.2):
    """Steps 1-4 of E(f, V) and the thresholds: (weak, strong) bool [H,W] (boundary.cu edge_stats_kernel ..
    sobel_nms_kernel)."""
    f = np.asarray(_np(f), dtype=np.float32).astype(np.float64).reshape(valid.shape)   # the kernels read fp32
    h, w = valid.shape
    none = np.zeros((h, w), dtype=bool)
    if not valid.any() or not np.isfinite(f[valid]).all():
        return none, none
    lo, hi = f[valid].min(), f[valid].max()
    if not hi > lo:
        return none, none
    fhat = np.zeros((h, w))
    fhat[valid] = (f[valid] - lo) / (hi - lo)
    one = valid.astype(np.float64)
    r, taps = gaussian_taps(sigma)

    def smooth(a, axis):
        n = a.shape[axis]
        pad = [(0, 0), (0, 0)]
        pad[axis] = (r, r)
        ap = np.pad(a, pad)
        acc = np.zeros_like(a)
        for k in range(2 * r + 1):
            sl = [slice(None), slice(None)]
            sl[axis] = slice(k, k + n)
            acc = acc + taps[k] * ap[tuple(sl)]
        return acc

    num = smooth(smooth(fhat, 1), 0)
    den = smooth(smooth(one, 1), 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(den > 0.0, num / den, 0.0)
    m = np.zeros((h, w))
    gx = np.zeros((h, w))
    gy = np.zeros((h, w))
    if h >= 3 and w >= 3:
        S = lambda dy, dx: s[1 + dy:h - 1 + dy, 1 + dx:w - 1 + dx]   # noqa: E731
        d0, d1, d2 = S(-1, 1) - S(-1, -1), S(0, 1) - S(0, -1), S(1, 1) - S(1, -1)
        e0, e1, e2 = S(1, -1) - S(-1, -1), S(1, 0) - S(-1, 0), S(1, 1) - S(-1, 1)
        gx[1:-1, 1:-1] = (d0 + 2.0 * d1) + d2
        gy[1:-1, 1:-1] = (e0 + 2.0 * e1) + e2
        m[1:-1, 1:-1] = np.sqrt(gx[1:-1, 1:-1] * gx[1:-1, 1:-1] + gy[1:-1, 1:-1] * gy[1:-1, 1:-1])
    cand = np.zeros((h, w), dtype=bool)
    if h >= 3 and w >= 3:
        vin = np.ones((h - 2, w - 2), dtype=bool)
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                vin &= valid[1 + dy:h - 1 + dy, 1 + dx:w - 1 + dx]
        cand[1:-1, 1:-1] = vin & (m[1:-1, 1:-1] > 0.0)
    ys, xs = np.nonzero(cand)
    gxc, gyc, mc = gx[ys, xs], gy[ys, xs], m[ys, xs]
    ax, ay = np.abs(gxc), np.abs(gyc)
    sx = np.where(gxc >= 0.0, 1, -1)
    sy = np.where(gyc >= 0.0, 1, -1)
    colwise = ax >= ay
    with np.errstate(invalid="ignore", divide="ignore"):
        wt = np.where(colwise, ay / ax, ax / ay)
    M = lambda dy, dx: m[ys + dy, xs + dx]                          # noqa: E731
    zero = np.zeros_like(sx)
    a1 = np.where(colwise, M(zero, sx), M(sy, zero))
    a2 = M(sy, sx)
    b1 = np.where(colwise, M(zero, -sx), M(-sy, zero))
    b2 = M(-sy, -sx)
    one_w = 1.0 - wt
    pa = a1 * one_w + a2 * wt
    pb = b1 * one_w + b2 * wt
    keep = (mc >= pa) & (mc >= pb)
    weak = np.zeros((h, w), dtype=bool)
    strong = np.zeros((h, w), dtype=bool)
    weak[ys, xs] = keep & (mc >= low)
    strong[ys, xs] = keep & (mc >= low) & (mc >= high)
    return weak, strong


def hysteresis(weak: np.ndarray, strong: np.ndarray) -> np.ndarray:
    """uint8: the weak pixels whose 8-connected weak component holds a strong pixel (a strong pixel counts as weak)."""
    weak = weak | strong
    lab, n = ndimage.label(weak, structure=np.ones((3, 3), dtype=int))
    good = np.zeros(n + 1, dtype=bool)
    good[np.unique(lab[strong])] = True
    good[0] = False
    return good[lab].astype(np.uint8)


def edges(f, valid: np.ndarray, sigma: float = math.sqrt(2.0), low: float = 0.1, high: float = 0.2) -> np.ndarray:
    """E(f, V) uint8 [H,W]."""
    return hysteresis(*weak_strong(f, valid, sigma, low, high))


def distance2(e) -> np.ndarray:
    """int64 [H,W]: the exact squared Euclidean distance to the nearest nonzero pixel; NO_EDGE everywhere without one."""
    e = _np(e, np.int64) != 0
    if not e.any():
        return np.full(e.shape, NO_EDGE, dtype=np.int64)
    idx = ndimage.distance_transform_edt(~e, return_distances=False, return_indices=True)
    yy, xx = np.indices(e.shape)
    dy, dx = idx[0] - yy, idx[1] - xx
    return dy.astype(np.int64) ** 2 + dx.astype(np.int64) ** 2


def _dist(d2: np.ndarray) -> np.ndarray:
    return np.where(d2 == NO_EDGE, np.inf, np.sqrt(np.maximum(d2, 0).astype(np.float64)))


def boundary_image(pred, gt, mask=None, gt_edges=None, sigma: float = math.sqrt(2.0), low: float = 0.1,
                   high: float = 0.2, max_dist: float = 10.0, min_depth: float = 1e-3,
                   max_depth: float = math.inf) -> dict:
    """One image's record (boundary.cu boundary_fold_kernel): acc, comp, n_pred, n_gt, n_a, nonfinite, no_gt, no_pred,
    and the edge maps eg, ep."""
    g = _np(gt)
    g = g.reshape(g.shape[-2:])
    v = valid_set(g, mask, min_depth, max_depth)
    p = _np(pred).reshape(g.shape)
    nonfinite = int((~np.isfinite(p[v])).sum())
    ep = edges(p, v, sigma, low, high)
    eg = (_np(gt_edges, np.int64).reshape(g.shape) != 0).astype(np.uint8) if gt_edges is not None else \
        edges(g, v, sigma, low, high)
    return dict(score(ep, eg, max_dist, nonfinite), eg=eg, ep=ep)


def score(ep, eg, max_dist: float = 10.0, nonfinite: int = 0) -> dict:
    """The errors of predicted edges ep against true edges eg ([H,W], nonzero = edge): acc, comp, n_pred, n_gt, n_a,
    nonfinite, no_gt, no_pred."""
    ep, eg = (_np(e, np.int64) != 0 for e in (ep, eg))
    dg, dp = _dist(distance2(eg)), _dist(distance2(ep))
    a = ep & (dg < max_dist)
    n_gt, n_pred, n_a = int(eg.sum()), int(ep.sum()), int(a.sum())
    bad = math.nan if nonfinite else 0.0
    no_gt, no_pred = n_gt == 0, n_gt > 0 and n_a == 0
    if no_gt:
        acc = comp = math.nan
    elif no_pred:
        acc = comp = max_dist + bad
    else:
        acc = float(dg[a].sum()) / n_a + bad
        comp = float(dp[eg].sum()) / n_gt + bad
    return {"acc": acc, "comp": comp, "n_pred": n_pred, "n_gt": n_gt, "n_a": n_a, "nonfinite": nonfinite,
            "no_gt": no_gt, "no_pred": no_pred}


def boundary_dataset(records: List[dict]) -> dict:
    """BoundaryMetrics.compute of the records folded in order."""
    sa = sc = 0.0
    n = 0
    for r in records:
        if not r["no_gt"]:
            sa += r["acc"]
            sc += r["comp"]
            n += 1
    return {"dbe_acc": sa / n if n else math.nan, "dbe_comp": sc / n if n else math.nan, "images": len(records),
            "no_gt_edges": sum(int(r["no_gt"]) for r in records),
            "no_pred_edges": sum(int(r["no_pred"]) for r in records),
            "pred_edge_pixels": sum(r["n_pred"] for r in records), "gt_edge_pixels": sum(r["n_gt"] for r in records)}


def record_row(r: dict) -> List[float]:
    """The record as odb_boundary_metrics_update writes it (ODB_BOUNDARY_RECORD doubles)."""
    return [r["acc"], r["comp"], float(r["n_pred"]), float(r["n_gt"]), float(r["n_a"]), float(r["nonfinite"]),
            float(r["no_gt"]), float(r["no_pred"])]


def batch_images(pred, gt, mask=None, gt_edges=None, **kw) -> List[dict]:
    """boundary_image of every image of a [B,(1,)H,W] batch."""
    b = pred.shape[0]
    pick = lambda t, i: None if t is None else t[i]                 # noqa: E731
    return [boundary_image(pred[i], gt[i], pick(mask, i), pick(gt_edges, i), **kw) for i in range(b)]


__all__ = ["gaussian_taps", "valid_set", "weak_strong", "hysteresis", "edges", "distance2", "boundary_image",
           "score", "boundary_dataset", "record_row", "batch_images", "NO_EDGE"]
