"""Sparse metric alignment restated in numpy float64 (omnidata_b200/csrc/sparse.cu, DESIGN.md §3 "Sparse metric
alignment").  The interpolation coordinates, the weights, the IRLS residual and the apply are written operation by
operation as the kernels round them; the normal equations are assembled densely and solved with numpy.linalg.solve
(the kernels sum per-region moments and solve the band by Cholesky, so the nodes agree to rounding, not to the bit)."""
from __future__ import annotations

import math
from typing import Optional

import numpy as np

STATUS_OK, STATUS_NO_POINTS, STATUS_DEGENERATE, STATUS_NONFINITE = 0, 1, 2, 3


def node_lerp(L: int, g: int):
    """Per position x < L: (i0, i1, f) with u = ((x + 0.5) g) / L - 0.5 clamped to [0, g - 1], i0 = floor(u),
    i1 = min(i0 + 1, g - 1), f = u - i0."""
    x = np.arange(L, dtype=np.float64)
    u = np.minimum(np.maximum(((x + 0.5) * g) / L - 0.5, 0.0), float(g - 1))
    i0 = np.floor(u)
    return i0.astype(np.int64), np.minimum(i0.astype(np.int64) + 1, g - 1), u - i0


def fields(nodes: np.ndarray, h: int, w: int):
    """S, T [h, w] float64 from nodes [gy, gx, 2]: (1 - fy) ((1 - fx) n00 + fx n01) + fy ((1 - fx) n10 + fx n11)."""
    gy, gx = nodes.shape[:2]
    y0, y1, fy = node_lerp(h, gy)
    x0, x1, fx = node_lerp(w, gx)
    ey, ex = (1.0 - fy)[:, None], (1.0 - fx)[None, :]
    fy, fx = fy[:, None], fx[None, :]
    out = []
    for c in range(2):
        n = nodes[..., c]
        top = ex * n[y0][:, x0] + fx * n[y0][:, x1]
        bot = ex * n[y1][:, x0] + fx * n[y1][:, x1]
        out.append(ey * top + fy * bot)
    return out


def points(sparse: np.ndarray, mask: Optional[np.ndarray], min_depth: float, max_depth: float) -> np.ndarray:
    """V: mask != 0, sparse finite, min_depth < sparse <= max_depth (metrics_oracle.depth_valid)."""
    g = sparse.astype(np.float64)
    with np.errstate(invalid="ignore"):
        v = np.isfinite(g) & (g > min_depth) & (g <= max_depth)
    return v if mask is None else v & (np.asarray(mask) != 0)


def normal_equations(a, y, wts, ys, xs, h, w, gy, gx, smooth):
    """Dense A, rhs of E = S w (S a + T - y)^2 + (smooth / n_e) S_{i~j} S_V ((s_i - s_j) a + (t_i - t_j))^2 over the
    points (a, y, weights w at rows ys, columns xs), unknowns (s_0, t_0, s_1, t_1, ...) in row-major node order."""
    K = gy * gx
    n = 2 * K
    y0, y1, fy = node_lerp(h, gy)
    x0, x1, fx = node_lerp(w, gx)
    ny = (y0[ys], y1[ys])
    nx = (x0[xs], x1[xs])
    py = (1.0 - fy[ys], fy[ys])
    px = (1.0 - fx[xs], fx[xs])
    node = [ny[c >> 1] * gx + nx[c & 1] for c in range(4)]
    phi = [py[c >> 1] * px[c & 1] for c in range(4)]
    A = np.zeros(n * n)
    rhs = np.zeros(n)
    for c in range(4):
        wc = wts * phi[c]
        rhs += np.bincount(2 * node[c], wc * a * y, minlength=n)
        rhs += np.bincount(2 * node[c] + 1, wc * y, minlength=n)
        for d in range(4):
            v = wc * phi[d]
            r, q = 2 * node[c], 2 * node[d]
            A += np.bincount(r * n + q, v * a * a, minlength=n * n)
            A += np.bincount(r * n + q + 1, v * a, minlength=n * n)
            A += np.bincount((r + 1) * n + q, v * a, minlength=n * n)
            A += np.bincount((r + 1) * n + q + 1, v, minlength=n * n)
    A = A.reshape(n, n)
    edges = [(k, k + 1) for k in range(K) if k % gx < gx - 1] + [(k, k + gx) for k in range(K - gx)]
    if edges:
        lam = smooth / len(edges)
        G = lam * np.array([[np.sum(a * a), np.sum(a)], [np.sum(a), float(a.size)]])
        for i, j in edges:
            for p, q, sgn in ((i, i, 1), (j, j, 1), (i, j, -1), (j, i, -1)):
                A[2 * p:2 * p + 2, 2 * q:2 * q + 2] += sgn * G
    return A, rhs


def fit(pred: np.ndarray, sparse: np.ndarray, mask: Optional[np.ndarray] = None, grid=(1, 1), space: str = "depth",
        smooth: float = 0.1, robust: Optional[float] = None, iterations: Optional[int] = None,
        min_depth: float = 1e-3, max_depth: float = math.inf):
    """One image [H, W]: (nodes float64 [gy, gx, 2], record [8]) as odb_sparse_align_fit defines them."""
    a_all = np.asarray(pred, dtype=np.float32).astype(np.float64)
    h, w = a_all.shape
    gy, gx = grid
    v = points(sparse, mask, min_depth, max_depth)
    ys, xs = np.nonzero(v)
    a = a_all[ys, xs]
    g = np.asarray(sparse, dtype=np.float32).astype(np.float64)[ys, xs]
    y = 1.0 / g if space == "disparity" else g
    n = a.size
    rec = np.zeros(8)
    rec[0] = n
    nan_nodes = np.full((gy, gx, 2), np.nan)
    if n < 2:
        rec[1:3] = STATUS_NO_POINTS, np.nan
        return nan_nodes, rec
    if not np.isfinite(a).all():
        rec[1:3] = STATUS_NONFINITE, np.nan
        return nan_nodes, rec
    iters = 1 if robust is None else (5 if iterations is None else iterations)
    wts = np.ones(n)
    nodes = None
    down = 0.0
    for it in range(iters):
        if it > 0:
            r = _residual(nodes, h, w, ys, xs, a, y)
            with np.errstate(divide="ignore"):
                wts = np.minimum(1.0, robust / np.abs(r))
            down = float(np.sum(wts < 1.0)) / n
        det = np.sum(wts * a * a) * np.sum(wts) - np.sum(wts * a) ** 2
        if not det > 0:
            rec[1:3] = STATUS_DEGENERATE, np.nan
            rec[3] = down
            return nan_nodes, rec
        A, rhs = normal_equations(a, y, wts, ys, xs, h, w, gy, gx, smooth)
        nodes = np.linalg.solve(A, rhs).reshape(gy, gx, 2)
    r = _residual(nodes, h, w, ys, xs, a, y)
    rec[2] = math.sqrt(float(np.sum(r * r)) / n)
    rec[3] = down
    return nodes, rec


def _residual(nodes, h, w, ys, xs, a, y):
    """r = (S a + T - y) / y at the points."""
    S, T = fields(nodes, h, w)
    return (S[ys, xs] * a + T[ys, xs] - y) / y


def apply(pred: np.ndarray, nodes: np.ndarray, space: str = "depth", min_depth: float = 1e-3,
          max_depth: float = math.inf) -> np.ndarray:
    """odb_sparse_align_apply on one image: float64 [H, W] before the one rounding to fp32 (NaN where pred is not
    finite or the nodes are NaN)."""
    a = np.asarray(pred, dtype=np.float32).astype(np.float64)
    S, T = fields(nodes, *a.shape)
    z = S * a + T
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        d = 1.0 / np.maximum(z, 1.0 / max_depth) if space == "disparity" else z.copy()
        d = np.minimum(np.maximum(d, min_depth), max_depth)
    d[~np.isfinite(a) | np.isnan(S) | np.isnan(T)] = np.nan
    return d


def depth_image_metric(pred, gt, mask=None, min_depth: float = 1e-3, max_depth: float = math.inf) -> dict:
    """odb_depth_metrics_update_metric on one image (metrics_oracle.depth_image without the fit): dh = clamp(p,
    min_depth, max_depth); the record's n, abs_rel, sq_rel, rmse, rmse_log, c1..c3, nonfinite."""
    p = np.asarray(pred, dtype=np.float32).astype(np.float64).reshape(-1)
    g = np.asarray(gt, dtype=np.float32).astype(np.float64).reshape(-1)
    v = points(g, None if mask is None else np.asarray(mask).reshape(-1), min_depth, max_depth)
    p, g = p[v], g[v]
    n = p.size
    nonfinite = int(np.sum(~np.isfinite(p)))
    rec = {"n": n, "nonfinite": nonfinite}
    if n == 0:
        rec.update(abs_rel=math.nan, sq_rel=math.nan, rmse=math.nan, rmse_log=math.nan, c1=0, c2=0, c3=0)
        return rec
    with np.errstate(invalid="ignore"):
        d = np.minimum(np.maximum(p, min_depth), max_depth)
        e = d - g
        lg = np.log(d) - np.log(g)
        r = np.maximum(d / g, g / d)
    bad = math.nan if nonfinite else 0.0
    rec.update(abs_rel=float(np.sum(np.abs(e) / g)) / n + bad, sq_rel=float(np.sum(e * e / g)) / n + bad,
               rmse=math.sqrt(float(np.sum(e * e)) / n) + bad, rmse_log=math.sqrt(float(np.sum(lg * lg)) / n) + bad)
    for k in range(3):
        rec[f"c{k + 1}"] = int(np.sum(r < 1.25 ** (k + 1))) + bad
    return rec
