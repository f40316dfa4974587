"""Evaluation metrics restated in float64 torch (omnidata_b200/csrc/metrics.cu, DESIGN.md §3 "Evaluation metrics").
Runs on any device.  Each definition names the kernel it mirrors; the per-pixel expressions are written operation by
operation as the kernels round them."""
from __future__ import annotations

import math
from typing import List, Optional

import torch

HIST_PER_DEGREE = 4096                         # ODB_NORMAL_HIST_PER_DEGREE
HIST_BINS = 180 * HIST_PER_DEGREE + 1


def _planes(t: torch.Tensor) -> torch.Tensor:
    return t.reshape(t.shape[0], -1).double()


def depth_valid(g: torch.Tensor, mask: Optional[torch.Tensor], min_depth: float, max_depth: float) -> torch.Tensor:
    """metrics.cu depth_valid: mask != 0, g finite, g > min_depth, g <= max_depth (inf: none)."""
    v = torch.isfinite(g) & (g > min_depth) & (g <= max_depth)
    return v if mask is None else v & (mask != 0)


def scale_shift(p: torch.Tensor, y: torch.Tensor):
    """metrics.cu depth_scale_shift: compute_scale_and_shift (L/midas_loss.py:10-30) on the five moments of the valid
    pixels; (0, 0) where det <= 0.  Returns (s, t, det)."""
    a00, a01, a11 = (p * p).sum(), p.sum(), float(p.numel())
    b0, b1 = (p * y).sum(), y.sum()
    det = a00 * a11 - a01 * a01
    if not bool(det > 0):
        return torch.zeros((), dtype=torch.float64), torch.zeros((), dtype=torch.float64), det
    return (a11 * b0 - a01 * b1) / det, (-a01 * b0 + a00 * b1) / det, det


def depth_image(pred: torch.Tensor, gt: torch.Tensor, mask: Optional[torch.Tensor] = None, space: str = "depth",
                min_depth: float = 1e-3, max_depth: float = math.inf) -> dict:
    """One image's record (metrics.cu depth_error_kernel / depth_fold_kernel): n, abs_rel, sq_rel, rmse, rmse_log,
    c1..c3 (delta counts), s, t, degenerate, nonfinite."""
    p, g = pred.reshape(-1).double(), gt.reshape(-1).double()
    m = None if mask is None else mask.reshape(-1)
    v = depth_valid(g, m, min_depth, max_depth)
    p, g = p[v], g[v]
    n = int(p.numel())
    y = 1.0 / g if space == "disparity" else g
    nonfinite = int((~torch.isfinite(p)).sum())
    s, t, det = scale_shift(p, y)
    rec = {"n": n, "s": float(s), "t": float(t), "degenerate": n > 0 and bool(det <= 0), "nonfinite": nonfinite}
    a = s * p + t
    if space == "disparity":
        d = 1.0 / torch.clamp(a, min=1.0 / max_depth)
    else:
        d = a
    d = torch.clamp(d, min=min_depth, max=max_depth)
    e = d - g
    e2 = e * e
    lg = torch.log(d) - torch.log(g)
    r = torch.maximum(d / g, g / d)
    c = [int((r < 1.25 ** k).sum()) for k in (1, 2, 3)]
    bad = math.nan if nonfinite else 0.0
    if n == 0:
        rec.update(abs_rel=math.nan, sq_rel=math.nan, rmse=math.nan, rmse_log=math.nan, c1=0, c2=0, c3=0)
        return rec
    rec.update(abs_rel=float((e.abs() / g).sum()) / n + bad, sq_rel=float((e2 / g).sum()) / n + bad,
               rmse=math.sqrt(float(e2.sum()) / n) + bad, rmse_log=math.sqrt(float((lg * lg).sum()) / n) + bad)
    for k in range(3):
        rec[f"c{k + 1}"] = c[k] + bad
    return rec


def depth_dataset(records: List[dict]) -> dict:
    """metrics.cu depth_fold_kernel + DepthMetrics.compute: image-order fold of the records of images with n > 0."""
    keys = ("abs_rel", "sq_rel", "rmse", "rmse_log", "delta1", "delta2", "delta3")
    sums = [0.0] * 7
    images = excluded = degenerate = pixels = 0
    for r in records:
        if r["n"] == 0:
            excluded += 1
            continue
        vals = [r["abs_rel"], r["sq_rel"], r["rmse"], r["rmse_log"]] + [r[f"c{k}"] / r["n"] for k in (1, 2, 3)]
        sums = [a + b for a, b in zip(sums, vals)]
        images += 1
        degenerate += int(r["degenerate"])
        pixels += r["n"]
    out = {k: (s / images if images else math.nan) for k, s in zip(keys, sums)}
    out.update(images=images, excluded=excluded, degenerate=degenerate, pixels=pixels)
    return out


def normal_angles(pred: torch.Tensor, gt: torch.Tensor, mask: Optional[torch.Tensor] = None):
    """metrics.cu normal_angle_kernel on one or more images [.., 3, H, W]: (finite angles in degrees of the pixels that
    take part, number of non-finite angles).  a = 2 p - 1, b = 2 g - 1, theta = atan2(|a x b|, a . b)."""
    p = pred.double().reshape(-1, 3, pred.shape[-2] * pred.shape[-1])
    q = gt.double().reshape(-1, 3, gt.shape[-2] * gt.shape[-1])
    a0, a1, a2 = (2.0 * p[:, k] - 1.0 for k in range(3))
    b0, b1, b2 = (2.0 * q[:, k] - 1.0 for k in range(3))
    na = torch.sqrt(a0 * a0 + a1 * a1 + a2 * a2)
    nb = torch.sqrt(b0 * b0 + b1 * b1 + b2 * b2)
    take = ~(na <= 1e-6) & ~(nb <= 1e-6)
    if mask is not None:
        take &= mask.reshape(take.shape) != 0
    x = a1 * b2 - a2 * b1
    y = a2 * b0 - a0 * b2
    z = a0 * b1 - a1 * b0
    cr = torch.sqrt(x * x + y * y + z * z)
    dot = a0 * b0 + a1 * b1 + a2 * b2
    th = torch.atan2(cr, dot) * (180.0 / 3.141592653589793)
    th = th[take]
    fin = torch.isfinite(th)
    return th[fin], int((~fin).sum())


def normal_dataset(angles: List[torch.Tensor], nonfinite: int = 0) -> dict:
    """Pooled statistics of the angles (NormalMetrics.compute): mean, rmse, pct_*, the counts, and the lower-median bin
    of the 1/4096-degree histogram with its centre."""
    th = torch.cat([a.reshape(-1).double().cpu() for a in angles]) if angles else torch.zeros(0, dtype=torch.float64)
    n = int(th.numel())
    out = {"pixels": n, "nonfinite": nonfinite}
    cnt = [int((th < lim).sum()) for lim in (11.25, 22.5, 30.0)]
    out.update({"n_11.25": cnt[0], "n_22.5": cnt[1], "n_30": cnt[2]})
    if n == 0:
        out.update(mean=math.nan, rmse=math.nan, median=math.nan, median_bin=-1,
                   **{"pct_11.25": math.nan, "pct_22.5": math.nan, "pct_30": math.nan})
        return out
    out.update(mean=float(th.sum()) / n, rmse=math.sqrt(float((th * th).sum()) / n))
    for k, c in zip(("pct_11.25", "pct_22.5", "pct_30"), cnt):
        out[k] = 100.0 * c / n
    bins = torch.clamp((th * HIST_PER_DEGREE).floor().long(), max=HIST_BINS - 1)
    k = int(bins.sort().values[(n - 1) // 2])
    out.update(median_bin=k, median=(k + 0.5) / HIST_PER_DEGREE)
    return out


def histogram(angles: torch.Tensor) -> torch.Tensor:
    """The int64 histogram odb_normal_metrics_update fills: floor(4096 theta) per finite angle."""
    bins = torch.clamp((angles.double() * HIST_PER_DEGREE).floor().long(), max=HIST_BINS - 1)
    return torch.bincount(bins.cpu(), minlength=HIST_BINS)
