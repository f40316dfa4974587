"""Metric depth from sparse measurements: the project's depth predictions are affine-invariant (an unknown scale and
shift), and a few measured depths of the same frame (LiDAR returns projected into the camera, SfM / SLAM points, a
depth sensor with holes) fix them.  On the device (csrc/sparse.cu).

    from omnidata_b200.sparse import SparseDepthAligner
    align = SparseDepthAligner(space="depth", grid=(1, 1), smooth=0.1, robust=None, iterations=None,
                               min_depth=1e-3, max_depth=None)
    metres = align(pred, sparse, mask)      # pred, sparse fp32 [B,H,W] or [B,1,H,W]; sparse in metres, 0 = none

`pred` is the output of any predictor (`model(x)`, `TiledPredictor`, `EnsemblePredictor`, `GuidedPredictor`) at the
sparse map's resolution.  Points are the pixels with mask != 0 and a finite sparse depth in (min_depth, max_depth].
The fit maps pred to S pred + T, where S and T are the bilinear resize of a gy x gx grid of (s, t) nodes: grid (1, 1)
is one least-squares scale and shift per image, finer grids let the map vary across the image (near against far,
centre against edge) with neighbouring nodes tied together by `smooth`.  In "disparity" space the map is fitted to
1 / depth (max_depth is then required).  `robust=delta` reweights the points by Huber IRLS on the relative residual,
so that LiDAR returns that leak across occlusion boundaries do not pull the fit; `iterations` solves (default 5).  The
default smooth = 0.1 is not tuned: there is no dataset here to tune it on.

Images with fewer than two points, with all predictions equal on the points, or with a non-finite prediction on a point
come out NaN everywhere, and their record says why.  Definition: DESIGN.md §3 "Sparse metric alignment" and
include/omnidata_b200.h; oracle/sparse_oracle.py restates it in float64.  Deterministic and independent of the batch;
after the first call at a shape, a call neither synchronises nor allocates beyond its output, so it can be captured in a
CUDA graph.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from . import _capi, ops
from .losses import _StepBuffers

MAX_NODES = _capi.SPARSE_MAX_NODES
STATUS = ("ok", "no_points", "degenerate", "nonfinite")     # record column 1


class SparseDepthAligner(_StepBuffers):
    """Fits scale and shift fields of a depth prediction to sparse metric depths and applies them (module docstring)."""

    def __init__(self, space: str = "depth", grid: Tuple[int, int] = (1, 1), smooth: float = 0.1,
                 robust: Optional[float] = None, iterations: Optional[int] = None, min_depth: float = 1e-3,
                 max_depth: Optional[float] = None):
        if space not in ("depth", "disparity"):
            raise ValueError(f"space must be 'depth' or 'disparity', got {space!r}")
        if space == "disparity" and max_depth is None:
            raise ValueError("space='disparity' needs max_depth (the fitted disparity is clamped to 1 / max_depth)")
        try:
            gy, gx = (int(v) for v in grid)
        except (TypeError, ValueError):
            raise ValueError(f"grid must be (gy, gx), got {grid!r}") from None
        if tuple(grid) != (gy, gx) or gy < 1 or gx < 1 or gy * gx > MAX_NODES:
            raise ValueError(f"grid must be (gy, gx) with gy, gx >= 1 and at most {MAX_NODES} nodes, got {grid!r}")
        smooth = float(smooth)
        if not math.isfinite(smooth) or smooth < 0 or (gy * gx > 1 and smooth <= 0):
            raise ValueError(f"smooth must be finite and > 0 with more than one node, got {smooth}")
        if robust is None:
            if iterations is not None:
                raise ValueError("iterations applies to robust fits only (robust=None runs one solve)")
            robust_v, iters = 0.0, 1
        else:
            robust_v = float(robust)
            if not (math.isfinite(robust_v) and robust_v > 0):
                raise ValueError(f"robust (the Huber threshold on the relative residual) must be finite and > 0, got "
                                 f"{robust}")
            iters = 5 if iterations is None else iterations
            if isinstance(iters, bool) or int(iters) != iters or not 2 <= iters <= 32:
                raise ValueError(f"iterations must be an integer in [2, 32], got {iterations}")
        min_depth = float(min_depth)
        max_depth = math.inf if max_depth is None else float(max_depth)
        if not (math.isfinite(min_depth) and min_depth >= 0.0) or not (max_depth > min_depth):
            raise ValueError(f"need 0 <= min_depth < max_depth, got min_depth={min_depth}, max_depth={max_depth}")
        if space == "disparity" and not math.isfinite(max_depth):
            raise ValueError("space='disparity' needs a finite max_depth")
        self.space, self.grid, self.smooth = space, (gy, gx), smooth
        self.robust = None if robust is None else robust_v
        self.iterations = int(iters)
        self.min_depth, self.max_depth = min_depth, max_depth
        self._robust = robust_v
        self._space = _capi.SPACE_DISPARITY if space == "disparity" else _capi.SPACE_DEPTH
        self._bufs = {}

    def _check_grid(self, name: str, h: int, w: int):
        gy, gx = self.grid
        if gy > h or gx > w:
            raise ValueError(f"{name}: grid {gy}x{gx} needs images of at least {gy}x{gx} pixels, got {h}x{w}")

    @_capi.on_tensor_device
    @torch.no_grad()
    def fit(self, pred: torch.Tensor, sparse: torch.Tensor,
            mask: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(nodes fp64 [B, gy, gx, 2], records fp64 [B, 8]) for pred, sparse fp32 [B,H,W] or [B,1,H,W] and mask None or
        uint8 / bool / fp32 (nonzero = valid).  A record is (n, status, RMS relative residual, fraction of points
        down-weighted in the last solve, 0, 0, 0, 0); status indexes STATUS.  Both are kept for the next call at this
        shape, which overwrites them."""
        b, h, w, _, _ = ops.check_metric_inputs("SparseDepthAligner.fit", pred, sparse, mask, 1)
        self._check_grid("SparseDepthAligner.fit", h, w)
        dev = pred.device
        ws = self._buf("workspace", (-(-ops.sparse_align_workspace_bytes(b, h, w, self.grid) // 8),), torch.float64,
                       dev)
        nodes = self._buf("nodes", (b, *self.grid, 2), torch.float64, dev)
        rec = self._buf("records", (b, _capi.SPARSE_RECORD), torch.float64, dev)
        ops.sparse_align_fit(pred, sparse, mask, self.grid, self._space, self.min_depth, self.max_depth, self.smooth,
                             self._robust, self.iterations, ws, nodes, rec)
        return nodes, rec

    @_capi.on_tensor_device
    @torch.no_grad()
    def apply(self, pred: torch.Tensor, nodes: torch.Tensor) -> torch.Tensor:
        """Metric depth fp32 [B,H,W] of pred fp32 [B,H,W] or [B,1,H,W] under nodes fp64 [B, gy, gx, 2] (from `fit`):
        clamped to [min_depth, max_depth], NaN where pred is not finite.  A new tensor."""
        b, h, w = ops.metrics_plane_shape(pred, 1)
        self._check_grid("SparseDepthAligner.apply", h, w)
        if tuple(nodes.shape) != (b, *self.grid, 2):
            raise ValueError(f"SparseDepthAligner.apply: nodes must be [{b}, {self.grid[0]}, {self.grid[1]}, 2], got "
                             f"{tuple(nodes.shape)}")
        out = torch.empty(b, h, w, dtype=torch.float32, device=pred.device)
        ops.sparse_align_apply(pred, nodes, out, self._space, self.min_depth, self.max_depth)
        return out

    def __call__(self, pred: torch.Tensor, sparse: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Metric depth fp32 [B,H,W]: `apply(pred, fit(pred, sparse, mask)[0])`."""
        nodes, _ = self.fit(pred, sparse, mask)
        return self.apply(pred, nodes)
