"""Evaluate depth and surface-normal predictions against ground truth on the device (csrc/metrics.cu).

    from omnidata_b200.metrics import DepthMetrics, NormalMetrics
    metric = DepthMetrics(space="depth", min_depth=1e-3, max_depth=None)
    for pred, gt, mask in batches:          # fp32 [B,H,W] or [B,1,H,W]; mask optional, uint8 / bool / fp32
        metric.update(pred, gt, mask)
    print(metric.compute())                 # {"abs_rel": ..., "delta1": ..., "images": ..., ...}

- DepthMetrics: per image, the prediction is aligned to the ground truth in scale and shift by least squares (in depth
  or, as the MiDaS zero-shot protocol does, in disparity), then AbsRel, SqRel, RMSE, RMSE_log and delta_1..3 are taken
  over the image's valid pixels; the dataset value of each is the mean over the images with at least one valid pixel.
- NormalMetrics: the angle between predicted and true normals, pooled over every valid pixel of the dataset: mean,
  median (to 2^-13 degree, from a dataset-wide histogram), RMSE and the percentages within 11.25, 22.5 and 30 degrees
  (the published OASIS surface-normal metrics, without the relative-normal AUC).
- BoundaryMetrics: the depth-boundary errors (DBE) of iBims-1: edges are detected in the prediction (and, unless given,
  in the ground truth) with a masked Canny detector; accuracy is the mean distance in pixels from predicted edges to
  true ones (those within max_dist), completeness the mean distance from true edges to predicted ones.  Csrc:
  boundary.cu.
- MeshMetrics: reconstructed meshes against ground-truth meshes, both sampled alike: accuracy (mean distance from the
  prediction to the truth), completion (the reverse), Chamfer-L1, and precision, recall and F-score at distance
  thresholds, optionally culled to what the cameras saw.  Csrc: mesh_metrics.cu.  Unlike the others its `update`
  synchronises (sample counts, bounding boxes).

Definitions: DESIGN.md §3 "Evaluation metrics" and include/omnidata_b200.h; oracle/metrics_oracle.py restates them in
float64.  The state lives in fixed device tensors.  `update` neither synchronises the host nor allocates after its first
call at a shape, so it can be captured in a CUDA graph; only `compute` synchronises.  The state after a dataset does not
depend on how the dataset was split into batches, and repeat runs give the same bits.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from . import _capi, ops
from .losses import _StepBuffers

DEPTH_KEYS = ("abs_rel", "sq_rel", "rmse", "rmse_log", "delta1", "delta2", "delta3")
DEPTH_COUNTS = ("images", "excluded", "degenerate", "pixels")
NORMAL_COUNTS = ("pixels", "nonfinite", "n_11.25", "n_22.5", "n_30")
BOUNDARY_COUNTS = ("images", "no_gt_edges", "no_pred_edges", "pred_edge_pixels", "gt_edge_pixels")


class _Metrics(_StepBuffers):
    _STATE: Dict[str, tuple] = {}

    def __init__(self):
        self._bufs = {}
        self._state: Optional[Dict[str, torch.Tensor]] = None

    def _state_on(self, device: torch.device) -> Dict[str, torch.Tensor]:
        if self._state is None:
            self._state = {k: torch.zeros(shape, dtype=dt, device=device) for k, (shape, dt) in self._STATE.items()}
        elif next(iter(self._state.values())).device != device:
            raise ValueError(f"{type(self).__name__}: the state lives on {next(iter(self._state.values())).device}, "
                             f"the inputs on {device}")
        return self._state

    def _host_state(self) -> Dict[str, torch.Tensor]:
        if self._state is None:
            return {k: torch.zeros(shape, dtype=dt) for k, (shape, dt) in self._STATE.items()}
        return {k: t.cpu() for k, t in self._state.items()}

    def reset(self):
        """Back to an empty dataset (the state tensors are zeroed in place: a captured update stays valid)."""
        if self._state is not None:
            for t in self._state.values():
                t.zero_()

    def all_reduce(self, group=None):
        """Replaces every rank's state by the fold of all ranks' states in rank order (torch.distributed all-gather of
        the fixed-size state).  Counts and the histogram are exact; the sums are deterministic for a given world size
        and sharding."""
        import torch.distributed as dist
        if self._state is None:
            dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else \
                torch.device("cpu")
            self._state_on(dev)
        world = dist.get_world_size(group)
        for t in self._state.values():
            parts = [torch.empty_like(t) for _ in range(world)]
            dist.all_gather(parts, t, group=group)
            acc = parts[0].clone()
            for p in parts[1:]:
                acc += p
            t.copy_(acc)


class DepthMetrics(_Metrics):
    """Scale/shift-aligned depth metrics (module docstring).  space "depth" fits s p + t to the depth, "disparity" to its
    inverse and needs max_depth; valid pixels have mask != 0 and a finite depth in (min_depth, max_depth].
    align=False (depth space only) scores a metric prediction, such as a SparseDepthAligner's output, as it is:
    d-hat = clamp(p, min_depth, max_depth)."""

    _STATE = {"sums": ((7,), torch.float64), "counts": ((4,), torch.int64)}

    def __init__(self, space: str = "depth", min_depth: float = 1e-3, max_depth: Optional[float] = None,
                 align: bool = True):
        super().__init__()
        if space not in ("depth", "disparity"):
            raise ValueError(f"space must be 'depth' or 'disparity', got {space!r}")
        if not align and space != "depth":
            raise ValueError("align=False scores metric depth as predicted and takes space='depth' only")
        if space == "disparity" and max_depth is None:
            raise ValueError("space='disparity' needs max_depth (the predicted disparity is clamped to 1 / max_depth)")
        min_depth = float(min_depth)
        max_depth = math.inf if max_depth is None else float(max_depth)
        if not (math.isfinite(min_depth) and min_depth >= 0.0) or not (max_depth > min_depth):
            raise ValueError(f"need 0 <= min_depth < max_depth, got min_depth={min_depth}, max_depth={max_depth}")
        self.space = space
        self.align = bool(align)
        self.min_depth, self.max_depth = min_depth, max_depth

    @_capi.on_tensor_device
    @torch.no_grad()
    def update(self, pred: torch.Tensor, gt: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Adds a batch: pred, gt fp32 [B,H,W] or [B,1,H,W]; mask None or uint8 / bool / fp32, nonzero = valid.
        Returns the batch's per-image records fp64 [B, 12] (include/omnidata_b200.h odb_depth_metrics_update), valid
        until the next update at this shape."""
        b, h, w, _, _ = ops.check_metric_inputs("DepthMetrics.update", pred, gt, mask, 1)
        st = self._state_on(pred.device)
        ws = self._buf("workspace", (ops.metrics_workspace_bytes(b, h, w) // 8,), torch.float64, pred.device)
        rec = self._buf("records", (b, _capi.DEPTH_RECORD), torch.float64, pred.device)
        space = _capi.SPACE_DISPARITY if self.space == "disparity" else _capi.SPACE_DEPTH
        ops.depth_metrics_update(pred, gt, mask, space, self.min_depth, self.max_depth, ws, rec, st["sums"],
                                 st["counts"], align=self.align)
        return rec

    def compute(self) -> dict:
        """Dataset values: the mean over images with valid pixels of each per-image metric (NaN before any such image),
        and the counts: images (with valid pixels), excluded (none valid), degenerate (det <= 0, aligned to 0),
        pixels (valid pixels)."""
        st = self._host_state()
        counts = [int(c) for c in st["counts"].tolist()]
        n = counts[0]
        out = {k: (s / n if n else math.nan) for k, s in zip(DEPTH_KEYS, st["sums"].tolist())}
        out.update(zip(DEPTH_COUNTS, counts))
        return out


class NormalMetrics(_Metrics):
    """Angular-error metrics of surface normals, pooled over all valid pixels (module docstring)."""

    _STATE = {"sums": ((2,), torch.float64), "counts": ((5,), torch.int64),
              "hist": ((_capi.NORMAL_HIST_BINS,), torch.int64)}

    @_capi.on_tensor_device
    @torch.no_grad()
    def update(self, pred: torch.Tensor, gt: torch.Tensor, mask: Optional[torch.Tensor] = None) -> None:
        """Adds a batch: pred, gt fp32 [B,3,H,W] in the model's output encoding [0, 1]; mask None or [B,(1,)H,W]
        uint8 / bool / fp32, nonzero = valid."""
        b, h, w, _, _ = ops.check_metric_inputs("NormalMetrics.update", pred, gt, mask, 3)
        st = self._state_on(pred.device)
        ws = self._buf("workspace", (ops.metrics_workspace_bytes(b, h, w) // 8,), torch.float64, pred.device)
        ops.normal_metrics_update(pred, gt, mask, ws, st["sums"], st["counts"], st["hist"])

    def compute(self) -> dict:
        """mean, median, rmse (degrees), pct_11.25 / pct_22.5 / pct_30 (percent of pixels), median_bin (the histogram
        bin of the lower median, -1 if none), and the counts: pixels (finite angles), nonfinite (excluded),
        n_11.25 / n_22.5 / n_30."""
        med = (-1.0, math.nan)
        if self._state is not None:
            buf = self._buf("median", (2,), torch.float64, self._state["hist"].device)
            ops.normal_metrics_median(self._state["hist"], buf)
            med = tuple(buf.tolist())
        st = self._host_state()
        counts = [int(c) for c in st["counts"].tolist()]
        n = counts[0]
        s, s2 = st["sums"].tolist()
        out = {"mean": s / n if n else math.nan, "median": med[1], "rmse": math.sqrt(s2 / n) if n else math.nan}
        for k, c in zip(("pct_11.25", "pct_22.5", "pct_30"), counts[2:]):
            out[k] = 100.0 * c / n if n else math.nan
        out["median_bin"] = int(med[0])
        out.update(zip(NORMAL_COUNTS, counts))
        return out


class BoundaryMetrics(_Metrics):
    """Depth-boundary errors (module docstring; DESIGN.md §3 "Depth-boundary metrics").  sigma, low and high configure
    the edge detector (Gaussian width in pixels, hysteresis thresholds on the Sobel magnitude of the depth normalised
    to [0, 1] over the valid pixels); predicted edges at max_dist pixels or more from every true edge are left out of
    the accuracy.  Valid pixels as in DepthMetrics: mask != 0 and a finite depth in (min_depth, max_depth]."""

    _STATE = {"sums": ((2,), torch.float64), "counts": ((5,), torch.int64)}

    def __init__(self, sigma: float = math.sqrt(2.0), low: float = 0.1, high: float = 0.2, max_dist: float = 10.0,
                 min_depth: float = 1e-3, max_depth: Optional[float] = None):
        super().__init__()
        sigma, low, high, max_dist = float(sigma), float(low), float(high), float(max_dist)
        min_depth = float(min_depth)
        max_depth = math.inf if max_depth is None else float(max_depth)
        if not (0.0 < sigma <= 4.0):
            raise ValueError(f"sigma must lie in (0, 4], got {sigma}")
        if not (math.isfinite(low) and math.isfinite(high) and 0.0 <= low <= high):
            raise ValueError(f"need finite 0 <= low <= high, got low={low}, high={high}")
        if not (math.isfinite(max_dist) and max_dist > 0.0):
            raise ValueError(f"max_dist must be finite and > 0, got {max_dist}")
        if not (math.isfinite(min_depth) and min_depth >= 0.0) or not (max_depth > min_depth):
            raise ValueError(f"need 0 <= min_depth < max_depth, got min_depth={min_depth}, max_depth={max_depth}")
        self.sigma, self.low, self.high, self.max_dist = sigma, low, high, max_dist
        self.min_depth, self.max_depth = min_depth, max_depth

    def _workspace(self, b, h, w, device):
        return self._buf("workspace", (-(-ops.boundary_workspace_bytes(b, h, w) // 8),), torch.float64, device)

    @_capi.on_tensor_device
    @torch.no_grad()
    def update(self, pred: torch.Tensor, gt: torch.Tensor, mask: Optional[torch.Tensor] = None,
               gt_edges: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Adds a batch: pred, gt fp32 [B,H,W] or [B,1,H,W]; mask None or uint8 / bool / fp32, nonzero = valid;
        gt_edges None (detected in gt) or uint8 / bool [B,(1,)H,W], nonzero = edge.  Returns the batch's per-image
        records fp64 [B, 8] (include/omnidata_b200.h odb_boundary_metrics_update), valid until the next update at this
        shape."""
        b, h, w, _, _ = ops.check_metric_inputs("BoundaryMetrics.update", pred, gt, mask, 1)
        if gt_edges is not None:
            ops._edge_map("BoundaryMetrics.update", gt_edges, b, h, w, "gt_edges")
        st = self._state_on(pred.device)
        ws = self._workspace(b, h, w, pred.device)
        rec = self._buf("records", (b, _capi.BOUNDARY_RECORD), torch.float64, pred.device)
        ops.boundary_metrics_update(pred, gt, mask, gt_edges, self.sigma, self.low, self.high, self.max_dist,
                                    self.min_depth, self.max_depth, ws, rec, st["sums"], st["counts"])
        return rec

    @_capi.on_tensor_device
    @torch.no_grad()
    def edges(self, depth: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The detector's edge map uint8 [B,H,W] (1 = edge) of depth fp32 [B,(1,)H,W], valid pixels taken from depth
        itself and the mask, for visualisation and tests.  A new tensor."""
        b, h, w, _, _ = ops.check_metric_inputs("BoundaryMetrics.edges", depth, depth, mask, 1)
        out = torch.empty(b, h, w, dtype=torch.uint8, device=depth.device)
        ops.depth_edges(depth, mask, self.sigma, self.low, self.high, self.min_depth, self.max_depth,
                        self._workspace(b, h, w, depth.device), out)
        return out

    def compute(self) -> dict:
        """dbe_acc, dbe_comp: the means over the images with ground-truth edges of the per-image accuracy and
        completeness in pixels (NaN before any such image), and the counts: images (all), no_gt_edges (excluded),
        no_pred_edges (no predicted edge within max_dist: both errors max_dist), pred_edge_pixels, gt_edge_pixels."""
        st = self._host_state()
        counts = [int(c) for c in st["counts"].tolist()]
        n = counts[0] - counts[1]
        acc, comp = st["sums"].tolist()
        out = {"dbe_acc": acc / n if n else math.nan, "dbe_comp": comp / n if n else math.nan}
        out.update(zip(BOUNDARY_COUNTS, counts))
        return out


MESH_COUNTS = ("scenes", "no_gt", "empty_pred", "pred_points", "gt_points", "pred_culled", "gt_culled")


class MeshMetrics(_Metrics):
    """Accuracy, completion, Chamfer-L1, precision, recall and F-score of reconstructed meshes against ground-truth
    meshes (DESIGN.md §3 "Mesh metrics"; csrc/mesh_metrics.cu).  Both meshes are sampled alike (`mesh.sample_surface`
    at density points per m^2, streams 0 and 1 of seed), so vertex density does not bias the result; thresholds (1 to
    4, metres) are the distances at which a point counts as matched (5 cm is the usual indoor value; density 1e4,
    about 1 cm spacing, is not tuned)."""

    _STATE = {"sums": ((3 + 3 * _capi.MESH_MAX_THRESHOLDS,), torch.float64), "counts": ((7,), torch.int64)}

    def __init__(self, thresholds=(0.05,), density: float = 1e4, seed: int = 0):
        super().__init__()
        try:
            self.thresholds = tuple(float(t) for t in ops.check_thresholds("MeshMetrics", thresholds))
        except _capi.OdbError as e:
            raise ValueError(str(e)) from None
        density = float(density)
        if not (math.isfinite(density) and density > 0):
            raise ValueError(f"MeshMetrics: density must be finite and > 0, got {density}")
        if not (isinstance(seed, int) and 0 <= seed < 2 ** 63):
            raise ValueError(f"MeshMetrics: seed must be an integer in [0, 2^63), got {seed!r}")
        self.density, self.seed = density, seed

    @_capi.on_tensor_device
    @torch.no_grad()
    def update(self, pred_vertices: torch.Tensor, pred_faces: torch.Tensor, gt_vertices: torch.Tensor,
               gt_faces: torch.Tensor, views=None, return_distances: bool = False):
        """Adds one scene: the predicted and the true mesh (vertices fp32 [V,3], faces int32 [F,3], on one device).
        views = (intrinsics, (h, w), poses [n,4,4] camera-to-world, host or device) culls both sample sets to what
        those cameras see (`mesh.frustum_mask`, max_depth 10 m, occlusion not modelled).  Returns the scene's record
        fp64 [1, MESH_RECORD] (include/omnidata_b200.h odb_mesh_metrics_update); with return_distances also a dict of
        the culled samples and their distances to the other mesh: pred_points fp32 [P,3], pred_distance fp64 [P],
        gt_points, gt_distance.  Synchronises: to read the sample counts, the kept counts and the bounding boxes."""
        from . import mesh
        dev = pred_vertices.device
        st = self._state_on(dev)
        P = mesh.sample_surface(pred_vertices, pred_faces, self.density, self.seed, 0)
        G = mesh.sample_surface(gt_vertices, gt_faces, self.density, self.seed, 1)
        culled = [0, 0]
        if views is not None:
            intrinsics, size, poses = views
            T = mesh.device_poses("MeshMetrics.update", poses, dev)
            kept = []
            for q, X in enumerate((P, G)):
                m = torch.empty(X.shape[0], dtype=torch.uint8, device=dev)
                mesh._value_error(ops.frustum_mask, X, intrinsics, size, T, 10.0, m)
                Y = mesh.compact(X, m)
                culled[q] = X.shape[0] - Y.shape[0]
                kept.append(Y)
            P, G = kept
        dp, _ = mesh.nearest(P, G)
        dg, _ = mesh.nearest(G, P)
        ws = self._buf("workspace", (max(1, ops.mesh_metrics_workspace_bytes(P.shape[0], G.shape[0]) // 8),),
                       torch.float64, dev)
        rec = torch.empty(_capi.MESH_RECORD, dtype=torch.float64, device=dev)
        ops.mesh_metrics_update(dp, dg, self.thresholds, culled[0], culled[1], ws, rec, st["sums"], st["counts"])
        rec = rec.unsqueeze(0)
        if return_distances:
            return rec, {"pred_points": P, "pred_distance": dp, "gt_points": G, "gt_distance": dg}
        return rec

    def compute(self) -> dict:
        """The means over scenes of accuracy, completion and chamfer (metres; over the scenes with both samples),
        and of precision@t, recall@t and fscore@t per threshold t (over the scenes with ground-truth samples; an
        empty prediction scores 0); NaN before any such scene.  Counts: scenes, no_gt (no ground-truth samples:
        excluded), empty_pred (no predicted samples), pred_points, gt_points (kept samples), pred_culled, gt_culled."""
        st = self._host_state()
        counts = [int(c) for c in st["counts"].tolist()]
        sums = st["sums"].tolist()
        n_prf = counts[0] - counts[1]
        n_dist = n_prf - counts[2]
        out = {k: (s / n_dist if n_dist else math.nan) for k, s in zip(("accuracy", "completion", "chamfer"), sums)}
        for q, t in enumerate(self.thresholds):
            for j, k in enumerate(("precision", "recall", "fscore")):
                out[f"{k}@{t:g}"] = sums[3 + 3 * q + j] / n_prf if n_prf else math.nan
        out.update(zip(MESH_COUNTS, counts))
        return out
