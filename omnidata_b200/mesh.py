"""Compare point sets and triangle meshes on the device (csrc/mesh_metrics.cu): surface sampling, exact nearest
neighbours and frustum culling, the parts of `metrics.MeshMetrics`.

    from omnidata_b200 import mesh
    pts = mesh.sample_surface(vertices, faces, density=1e4, seed=0, stream=0)   # fp32 [N,3], about 1 cm apart
    dist, idx = mesh.nearest(query, reference)          # fp64 [M], int32 [M]: exact, ties to the smaller index
    keep = mesh.frustum_mask(pts, (fx, fy, cx, cy), (h, w), poses)   # uint8 [N]: 1 where some camera sees the point
    seen = mesh.compact(pts, keep)                      # the kept points, in order

Definitions in DESIGN.md §3 "Mesh metrics" and include/omnidata_b200.h; oracle/mesh_oracle.py restates them in
float64.  Every result is bit-reproducible.  `sample_surface` synchronises once to read the sample count, `nearest`
once to read the reference set's bounding box, and `compact` once to read the kept count.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import numpy as np
import torch

from . import _capi, ops

# Points per m^2 of the evaluation's surface samples: about 1 cm apart.  Not tuned.
DEFAULT_DENSITY = 1e4
# The default grid of `nearest` has at most this many cells per reference point (and at most NN_MAX_CELLS).  It sets
# the speed only, never a result; 8 was not tuned beyond a check on the analytic room.
CELLS_PER_POINT = 8


def _value_error(fn, *args, **kw):
    try:
        return fn(*args, **kw)
    except _capi.OdbError as e:
        raise ValueError(str(e)) from None


def _f64_workspace(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(1, -(-nbytes // 8)), dtype=torch.float64, device=device)


@_capi.on_tensor_device
@torch.no_grad()
def sample_surface(vertices: torch.Tensor, faces: torch.Tensor, density: float = DEFAULT_DENSITY, seed: int = 0,
                   stream: int = 0) -> torch.Tensor:
    """Random points on the mesh (vertices fp32 [V,3], faces int32 [F,3] on the device), density points per m^2 in
    expectation: face t gets floor(A_t density + xi_t) points, uniform on the triangle, ordered by (face, k).  seed and
    stream select the counter-based generator's sequence (MeshMetrics uses stream 0 for the prediction, 1 for the
    ground truth).  Returns fp32 [N,3].  ValueError for a face index outside [0, V), a non-finite vertex used by a face
    or more than MESH_MAX_POINTS samples, before any sample is written.  Synchronises once."""
    name = "sample_surface"
    _, nf = _value_error(ops.check_mesh, name, vertices, faces)
    density = float(density)
    if not (math.isfinite(density) and density > 0):
        raise ValueError(f"{name}: density must be finite and > 0, got {density}")
    dev = vertices.device
    ws = _f64_workspace(ops.mesh_sample_workspace_bytes(nf), dev)
    info = torch.empty(2, dtype=torch.int64, device=dev)
    _value_error(ops.mesh_sample_count, vertices, faces, density, seed, stream, ws, info)
    total, flags = info.tolist()
    if flags & 1:
        raise ValueError(f"{name}: a face index lies outside [0, {vertices.shape[0]})")
    if flags & 2:
        raise ValueError(f"{name}: a face uses a non-finite vertex")
    if total > _capi.MESH_MAX_POINTS:
        raise ValueError(f"{name}: {total} samples exceed the limit of {_capi.MESH_MAX_POINTS} per call; lower the "
                         "density")
    out = torch.empty(total, 3, dtype=torch.float32, device=dev)
    ops.mesh_sample_emit(vertices, faces, seed, stream, ws, out)
    return out


def default_cell(lo, hi, n_ref: int) -> float:
    """The grid cell size `nearest` uses by default: the smallest h (by bisection) for which the box [lo, hi] has at
    most min(CELLS_PER_POINT n_ref, NN_MAX_CELLS) cells of h per side; 1 for a box of one point."""
    lo, hi = [float(v) for v in lo], [float(v) for v in hi]
    ext = max(h - l for l, h in zip(lo, hi))
    if ext == 0.0:
        return 1.0
    target = max(1, min(CELLS_PER_POINT * n_ref, _capi.NN_MAX_CELLS))
    grid = lambda h: ops.nn_grid_cells(lo + hi + [h])          # noqa: E731
    a, b = ext / target, 2.0 * ext                              # grid(a) > target >= grid(b) = 1
    for _ in range(64):
        m = 0.5 * (a + b)
        if m <= a or m >= b:
            break
        if grid(m) <= target:
            b = m
        else:
            a = m
    return b


def _key_to_float(keys: np.ndarray) -> np.ndarray:
    k = keys.astype(np.int32)
    return np.where(k >= 0, k, k ^ np.int32(0x7FFFFFFF)).astype(np.int32).view(np.float32).astype(np.float64)


@_capi.on_tensor_device
@torch.no_grad()
def nearest(query: torch.Tensor, reference: torch.Tensor, cell: Optional[float] = None
            ) -> Tuple[torch.Tensor, torch.Tensor]:
    """For each query point (fp32 [M,3]) its nearest reference point (fp32 [N,3]): (distance fp64 [M], index int32
    [M]), exact: d^2 = (dx^2 + dy^2) + dz^2 in fp64 round-to-nearest, ties to the smallest index; (+inf, -1) for an
    empty reference.  cell: the grid's cell size in metres (default: default_cell); it changes the time, never a
    result.  ValueError for non-finite coordinates.  Synchronises once to read the reference's bounding box."""
    name = "nearest"
    nq = _value_error(ops.check_points, name, query, "query")
    nr = _value_error(ops.check_points, name, reference, "reference")
    dev = ops._same_device(query, reference)
    box = torch.empty(7, dtype=torch.int32, device=dev)
    ops.nn_bounds(reference, query, box)
    b = box.cpu().numpy()
    if b[6] & 1:
        raise ValueError(f"{name}: the reference has a non-finite coordinate")
    if b[6] & 2:
        raise ValueError(f"{name}: the query has a non-finite coordinate")
    dist = torch.empty(nq, dtype=torch.float64, device=dev)
    index = torch.empty(nq, dtype=torch.int32, device=dev)
    if nr == 0:
        ops.nn_query(query, 0, None, None, dist, index)
        return dist, index
    lo, hi = _key_to_float(b[:3]), _key_to_float(b[3:6])
    h = default_cell(lo, hi, nr) if cell is None else float(cell)
    if not (math.isfinite(h) and h > 0):
        raise ValueError(f"{name}: cell must be finite and > 0, got {cell}")
    grid = np.concatenate([lo, hi, [h]])
    if ops.nn_grid_cells(grid) > _capi.NN_MAX_CELLS:
        raise ValueError(f"{name}: cell {h} gives {ops.nn_grid_cells(grid)} cells, at most {_capi.NN_MAX_CELLS}")
    ws = _f64_workspace(ops.nn_workspace_bytes(nr, grid), dev)
    ops.nn_build(reference, grid, ws)
    ops.nn_query(query, nr, grid, ws, dist, index)
    return dist, index


def device_poses(name: str, poses, device) -> torch.Tensor:
    """Camera-to-world poses, host or device [n,4,4] / [4,4], checked by ops.check_poses, as a device fp64 [n,16]."""
    if isinstance(poses, torch.Tensor):
        poses = poses.detach().cpu()
    T = _value_error(ops.check_poses, name, poses)
    return torch.from_numpy(T).to(device)


@_capi.on_tensor_device
@torch.no_grad()
def frustum_mask(points: torch.Tensor, intrinsics, size: Tuple[int, int], poses, max_depth: float = 10.0
                 ) -> torch.Tensor:
    """uint8 [N]: 1 where at least one camera sees the point (fp32 [N,3]): in its frame 0 < z <= max_depth and the
    nearest pixel lies in the h x w image (TSDFVolume.integrate's projection).  poses: host or device [n,4,4]
    camera-to-world; they go to the device once, so thousands of frames cost no kernel-parameter space.  Occlusion is
    not modelled: a point behind a wall in a camera's frustum counts as seen."""
    name = "frustum_mask"
    n = _value_error(ops.check_points, name, points)
    T = device_poses(name, poses, points.device)
    mask = torch.empty(n, dtype=torch.uint8, device=points.device)
    _value_error(ops.frustum_mask, points, intrinsics, size, T, float(max_depth), mask)
    return mask


@_capi.on_tensor_device
@torch.no_grad()
def compact(points: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """The points (fp32 [N,3]) where mask (uint8 [N]) is nonzero, in order: an integer scan, so deterministic.
    Synchronises once."""
    n = _value_error(ops.check_points, "compact", points)
    dev = points.device
    ws = _f64_workspace(ops.compact_workspace_bytes(n), dev)
    out = torch.empty(n, 3, dtype=torch.float32, device=dev)
    count = torch.empty(1, dtype=torch.int64, device=dev)
    _value_error(ops.compact_points, points, mask, ws, out, count)
    return out[:int(count.item())]
