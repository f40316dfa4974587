"""Depth-normal fusion: one consistent geometry from the project's two networks.  The depth prediction is
affine-invariant (its shift is unknown and bends every back-projected surface), and the depth and normal predictions of
the same frame disagree.  `DepthNormalFusion` solves for the depth whose back-projection agrees with the predicted
normals while staying close to the predicted depth, and recovers the shift from the normals.  `depth_normals` gives the
normals a depth map implies, so the two networks' disagreement can be measured (`NormalMetrics`).  On the device
(csrc/fusion.cu).

    from omnidata_b200.fusion import DepthNormalFusion, depth_normals
    fuse = DepthNormalFusion(weight=0.1, shift=True, jump=0.02, iterations=1000, tol=1e-8, axes=(1, -1, -1))
    fused, records = fuse.fit(depth, normals, (fx, fy, cx, cy), mask=None)
    n = depth_normals(fused, (fx, fy, cx, cy))          # fp32 [B,3,H,W] in the normal model's encoding

depth fp32 [B,H,W] or [B,1,H,W] is z-depth (the clamped relative prediction, or metres from `SparseDepthAligner`);
normals fp32 [B,3,H,W] are the normal model's output in [0, 1] at the same resolution; the intrinsics are in pixels of
that resolution.  Each 4-neighbour edge whose ends have similar normals and no depth step (|a_q - a_p| <= jump times
the image's depth range) asks the 3-D step between its ends to be orthogonal to their mean normal (Nehab et al.,
SIGGRAPH 2005, in perspective form, linear in depth); `weight` ties z to the prediction plus a shift t.  The solve is
Jacobi-preconditioned conjugate gradients in fp64.  `axes` maps the model's encoding to the camera frame (x right, y
down, z forward): the default reads it as x right, y up, z towards the camera, our belief about the Omnidata
convention that has not been checked against a trained checkpoint (DESIGN.md §3 "Depth-normal fusion" says how to
check it).  The defaults weight = 0.1 and jump = 0.02 are not tuned.

Definition: DESIGN.md §3 and include/omnidata_b200.h; oracle/fusion_oracle.py restates it in float64.  Deterministic
and independent of the batch; after the first call at a shape, a call neither synchronises nor allocates beyond its
output, so it can be captured in a CUDA graph.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence, Tuple

import torch

from . import _capi, ops
from .losses import _StepBuffers

STATUS = ("converged", "empty", "flat", "not_converged")     # record column 1
DEFAULT_AXES = (1, -1, -1)


def _check_axes(axes) -> Tuple[int, int, int]:
    try:
        t = tuple(axes)
    except TypeError:
        raise ValueError(f"axes must be three signs +-1, got {axes!r}") from None
    if len(t) != 3 or any(isinstance(v, bool) or v not in (1, -1) for v in t):
        raise ValueError(f"axes must be three signs +-1, got {axes!r}")
    return tuple(int(v) for v in t)


def _check_jump(jump) -> float:
    jump = float(jump)
    if not (math.isfinite(jump) and jump > 0):
        raise ValueError(f"jump must be finite and > 0, got {jump}")
    return jump


def _intrinsics(name: str, intrinsics) -> Tuple[float, float, float, float]:
    try:
        return ops.check_intrinsics(name, intrinsics)
    except _capi.OdbError as e:
        raise ValueError(str(e)) from None


class DepthNormalFusion(_StepBuffers):
    """Fuses a depth prediction with the normal prediction of the same frame (module docstring)."""

    def __init__(self, weight: float = 0.1, shift: bool = True, jump: float = 0.02, iterations: int = 1000,
                 tol: float = 1e-8, axes: Sequence[int] = DEFAULT_AXES):
        weight, tol = float(weight), float(tol)
        if not (math.isfinite(weight) and weight > 0):
            raise ValueError(f"weight must be finite and > 0, got {weight}")
        if not isinstance(shift, bool):
            raise ValueError(f"shift must be a bool, got {shift!r}")
        if isinstance(iterations, bool) or int(iterations) != iterations or not 1 <= iterations <= 10000:
            raise ValueError(f"iterations must be an integer in [1, 10000], got {iterations}")
        if not (math.isfinite(tol) and 0 < tol < 1):
            raise ValueError(f"tol must lie in (0, 1), got {tol}")
        self.weight, self.shift, self.jump = weight, shift, _check_jump(jump)
        self.iterations, self.tol, self.axes = int(iterations), tol, _check_axes(axes)
        self._bufs = {}

    @_capi.on_tensor_device
    @torch.no_grad()
    def fit(self, depth: torch.Tensor, normals: torch.Tensor, intrinsics,
            mask: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(fused fp32 [B,H,W], records fp64 [B, 8]).  fused is NaN off V = {mask != 0, depth finite} and for status 1
        and 2.  A record is (|V|, status, kept edges, iterations run, final |r| / |b|, t, RMS over V of fused - depth -
        t, 0); status indexes STATUS.  The records are kept for the next call at this shape, which overwrites them."""
        name = "DepthNormalFusion.fit"
        k = _intrinsics(name, intrinsics)
        b, h, w = ops.metrics_plane_shape(depth, 1, "depth")
        if tuple(normals.shape) != (b, 3, h, w):
            raise ValueError(f"{name}: normals must be [{b}, 3, {h}, {w}] for depth {tuple(depth.shape)}, got "
                             f"{tuple(normals.shape)}")
        if mask is not None and tuple(mask.shape) not in ((b, h, w), (b, 1, h, w)):
            raise ValueError(f"{name}: mask must be [B,H,W] or [B,1,H,W] for depth {tuple(depth.shape)}, got "
                             f"{tuple(mask.shape)}")
        dev = depth.device
        ws = self._buf("workspace", (-(-ops.fusion_workspace_bytes(b, h, w) // 8),), torch.float64, dev)
        rec = self._buf("records", (b, _capi.FUSION_RECORD), torch.float64, dev)
        out = torch.empty(b, h, w, dtype=torch.float32, device=dev)
        ops.depth_normal_fusion(depth, normals, mask, k, self.axes, self.jump, self.weight, self.shift,
                                self.iterations, self.tol, ws, out, rec)
        return out, rec

    def __call__(self, depth: torch.Tensor, normals: torch.Tensor, intrinsics,
                 mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The fused depth fp32 [B,H,W] alone."""
        return self.fit(depth, normals, intrinsics, mask)[0]


@_capi.on_tensor_device
@torch.no_grad()
def depth_normals(depth: torch.Tensor, intrinsics, axes: Sequence[int] = DEFAULT_AXES, jump: float = 0.02,
                  mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The normals fp32 [B,3,H,W] that depth fp32 [B,H,W] or [B,1,H,W] implies, in the normal model's encoding
    (axes n + 1) / 2 and facing the camera; NaN off V and where no kept edge gives a tangent."""
    name = "depth_normals"
    k = _intrinsics(name, intrinsics)
    axes, jump = _check_axes(axes), _check_jump(jump)
    b, h, w = ops.metrics_plane_shape(depth, 1, "depth")
    ws = torch.empty(-(-ops.depth_normals_workspace_bytes(b, h, w) // 8), dtype=torch.float64, device=depth.device)
    out = torch.empty(b, 3, h, w, dtype=torch.float32, device=depth.device)
    ops.depth_normals(depth, mask, k, axes, jump, ws, out)
    return out
