"""Fuse posed depth frames into one 3-D model: a dense truncated signed-distance (TSDF) volume on the device, with
integration of depth frames, raycasting of depth from the model and marching-tetrahedra mesh extraction
(csrc/volume.cu).

    from omnidata_b200.volume import TSDFVolume, write_ply
    vol = TSDFVolume(origin=(x0, y0, z0), voxel=0.02, dims=(nx, ny, nz), trunc=None, color=False)
    vol.integrate(depth, (fx, fy, cx, cy), cam_to_world, rgb=None)  # depth fp32 [B,H,W] metres; poses [B,4,4] host
    rendered = vol.raycast((fx, fy, cx, cy), cam_to_world, (h, w))    # fp32 [h,w] z-depth, 0 where nothing is hit
    depth, rgb = vol.raycast(K, cam_to_world, (h, w), color=True)     # color=True volumes: also fp32 [3,h,w], NaN: none
    vertices, faces, colors = vol.extract_mesh()                      # fp32 [V,3], int32 [F,3], fp32 [V,3] | None
    write_ply("mesh.ply", vertices, faces, colors)

Frames are OpenCV's (x right, y down, z forward, integer pixel centres); intrinsics are in pixels of the depth map; a
pose is the 4 x 4 camera-to-world matrix [R t; 0 0 0 1] (ScanNet's pose/*.txt).  The grid holds the points
X(i, j, k) = origin + voxel (i, j, k); each stores the TSDF F in [-1, 1] and the number of observations W (and, with
color=True, the mean RGB).  Depth is 0 or NaN where nothing was measured, so `SparseDepthAligner` output integrates as it
is.  A depth prediction in metres has a per-frame scale and shift error; fitting it with `SparseDepthAligner(grid=(1,
1))` to the volume's raycast at the frame's pose aligns it to what is already fused (reconstruct.py does this).

The default truncation, 3 voxels, is not tuned.  Definitions: DESIGN.md §3 "TSDF volumes" and include/omnidata_b200.h;
oracle/volume_oracle.py restates them in float64.  Every result is bit-reproducible, and integrating frames in one call
or several gives the same bits.  `integrate` and `raycast` neither synchronise nor allocate beyond their output (the
poses go to the kernels by value), so they can be captured in a CUDA graph; `extract_mesh` synchronises once to size
its outputs.
"""
from __future__ import annotations

import math
from pathlib import Path
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _capi, ops
from .losses import _StepBuffers

MAX_DIM = _capi.TSDF_MAX_DIM
MAX_POINTS = _capi.TSDF_MAX_POINTS


def _value_error(fn, *args):
    try:
        return fn(*args)
    except _capi.OdbError as e:
        raise ValueError(str(e)) from None


class TSDFVolume(_StepBuffers):
    """A dense TSDF grid of dims = (nx, ny, nz) points from origin with spacing voxel (module docstring).  trunc: the
    truncation distance in metres (default 3 voxels, not tuned); color: also keep mean RGB per point.  Storage is 8 bytes
    per point (20 with colour): 2.1 GB (5.4 GB) at the limit of 2^28 points."""

    def __init__(self, origin: Sequence[float], voxel: float, dims: Sequence[int], trunc: Optional[float] = None,
                 color: bool = False, device=None):
        voxel = float(voxel)
        self.dims, self.origin = _value_error(ops.check_volume_grid, "TSDFVolume", dims, origin, voxel)
        self.voxel = voxel
        self.trunc = 3.0 * voxel if trunc is None else float(trunc)
        if not (math.isfinite(self.trunc) and self.trunc > 0):
            raise ValueError(f"trunc must be finite and > 0, got {trunc}")
        if not isinstance(color, bool):
            raise ValueError(f"color must be a bool, got {color!r}")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise ValueError(f"TSDFVolume lives on a CUDA device (no CPU path exists), got {self.device}")
        nx, ny, nz = self.dims
        self._data = torch.zeros(5 if color else 2, nz, ny, nx, dtype=torch.float32, device=self.device)
        self._bufs = {}

    @property
    def tsdf(self) -> torch.Tensor:
        """F fp32 [nz, ny, nx] (a view; index [k, j, i])."""
        return self._data[0]

    @property
    def weight(self) -> torch.Tensor:
        """W fp32 [nz, ny, nx] (a view): the number of observations of each point."""
        return self._data[1]

    @property
    def color(self) -> Optional[torch.Tensor]:
        """Mean RGB fp32 [3, nz, ny, nx] (a view), or None without colour."""
        return self._data[2:5] if self._data.shape[0] == 5 else None

    def reset(self):
        """Forgets every observation (F = W = 0, colour 0)."""
        self._data.zero_()

    @torch.no_grad()
    def integrate(self, depth: torch.Tensor, intrinsics, cam_to_world, rgb: Optional[torch.Tensor] = None):
        """Fuses depth fp32 [B,H,W] or [H,W] in metres (0 / NaN: no measurement) seen from cam_to_world ([B,4,4] or
        [4,4], numpy or a CPU tensor) into the volume.  rgb fp32 [B,3,H,W] or [3,H,W] exactly when the volume keeps
        colour.  Frames are applied in order."""
        name = "TSDFVolume.integrate"
        if depth.dim() == 2:
            depth = depth.unsqueeze(0)
            rgb = None if rgb is None else rgb.unsqueeze(0)
        if depth.dim() != 3:
            raise ValueError(f"{name}: depth must be [B,H,W] or [H,W], got {tuple(depth.shape)}")
        b, h, w = depth.shape
        if depth.device != self.device or depth.dtype != torch.float32:
            raise ValueError(f"{name}: depth must be fp32 on {self.device}, got {depth.dtype} on {depth.device}")
        if (rgb is None) != (self.color is None):
            raise ValueError(f"{name}: pass rgb exactly when the volume keeps colour (color={self.color is not None})")
        if rgb is not None and (tuple(rgb.shape) != (b, 3, h, w) or rgb.device != self.device or
                                rgb.dtype != torch.float32):
            raise ValueError(f"{name}: rgb must be fp32 [{b}, 3, {h}, {w}] on {self.device}, got {rgb.dtype} "
                             f"{tuple(rgb.shape)} on {rgb.device}")
        k = _value_error(ops.check_intrinsics, name, intrinsics)
        T = _value_error(ops.check_poses, name, cam_to_world)
        if T.shape[0] != b:
            raise ValueError(f"{name}: {b} depth frames but {T.shape[0]} poses")
        _value_error(ops._check_planes, name, b, h, w)
        with torch.cuda.device(self.device):
            ops.tsdf_integrate(self.tsdf, self.weight, self.color, self.dims, self.origin, self.voxel, self.trunc,
                               depth.contiguous(), None if rgb is None else rgb.contiguous(), k, cam_to_world)

    @torch.no_grad()
    def raycast(self, intrinsics, cam_to_world, size: Tuple[int, int], step: Optional[float] = None,
                color: bool = False):
        """The z-depth fp32 [H,W] (size = (H, W)) of the first surface seen from cam_to_world ([4,4] host), 0 where no
        surface is hit.  step: the march's sample spacing along the ray (default half a voxel).  color=True (a volume
        that keeps colour): (depth, rgb fp32 [3,H,W]), the same depth and the mean colour at the hit, NaN where there
        is none."""
        name = "TSDFVolume.raycast"
        if not isinstance(color, bool):
            raise ValueError(f"{name}: color must be a bool, got {color!r}")
        if color and self.color is None:
            raise ValueError(f"{name}: color=True needs a volume that keeps colour (TSDFVolume(..., color=True))")
        k = _value_error(ops.check_intrinsics, name, intrinsics)
        T = _value_error(ops.check_poses, name, cam_to_world)
        if T.shape[0] != 1:
            raise ValueError(f"{name}: one pose [4,4], got {T.shape[0]}")
        try:
            h, w = (int(v) for v in size)
        except (TypeError, ValueError):
            raise ValueError(f"{name}: size must be (H, W), got {size!r}") from None
        _value_error(ops._check_planes, name, 1, h, w)
        step = 0.5 * self.voxel if step is None else float(step)
        if not (math.isfinite(step) and self.voxel / 64 <= step <= self.voxel):
            raise ValueError(f"{name}: step must lie in [voxel / 64, voxel], got {step}")
        out = torch.empty(h, w, dtype=torch.float32, device=self.device)
        if not color:
            with torch.cuda.device(self.device):
                ops.tsdf_raycast(self.tsdf, self.weight, self.dims, self.origin, self.voxel, k, cam_to_world, step,
                                 out)
            return out
        rgb = torch.empty(3, h, w, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            ops.tsdf_raycast_color(self.tsdf, self.weight, self.color, self.dims, self.origin, self.voxel, k,
                                   cam_to_world, step, out, rgb)
        return out, rgb

    @torch.no_grad()
    def extract_mesh(self) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """(vertices fp32 [V,3] in world coordinates, faces int32 [F,3], colors fp32 [V,3] or None): the marching-
        tetrahedra surface F = 0 of the observed points, normals (right-handed winding) pointing from F < 0 to F > 0,
        towards the cameras.  Synchronises once to read the two counts."""
        ws = self._buf("mesh_ws", (-(-ops.tsdf_mesh_workspace_bytes(self.dims) // 8),), torch.float64, self.device)
        counts = self._buf("mesh_counts", (2,), torch.int64, self.device)
        with torch.cuda.device(self.device):
            ops.tsdf_mesh_count(self.tsdf, self.weight, self.dims, ws, counts)
            nv, nf = counts.tolist()
            verts = torch.empty(nv, 3, dtype=torch.float32, device=self.device)
            faces = torch.empty(nf, 3, dtype=torch.int32, device=self.device)
            colors = None if self.color is None else torch.empty(nv, 3, dtype=torch.float32, device=self.device)
            if nv:
                ops.tsdf_mesh_emit(self.tsdf, self.weight, self.color, self.dims, self.origin, self.voxel, ws, verts,
                                   faces, colors)
        return verts, faces, colors


def write_ply(path, vertices, faces, colors=None):
    """Writes a binary little-endian PLY: float x, y, z per vertex (and uchar red, green, blue from colors in [0, 1],
    rounded), and the faces as uchar-counted int lists.  Arrays may be tensors on any device or numpy."""
    def host(a, dtype):
        a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
        return np.ascontiguousarray(a, dtype=dtype)
    v, f = host(vertices, "<f4").reshape(-1, 3), host(faces, "<i4").reshape(-1, 3)
    if f.size and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError("write_ply: a face index lies outside the vertices")
    props = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}", "property float x",
              "property float y", "property float z"]
    if colors is not None:
        c = host(colors, np.float64).reshape(-1, 3)
        if c.shape != v.shape:
            raise ValueError(f"write_ply: colors must be [{len(v)}, 3], got {c.shape}")
        props += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        header += ["property uchar red", "property uchar green", "property uchar blue"]
    header += [f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]
    vrec = np.empty(len(v), dtype=props)
    for a, key in enumerate("xyz"):
        vrec[key] = v[:, a]
    if colors is not None:
        q = np.rint(np.clip(np.nan_to_num(c), 0.0, 1.0) * 255.0).astype(np.uint8)
        for a, key in enumerate(("red", "green", "blue")):
            vrec[key] = q[:, a]
    frec = np.empty(len(f), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    frec["n"] = 3
    frec["idx"] = f
    with open(Path(path), "wb") as fh:
        fh.write(("\n".join(header) + "\n").encode("ascii"))
        fh.write(vrec.tobytes())
        fh.write(frec.tobytes())
