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


BLOCK_RANGE = _capi.SPARSE_TSDF_BLOCK_RANGE
MAX_BLOCKS = _capi.SPARSE_TSDF_MAX_BLOCKS


class SparseTSDFVolume(_StepBuffers):
    """A TSDF volume without a box (csrc/sparse_volume.cu): the points X(p) = origin + voxel p, p in Z^3, stored in
    blocks of 8^3 that are allocated where depth is seen, so a scene of any extent fuses without knowing its bounds.
    A drop-in for TSDFVolume's integrate, raycast, extract_mesh and reset, with the same per-point arithmetic.

    A pixel with finite depth d, 0 < d <= max_depth, allocates every block meeting the box of its ray segment from
    z = d - trunc to z = d + trunc (max_depth, default 10 m and not tuned, limits allocation only).  Each block
    records the frame that first allocated it, counting frames from construction or reset(), and its points update
    only from that frame on, so the result does not depend on how frames are split into calls.  Block ids follow
    (birth frame, block key).  Storage is 2 KB per block (5 KB with colour); at most MAX_BLOCKS = 2^21 blocks (4.3 GB,
    10.7 GB with colour, 2^30 points), and block coordinates stay within +-BLOCK_RANGE = 2^20.  `integrate`
    synchronises once to read the number of new blocks (again when its hash table has to grow); `raycast` neither
    synchronises nor allocates beyond its output, so it can be captured in a CUDA graph.  Definitions: DESIGN.md §3
    "Sparse TSDF volumes"; oracle/sparse_volume_oracle.py restates them in float64."""

    _INITIAL_BLOCKS = 1024
    _INITIAL_TABLE = 1 << 14

    def __init__(self, voxel: float, trunc: Optional[float] = None, color: bool = False,
                 origin: Sequence[float] = (0.0, 0.0, 0.0), max_depth: float = 10.0, device=None):
        voxel = float(voxel)
        self.origin = _value_error(ops.check_volume_grid, "SparseTSDFVolume", (2, 2, 2), origin, voxel)[1]
        self.voxel = voxel
        self.trunc = 3.0 * voxel if trunc is None else float(trunc)
        if not (math.isfinite(self.trunc) and self.trunc > 0):
            raise ValueError(f"trunc must be finite and > 0, got {trunc}")
        self.max_depth = float(max_depth)
        if not (math.isfinite(self.max_depth) and self.max_depth > 0):
            raise ValueError(f"max_depth must be finite and > 0, got {max_depth}")
        if not isinstance(color, bool):
            raise ValueError(f"color must be a bool, got {color!r}")
        if any(abs(math.floor(o / (8.0 * voxel))) >= BLOCK_RANGE for o in self.origin):
            raise ValueError(f"SparseTSDFVolume: the origin {self.origin} lies {BLOCK_RANGE} or more blocks of "
                             f"8 x {voxel} m from the world's zero")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise ValueError(f"SparseTSDFVolume lives on a CUDA device (no CPU path exists), got {self.device}")
        self._channels = 5 if color else 2
        self._bufs = {}
        self._alloc_pool(self._INITIAL_BLOCKS)
        self._alloc_table(self._INITIAL_TABLE)
        self._bbox = torch.empty(6, dtype=torch.int32, device=self.device)
        self.reset()

    # -------------------------------------------------------------- state
    def _alloc_pool(self, cap: int):
        dev = self.device
        self._data = torch.empty(cap, self._channels, 512, dtype=torch.float32, device=dev)
        self._keys = torch.empty(cap, dtype=torch.int64, device=dev)
        self._birth = torch.empty(cap, dtype=torch.int32, device=dev)
        self._nbr = torch.empty(cap, 8, dtype=torch.int32, device=dev)

    def _alloc_table(self, size: int):
        dev = self.device
        self._tkeys = torch.empty(size, dtype=torch.int64, device=dev)
        self._tids = torch.empty(size, dtype=torch.int32, device=dev)
        self._tbirth = torch.empty(size, dtype=torch.int32, device=dev)
        self._scratch = torch.zeros(2 + size, dtype=torch.int32, device=dev)

    def _desc(self, blocks: Optional[int] = None):
        return ops.sparse_tsdf_desc(self._data, self._keys, self._birth, self._nbr, self._tkeys, self._tids,
                                    self._tbirth, self._bbox, self._scratch, self.blocks if blocks is None else blocks,
                                    self.origin, self.voxel)

    def reset(self):
        """Forgets every block and observation; frames count from 0 again."""
        self.blocks = 0
        self.frames = 0
        big = torch.iinfo(torch.int32)
        self._bbox.copy_(torch.tensor([big.max] * 3 + [big.min] * 3, dtype=torch.int32))
        with torch.cuda.device(self.device):
            ops.sparse_tsdf_rebuild(self._desc(), self.device)

    @property
    def block_keys(self) -> torch.Tensor:
        """int64 [blocks]: the packed block coordinates in id order (include/omnidata_b200.h)."""
        return self._keys[:self.blocks]

    @property
    def block_coords(self) -> torch.Tensor:
        """int64 [blocks, 3]: the (x, y, z) block coordinates in id order; block b holds the points 8 b + (0..7)^3."""
        k = self.block_keys
        m = (1 << 21) - 1
        return torch.stack([k & m, (k >> 21) & m, k >> 42], 1) - BLOCK_RANGE

    @property
    def block_birth(self) -> torch.Tensor:
        """int32 [blocks]: the frame that allocated each block."""
        return self._birth[:self.blocks]

    @property
    def tsdf(self) -> torch.Tensor:
        """F fp32 [blocks, 8, 8, 8] (a view; index [id, k, j, i])."""
        return self._data[:self.blocks, 0].view(-1, 8, 8, 8)

    @property
    def weight(self) -> torch.Tensor:
        """W fp32 [blocks, 8, 8, 8] (a view)."""
        return self._data[:self.blocks, 1].view(-1, 8, 8, 8)

    @property
    def color(self) -> Optional[torch.Tensor]:
        """Mean RGB fp32 [blocks, 3, 8, 8, 8] (a view), or None without colour."""
        return self._data[:self.blocks, 2:5].view(-1, 3, 8, 8, 8) if self._channels == 5 else None

    def bounds(self):
        """((x0, y0, z0), (x1, y1, z1)): the first and last point of the allocated blocks' bounding box in world
        coordinates, or None when nothing is allocated.  Synchronises."""
        if self.blocks == 0:
            return None
        b = self._bbox.tolist()
        lo = tuple(o + self.voxel * (8 * b[a]) for a, o in enumerate(self.origin))
        return lo, tuple(o + self.voxel * (8 * b[3 + a] + 7) for a, o in enumerate(self.origin))

    @torch.no_grad()
    def to_dense(self):
        """(origin, dims, F, W, C) of the allocated blocks' bounding box as a dense grid: origin = the volume's origin +
        voxel 8 bmin, dims = (nx, ny, nz), F, W fp32 [nz, ny, nx] and C fp32 [3, nz, ny, nx] or None, with F = W = 0
        (and colour 0) at unallocated points.  For tests and interop; synchronises."""
        if self.blocks == 0:
            return self.origin, (0, 0, 0), None, None, None
        b = self._bbox.tolist()
        nb = [b[3 + a] - b[a] + 1 for a in range(3)]
        ch = self._channels
        dense = torch.zeros(ch, 8 * nb[2], 8 * nb[1], 8 * nb[0], dtype=torch.float32, device=self.device)
        rel = self.block_coords - torch.tensor(b[:3], device=self.device)
        view = dense.view(ch, nb[2], 8, nb[1], 8, nb[0], 8).permute(1, 3, 5, 0, 2, 4, 6)
        view[rel[:, 2], rel[:, 1], rel[:, 0]] = self._data[:self.blocks].view(-1, ch, 8, 8, 8)
        origin = tuple(o + self.voxel * (8 * b[a]) for a, o in enumerate(self.origin))
        dims = (8 * nb[0], 8 * nb[1], 8 * nb[2])
        return origin, dims, dense[0], dense[1], dense[2:5] if ch == 5 else None

    def _check_centres(self, name, T):
        """ValueError unless every camera centre lies, with max_depth + trunc around it, inside the block range."""
        reach = (self.max_depth + self.trunc) / (8.0 * self.voxel)
        for t in T.reshape(-1, 16)[:, [3, 7, 11]]:
            for a in range(3):
                b = (t[a] - self.origin[a]) / (8.0 * self.voxel)
                if not abs(b) + reach < BLOCK_RANGE - 1:
                    raise ValueError(f"{name}: a camera centre {tuple(t)} lies outside the sparse volume's block "
                                     f"range (+-{BLOCK_RANGE} blocks of 8 x {self.voxel} m around the origin, less "
                                     f"max_depth + trunc)")

    # -------------------------------------------------------------- integrate / raycast / extract
    @torch.no_grad()
    def integrate(self, depth: torch.Tensor, intrinsics, cam_to_world, rgb: Optional[torch.Tensor] = None):
        """TSDFVolume.integrate's arguments and arithmetic; allocates the frames' blocks first.  ValueError, with the
        volume unchanged, when the blocks would exceed MAX_BLOCKS or a camera centre lies outside the block range."""
        name = "SparseTSDFVolume.integrate"
        if depth.dim() == 2:
            depth = depth.unsqueeze(0)
            rgb = None if rgb is None else rgb.unsqueeze(0)
        if depth.dim() != 3:
            raise ValueError(f"{name}: depth must be [B,H,W] or [H,W], got {tuple(depth.shape)}")
        b, h, w = depth.shape
        if depth.device != self.device or depth.dtype != torch.float32:
            raise ValueError(f"{name}: depth must be fp32 on {self.device}, got {depth.dtype} on {depth.device}")
        if (rgb is None) != (self._channels == 2):
            raise ValueError(f"{name}: pass rgb exactly when the volume keeps colour (color={self._channels == 5})")
        if rgb is not None and (tuple(rgb.shape) != (b, 3, h, w) or rgb.device != self.device or
                                rgb.dtype != torch.float32):
            raise ValueError(f"{name}: rgb must be fp32 [{b}, 3, {h}, {w}] on {self.device}, got {rgb.dtype} "
                             f"{tuple(rgb.shape)} on {rgb.device}")
        k = _value_error(ops.check_intrinsics, name, intrinsics)
        T = _value_error(ops.check_poses, name, cam_to_world)
        if T.shape[0] != b:
            raise ValueError(f"{name}: {b} depth frames but {T.shape[0]} poses")
        _value_error(ops._check_planes, name, b, h, w)
        self._check_centres(name, T)
        if self.frames + b > torch.iinfo(torch.int32).max:
            raise ValueError(f"{name}: more than 2^31 - 1 frames since the last reset")
        depth = depth.contiguous()
        T = T.reshape(-1, 4, 4)
        dev = self.device
        with torch.cuda.device(dev):
            while True:
                ops.sparse_tsdf_mark(self._desc(), dev, self.trunc, self.max_depth, depth, k, T, self.frames)
                n_new, full = self._scratch[:2].tolist()
                if not full and self.blocks + n_new <= self._tkeys.numel() // 2:
                    break
                if self._tkeys.numel() >= 2 * MAX_BLOCKS:
                    n_new = MAX_BLOCKS + 1 - self.blocks          # the limit is exceeded whatever the exact count
                    break
                self._alloc_table(2 * self._tkeys.numel())
                ops.sparse_tsdf_rebuild(self._desc(), dev)
            if self.blocks + n_new > MAX_BLOCKS:
                ops.sparse_tsdf_rebuild(self._desc(), dev)      # forget the uncommitted marks
                raise ValueError(f"{name}: the frames need more than MAX_BLOCKS = {MAX_BLOCKS} blocks of 8^3 points "
                                 f"({self.blocks} allocated); use a coarser voxel or a smaller max_depth")
            if self.blocks + n_new > self._data.shape[0]:
                cap = self._data.shape[0]
                while cap < self.blocks + n_new:
                    cap *= 2
                old = (self._data, self._keys, self._birth, self._nbr)
                self._alloc_pool(min(cap, MAX_BLOCKS))
                for new, o in zip((self._data, self._keys, self._birth, self._nbr), old):
                    new[:self.blocks] = o[:self.blocks]
            if n_new:
                ws = self._buf("commit_ws", (-(-ops.sparse_tsdf_commit_workspace_bytes(n_new) // 8),), torch.float64,
                               dev)
                ops.sparse_tsdf_commit(self._desc(), dev, n_new, ws)
                self.blocks += n_new
            ops.sparse_tsdf_integrate(self._desc(), dev, self.trunc, depth, None if rgb is None else rgb.contiguous(),
                                      k, T, self.frames)
        self.frames += b

    @torch.no_grad()
    def raycast(self, intrinsics, cam_to_world, size: Tuple[int, int], step: Optional[float] = None,
                color: bool = False):
        """TSDFVolume.raycast over the allocated blocks' bounding box, with unallocated points unobserved; the march
        skips unallocated blocks without changing a bit of the result."""
        name = "SparseTSDFVolume.raycast"
        if not isinstance(color, bool):
            raise ValueError(f"{name}: color must be a bool, got {color!r}")
        if color and self._channels != 5:
            raise ValueError(f"{name}: color=True needs a volume that keeps colour (SparseTSDFVolume(..., color=True))")
        k = _value_error(ops.check_intrinsics, name, intrinsics)
        T = _value_error(ops.check_poses, name, cam_to_world)
        if T.shape[0] != 1:
            raise ValueError(f"{name}: one pose [4,4], got {T.shape[0]}")
        self._check_centres(name, T)
        try:
            h, w = (int(v) for v in size)
        except (TypeError, ValueError):
            raise ValueError(f"{name}: size must be (H, W), got {size!r}") from None
        _value_error(ops._check_planes, name, 1, h, w)
        step = 0.5 * self.voxel if step is None else float(step)
        if not (math.isfinite(step) and self.voxel / 64 <= step <= self.voxel):
            raise ValueError(f"{name}: step must lie in [voxel / 64, voxel], got {step}")
        out = torch.empty(h, w, dtype=torch.float32, device=self.device)
        rgb = torch.empty(3, h, w, dtype=torch.float32, device=self.device) if color else None
        with torch.cuda.device(self.device):
            ops.sparse_tsdf_raycast(self._desc(), self.device, k, T.reshape(4, 4), step, out, rgb)
        return (out, rgb) if color else out

    @torch.no_grad()
    def extract_mesh(self) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """TSDFVolume.extract_mesh over the allocated points: vertex ids in (block id, point, direction) order, faces
        in (block id, cell, tetrahedron, triangle) order.  Synchronises once to read the two counts."""
        dev = self.device
        ws = self._buf("mesh_ws", (-(-ops.sparse_tsdf_mesh_workspace_bytes(self.blocks) // 8),), torch.float64, dev)
        counts = self._buf("mesh_counts", (2,), torch.int64, dev)
        desc = self._desc()
        with torch.cuda.device(dev):
            ops.sparse_tsdf_mesh_count(desc, dev, ws, counts)
            nv, nf = counts.tolist()
            if nv >= 2 ** 31:
                raise ValueError(f"SparseTSDFVolume.extract_mesh: {nv} vertices exceed int32 face indices")
            verts = torch.empty(nv, 3, dtype=torch.float32, device=dev)
            faces = torch.empty(nf, 3, dtype=torch.int32, device=dev)
            colors = None if self._channels == 2 else torch.empty(nv, 3, dtype=torch.float32, device=dev)
            if nv:
                ops.sparse_tsdf_mesh_emit(desc, dev, ws, verts, faces, colors)
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


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4",
              "float32": "f4", "double": "f8", "float64": "f8"}


def read_ply(path):
    """Reads a triangle or polygon mesh PLY (binary little-endian or ascii): (vertices fp32 [V,3], faces int32 [F,3],
    colors fp32 [V,3] in [0, 1] or None) as numpy arrays.  Vertex x, y, z may be float or double; other vertex
    properties of any scalar type are skipped except red, green, blue (uchar read as q / 255).  Faces are a list of
    int / uint indices with a uchar, ushort, int or uint count; polygons are fan-triangulated ((v0, v_i, v_i+1)), so
    Replica's quads read as two triangles each.  Other elements must have scalar properties only and are skipped.
    ValueError, naming the file, for big-endian files, missing x / y / z, indices outside the vertices, polygons of
    fewer than 3 vertices and truncated files.  Reads what write_ply writes exactly."""
    path = Path(path)

    def bad(msg):
        return ValueError(f"read_ply: {path}: {msg}")

    data = path.read_bytes()

    def parse():
        end = data.find(b"end_header")
        if not data.startswith(b"ply") or end < 0:
            raise bad("not a PLY file")
        nl = data.find(b"\n", end)
        if nl < 0:
            raise bad("truncated header")
        body = nl + 1
        fmt, elements = None, []
        for line in data[:end].decode("ascii", errors="replace").splitlines()[1:]:
            tok = line.split()
            if not tok or tok[0] in ("comment", "obj_info"):
                continue
            if tok[0] == "format":
                fmt = tok[1] if len(tok) > 1 else None
            elif tok[0] == "element" and len(tok) == 3:
                if int(tok[2]) < 0:
                    raise bad(f"negative element count in {line!r}")
                elements.append((tok[1], int(tok[2]), []))
            elif tok[0] == "property" and elements:
                if tok[1] == "list" and len(tok) == 5:
                    if tok[2] not in _PLY_TYPES or tok[3] not in _PLY_TYPES:
                        raise bad(f"unknown property type in {line!r}")
                    elements[-1][2].append((tok[4], "list", _PLY_TYPES[tok[2]], _PLY_TYPES[tok[3]]))
                elif len(tok) == 3 and tok[1] in _PLY_TYPES:
                    elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
                else:
                    raise bad(f"cannot parse {line!r}")
            else:
                raise bad(f"cannot parse {line!r}")
        if fmt == "binary_big_endian":
            raise bad("big-endian PLY is not supported")
        if fmt not in ("binary_little_endian", "ascii"):
            raise bad(f"unknown format {fmt!r}")
        ascii_ = fmt == "ascii"
        tokens = data[body:].split() if ascii_ else None
        pos = 0                                                   # byte offset (binary) or token index (ascii)
        verts = colors = faces = None
        for name, count, props in elements:
            lists = [p for p in props if p[1] == "list"]
            if name == "face":
                if len(props) != 1 or not lists or lists[0][0] not in ("vertex_indices", "vertex_index"):
                    raise bad("faces must have exactly one list property vertex_indices")
                _, _, ct, it = lists[0]
                if ct not in ("u1", "u2", "i4", "u4") or it not in ("i4", "u4"):
                    raise bad("face lists need a uchar / ushort / int / uint count and int / uint indices")
                polys, pos = _ply_lists(tokens, data, pos, count, ct, it, ascii_, bad)
                faces = _fan(polys, bad)
                continue
            if lists:
                raise bad(f"element {name!r} has a list property; only faces may")
            dt = np.dtype([(p[0], "<" + p[1]) for p in props])
            if ascii_:
                if pos + count * len(props) > len(tokens):
                    raise bad(f"truncated element {name!r}")
                cols = np.asarray(tokens[pos:pos + count * len(props)], dtype=np.float64).reshape(count, len(props))
                pos += count * len(props)
                rec = {p[0]: cols[:, q] for q, p in enumerate(props)}
            else:
                if pos + count * dt.itemsize > len(data) - body:
                    raise bad(f"truncated element {name!r}")
                arr = np.frombuffer(data, dtype=dt, count=count, offset=body + pos)
                pos += count * dt.itemsize
                rec = {p[0]: arr[p[0]] for p in props}
            if name == "vertex":
                types = {p[0]: p[1] for p in props}
                if not all(types.get(k) in ("f4", "f8") for k in "xyz"):
                    raise bad("vertices need float or double x, y, z")
                verts = np.stack([np.asarray(rec[k]).astype(np.float32) for k in "xyz"], 1)
                if all(k in types for k in ("red", "green", "blue")):
                    scale = {"u1": 255.0, "u2": 65535.0}.get(types["red"], 1.0)
                    colors = np.stack([(np.asarray(rec[k], np.float64) / scale).astype(np.float32)
                                       for k in ("red", "green", "blue")], 1)
        if verts is None:
            raise bad("no vertex element")
        if faces is None:
            faces = np.zeros((0, 3), np.int64)
        if faces.size and (faces.min() < 0 or faces.max() >= len(verts)):
            raise bad("a face index lies outside the vertices")
        return np.ascontiguousarray(verts), faces.astype(np.int32).reshape(-1, 3), colors

    try:
        return parse()
    except (ValueError, IndexError, OverflowError) as e:   # a malformed number or count: name the file
        if str(path) in str(e):
            raise
        raise bad(f"malformed file ({e})") from None


def _ply_lists(tokens, data, pos, count, ct, it, ascii_, bad):
    """The polygons of a face element: a list of int64 arrays [n_i] (all of one length: an array [F, n])."""
    if ascii_:
        polys = []
        for _ in range(count):
            if pos >= len(tokens):
                raise bad("truncated faces")
            n = int(tokens[pos])
            if pos + 1 + n > len(tokens):
                raise bad("truncated faces")
            polys.append(np.asarray(tokens[pos + 1:pos + 1 + n], dtype=np.int64))
            pos += 1 + n
        return polys, pos
    body = data.index(b"\n", data.find(b"end_header")) + 1
    cs, isz = np.dtype(ct).itemsize, np.dtype(it).itemsize
    if count == 0:
        return np.zeros((0, 3), np.int64), pos
    if body + pos + cs > len(data):
        raise bad("truncated faces")
    n0 = int(np.frombuffer(data, dtype="<" + ct, count=1, offset=body + pos)[0])
    # Read at the stride of n0-gons.  Exact whenever every count read so equals n0: record r's count is read at its
    # true offset as long as records 0..r-1 are n0-gons, so the first polygon of another size is read where it lies
    # and fails the check; no misaligned field is ever compared.
    uniform = np.dtype([("n", "<" + ct), ("i", "<" + it, (n0,))])
    if body + pos + count * uniform.itemsize <= len(data):
        arr = np.frombuffer(data, dtype=uniform, count=count, offset=body + pos)
        if (arr["n"] == n0).all():
            return arr["i"].astype(np.int64).reshape(count, n0), pos + count * uniform.itemsize
    polys = []                                                # mixed polygon sizes: one at a time
    for _ in range(count):
        if body + pos + cs > len(data):
            raise bad("truncated faces")
        n = int(np.frombuffer(data, dtype="<" + ct, count=1, offset=body + pos)[0])
        if body + pos + cs + n * isz > len(data):
            raise bad("truncated faces")
        polys.append(np.frombuffer(data, dtype="<" + it, count=n, offset=body + pos + cs).astype(np.int64))
        pos += cs + n * isz
    return polys, pos


def _fan(polys, bad) -> np.ndarray:
    """Fan triangulation (v0, v_i, v_i+1), i = 1 .. n - 2, of each polygon, in polygon order."""
    if isinstance(polys, np.ndarray):
        n = polys.shape[1] if polys.ndim == 2 else 3
        if len(polys) and n < 3:
            raise bad(f"a face has {n} vertices")
        if not len(polys):
            return np.zeros((0, 3), np.int64)
        return np.stack([np.stack([polys[:, 0], polys[:, i], polys[:, i + 1]], 1) for i in range(1, n - 1)],
                        1).reshape(-1, 3)
    out = []
    for p in polys:
        if len(p) < 3:
            raise bad(f"a face has {len(p)} vertices")
        out.extend((p[0], p[i], p[i + 1]) for i in range(1, len(p) - 1))
    return np.asarray(out, np.int64).reshape(-1, 3)
