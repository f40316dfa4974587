"""Float64 restatement of the sparse TSDF volume (DESIGN.md §3 "Sparse TSDF volumes", csrc/sparse_volume.cu) in numpy,
for small scenes: block allocation (the exact block set, birth frames and ids), the birth-masked integration (built on
volume_oracle.integrate with index_offset), the raycast (volume_oracle's full, unskipped march over the dense grid of the
allocated blocks' bounding box) and extraction through that dense grid.

Blocks hold the points p = 8 b + (0..7)^3; a block's key packs (bz, by, bx) + 2^20 into 21 bits each, bz highest."""
from __future__ import annotations

import numpy as np

from . import color_volume_oracle, volume_oracle

BLOCK_RANGE = 1 << 20


def pack_key(b) -> int:
    bx, by, bz = (int(v) + BLOCK_RANGE for v in b)
    return (bz << 42) | (by << 21) | bx


def unpack_key(k: int):
    m = (1 << 21) - 1
    return (k & m) - BLOCK_RANGE, ((k >> 21) & m) - BLOCK_RANGE, (k >> 42) - BLOCK_RANGE


def pixel_block_boxes(depth, K, pose, origin, voxel, trunc, max_depth):
    """(lo, hi) int64 [P, 3]: the block box of each allocating pixel of depth [H,W] seen from pose (the box of its ray
    segment's two endpoints, z = d -+ trunc), in the kernel's fp64 operation order."""
    depth = np.asarray(depth, np.float32)
    h, w = depth.shape
    fx, fy, cx, cy = (float(v) for v in K)
    T = np.asarray(pose, np.float64).reshape(4, 4)
    y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    d = depth.astype(np.float64)
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(d) & (d > 0) & (d <= max_depth)
    d, rx, ry = d[ok], ((x - cx) / fx)[ok], ((y - cy) / fy)[ok]
    blocks = []
    for z in (d - trunc, d + trunc):
        xc, yc = z * rx, z * ry
        X = [((T[a, 0] * xc + T[a, 1] * yc) + T[a, 2] * z) + T[a, 3] for a in range(3)]
        blocks.append(np.stack([np.floor(((X[a] - origin[a]) / voxel) * 0.125) for a in range(3)], 1))
    lo, hi = np.minimum(*blocks), np.maximum(*blocks)
    inside = (lo > -BLOCK_RANGE).all(1) & (hi < BLOCK_RANGE).all(1)
    return lo[inside].astype(np.int64), hi[inside].astype(np.int64)


def frame_blocks(depth, K, pose, origin, voxel, trunc, max_depth) -> set:
    """The set of block keys one frame allocates."""
    lo, hi = pixel_block_boxes(depth, K, pose, origin, voxel, trunc, max_depth)
    keys = set()
    if len(lo) == 0:
        return keys
    ext = (hi - lo).max(0)
    for dz in range(ext[2] + 1):
        for dy in range(ext[1] + 1):
            for dx in range(ext[0] + 1):
                off = np.array([dx, dy, dz])
                sel = (off <= hi - lo).all(1)
                b = lo[sel] + off
                packed = ((b[:, 2] + BLOCK_RANGE) << 42) | ((b[:, 1] + BLOCK_RANGE) << 21) | (b[:, 0] + BLOCK_RANGE)
                keys.update(int(k) for k in np.unique(packed))
    return keys


class SparseVolume:
    """The oracle's sparse volume: keys int64 [n] and birth int32 [n] in id order, data float32 [n, 2 or 5, 512]."""

    def __init__(self, voxel, trunc=None, color=False, origin=(0.0, 0.0, 0.0), max_depth=10.0):
        self.voxel, self.origin = float(voxel), tuple(float(v) for v in origin)
        self.trunc = 3.0 * self.voxel if trunc is None else float(trunc)
        self.max_depth, self.ch = float(max_depth), 5 if color else 2
        self.keys = np.zeros(0, np.int64)
        self.birth = np.zeros(0, np.int32)
        self.data = np.zeros((0, self.ch, 512), np.float32)
        self.frames = 0

    def allocate(self, depth, K, poses):
        """Allocates the blocks of frames depth [B,H,W] at poses [B,4,4], numbered from self.frames: new ids in the
        order (birth frame, key)."""
        known = set(int(k) for k in self.keys)
        birth = {}
        for f, (dm, T) in enumerate(zip(np.asarray(depth, np.float32), np.asarray(poses, np.float64).reshape(-1, 4, 4))):
            for k in frame_blocks(dm, K, T, self.origin, self.voxel, self.trunc, self.max_depth):
                if k not in known and k not in birth:
                    birth[k] = self.frames + f
        new = sorted(birth.items(), key=lambda kv: (kv[1], kv[0]))
        self.keys = np.concatenate([self.keys, np.array([k for k, _ in new], np.int64)])
        self.birth = np.concatenate([self.birth, np.array([g for _, g in new], np.int32)])
        self.data = np.concatenate([self.data, np.zeros((len(new), self.ch, 512), np.float32)])

    def coords(self) -> np.ndarray:
        return np.array([unpack_key(int(k)) for k in self.keys], np.int64).reshape(-1, 3)

    def bbox(self):
        c = self.coords()
        return c.min(0), c.max(0)

    def _dense(self, values, fill):
        """values [n, ...per-point..., 512] scattered into the bounding box grid [..., nz, ny, nx]."""
        bmin, bmax = self.bbox()
        nb = bmax - bmin + 1
        lead = values.shape[1:-1]
        out = np.full(lead + (nb[2], 8, nb[1], 8, nb[0], 8), fill, values.dtype)
        rel = self.coords() - bmin
        v = values.reshape((len(values),) + lead + (8, 8, 8))
        for q, (bx, by, bz) in enumerate(rel):
            out[..., bz, :, by, :, bx, :] = v[q]
        return out.reshape(lead + (8 * nb[2], 8 * nb[1], 8 * nb[0]))

    def _undense(self, grid):
        bmin, _ = self.bbox()
        out = []
        for bx, by, bz in self.coords() - bmin:
            out.append(grid[..., 8 * bz:8 * bz + 8, 8 * by:8 * by + 8, 8 * bx:8 * bx + 8].reshape(grid.shape[:-3] +
                                                                                                    (512,)))
        return np.stack(out)

    def integrate(self, depth, K, poses, rgb=None):
        """Allocation, then every frame g at the points whose block has birth <= g (volume_oracle.integrate)."""
        depth = np.asarray(depth, np.float32).reshape((-1,) + np.shape(depth)[-2:])
        poses = np.asarray(poses, np.float64).reshape(-1, 4, 4)
        self.allocate(depth, K, poses)
        if len(self.keys):
            bmin, _ = self.bbox()
            offset = tuple(int(v) for v in 8 * bmin)
            F, W = self._dense(self.data[:, 0], 0.0), self._dense(self.data[:, 1], 0.0)
            C = self._dense(self.data[:, 2:5], 0.0) if self.ch == 5 else None
            born = self._dense(np.repeat(self.birth[:, None], 512, 1), np.iinfo(np.int32).max)
            for f in range(len(depth)):
                g = self.frames + f
                Fn, Wn, Cn = volume_oracle.integrate(F, W, C, self.origin, self.voxel, self.trunc, depth[f:f + 1], K,
                                                     poses[f:f + 1], None if rgb is None else np.asarray(rgb)[f:f + 1],
                                                     index_offset=offset)
                m = born <= g
                F, W = np.where(m, Fn, F), np.where(m, Wn, W)
                if C is not None:
                    C = np.where(m, Cn, C)
            self.data[:, 0], self.data[:, 1] = self._undense(F), self._undense(W)
            if C is not None:
                self.data[:, 2:5] = self._undense(C)
        self.frames += len(depth)

    def to_dense(self):
        """(origin, dims, F, W, C) of the bounding box grid, as SparseTSDFVolume.to_dense."""
        bmin, bmax = self.bbox()
        origin = tuple(self.origin[a] + self.voxel * float(8 * bmin[a]) for a in range(3))
        dims = tuple(int(v) for v in 8 * (bmax - bmin + 1))
        F, W = self._dense(self.data[:, 0], 0.0), self._dense(self.data[:, 1], 0.0)
        C = self._dense(self.data[:, 2:5], 0.0) if self.ch == 5 else None
        return origin, dims, F, W, C

    def raycast(self, K, pose, size, step=None, color=False):
        """The full, unskipped march of volume_oracle.raycast (color: color_volume_oracle.raycast_color) over the
        bounding box grid; zeros (and NaN colour) when nothing is allocated."""
        step = 0.5 * self.voxel if step is None else step
        if len(self.keys) == 0:
            z = np.zeros(size, np.float32)
            return (z, np.full((3,) + tuple(size), np.nan, np.float32)) if color else z
        lo, _, F, W, C = self.to_dense()
        if color:
            return color_volume_oracle.raycast_color(F, W, C, lo, self.voxel, K, pose, size, step)
        return volume_oracle.raycast(F, W, lo, self.voxel, K, pose, size, step)

    def extract_mesh(self):
        """volume_oracle.extract_mesh of the bounding box grid with the sparse lattice's vertex positions (dense
        (k, j, i, direction) order, not the kernels' block order)."""
        _, _, F, W, C = self.to_dense()
        bmin, _ = self.bbox()
        return volume_oracle.extract_mesh(F, W, C, self.origin, self.voxel,
                                          index_offset=tuple(int(v) for v in 8 * bmin))
