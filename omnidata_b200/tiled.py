"""Predict depth and normals on images of any size: tiled inference with on-device alignment and blending.

    from omnidata_b200.tiled import TiledPredictor
    pred = TiledPredictor(model, tile=(384, 384), overlap=64, max_batch=32)
    depth = pred(x)          # x: float [B,3,H,W] on the model's device, any H, W >= 1
    anchored = TiledPredictor(model, anchor=(768, 1024))     # depth: tiles fitted to a whole-image forward

`model(x)` takes H, W multiples of 32 with at most 4 096 patches.  TiledPredictor cuts the image into overlapping tiles
of a size the model takes (`tile_grid`), runs them through `model` itself in chunks of at most `max_batch` tiles, and
merges the predictions at the image's own size (csrc/tiled.cu):

- depth (`num_channels == 1`): the depth model is affine-invariant (trained with the MiDaS scale-and-shift-invariant
  loss), so each tile's prediction carries its own unknown scale and shift.  One least-squares problem per image finds a
  scale s_i and shift t_i per tile that make neighbouring tiles agree on their overlaps, with a small ridge towards
  s = 1, t = 0 that fixes the global affine gauge (include/omnidata_b200.h, odb_tile_align_solve);
- depth with `anchor=(h, w)`: the image is also resized to h x w (antialiased bilinear) and run through `model` whole;
  that prediction, resampled to the image's size, replaces the ridge: each tile's (s_i, t_i) is pulled towards fitting
  it, so the merge lands in the whole-image prediction's affine frame (odb_tile_align_solve_anchored).  One extra
  forward per image;
- normals: blended as predicted (s = 1, t = 0).

The blend weights fall off linearly over `overlap` pixels towards tile edges inside the image, and not at the image
border.  The result has the model's output layout at the input's size: [B,H,W] for one channel, else [B,C,H,W].
Inference only; the merge is deterministic and does not depend on the batch.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from . import _capi, ops
from .model import DPTDepthModel, check_input_size

MAX_TILES = _capi.TILE_MAX_TILES          # tiles per image the alignment solve takes (ODB_TILE_MAX_TILES)


def _axis(length: int, t: int, overlap: int) -> List[int]:
    if length <= t:
        return [0]
    n = -(-(length - overlap) // (t - overlap))
    return [(2 * k * (length - t) + n - 1) // (2 * (n - 1)) for k in range(n)]      # round(k (L - t) / (n - 1)), halves up


def tile_grid(H: int, W: int, tile: Tuple[int, int], overlap: int) -> Tuple[List[int], List[int]]:
    """Tile origins (rows, columns) of an H x W image: per axis of length L and tile length t, one tile at 0 when
    L <= t (the gather replicates the image's edge up to t), else n = ceil((L - overlap) / (t - overlap)) tiles at
    round(k (L - t) / (n - 1)).  Every tile lies inside the image and neighbours overlap by at least `overlap`.  Tiles
    are numbered row-major.  (csrc/tiled.cu: tile_count, tile_origin)"""
    return _axis(H, tile[0], overlap), _axis(W, tile[1], overlap)


def check_inference_input(name: str, model, x: torch.Tensor):
    """Refuses, before anything is launched, an input the predictor `name` does not take: `model` in training mode, x
    requiring grad, x not on a CUDA device, or x not [B,3,H,W]."""
    if getattr(model, "training", False):
        raise ValueError(f"{name} is inference only: call model.eval() first")
    if x.requires_grad:
        raise ValueError(f"{name} is inference only: x must not require grad")
    if not x.is_cuda:
        raise _capi.OdbError(f"{name} runs on a CUDA (sm_90a) device only; there is no CPU fallback")
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError(f"expected input [B,3,H,W], got {tuple(x.shape)}")


def check_predictor_size(predictor, h: int, w: int):
    """ValueError for an input size `predictor` refuses, before anything is launched: the forward's size rule for a
    `DPTDepthModel`, the tile cap for a `TiledPredictor`, [1, 65535] for anything else."""
    if isinstance(predictor, DPTDepthModel):
        check_input_size(h, w, predictor.arch["hybrid"], autograd=False)
    elif isinstance(predictor, TiledPredictor):
        predictor._grid(1, h, w)
    elif not (1 <= h <= 65535 and 1 <= w <= 65535):
        raise ValueError(f"member sizes must lie in [1, 65535], got {h}x{w}")


def chunked_forward(model, x: torch.Tensor, max_batch: int, out: torch.Tensor):
    """Runs `model` over x [B,3,h,w] in chunks of at most `max_batch` images into the preallocated fp32 out [B,C,H,W]:
    each chunk's prediction is copied, or resized (ops.resize_bilinear) where h x w differs from H x W."""
    C, H, W = out.shape[1:]
    h, w = x.shape[2:]
    for i in range(0, x.shape[0], max_batch):
        y = model(x[i:i + max_batch])
        n = y.shape[0]
        y = y.reshape(n, C, h, w)
        if (h, w) == (H, W):
            out[i:i + n].copy_(y)
        else:
            ops.resize_bilinear(y.float().contiguous(), out[i:i + n])


class TiledPredictor:
    """Runs `model` on overlapping tiles of any-size images and merges the predictions (module docstring)."""

    def __init__(self, model, tile: Tuple[int, int] = (384, 384), overlap: int = 64, max_batch: int = 32,
                 anchor: Optional[Tuple[int, int]] = None):
        th, tw = int(tile[0]), int(tile[1])
        check_input_size(th, tw, model.arch["hybrid"], autograd=False)
        if not 0 <= overlap < min(th, tw) / 2:
            raise ValueError(f"overlap must lie in [0, min(tile) / 2), got {overlap} for tile {th}x{tw}")
        if max_batch < 1:
            raise ValueError(f"max_batch must be at least 1, got {max_batch}")
        if anchor is not None:
            if model.num_channels != 1:
                raise ValueError(f"anchor applies to depth models only, got a model with {model.num_channels} channels")
            anchor = (int(anchor[0]), int(anchor[1]))
            check_input_size(anchor[0], anchor[1], model.arch["hybrid"], autograd=False)
        self.model = model
        self.tile = (th, tw)
        self.overlap = int(overlap)
        self.max_batch = int(max_batch)
        self.anchor = anchor

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        """The merged prediction of x float [B,3,H,W]: [B,H,W] for a one-channel model, else [B,C,H,W]."""
        pred = self.tile_predictions(x)
        g = self.anchor_prediction(x) if self.anchor is not None else None
        return self.merge(pred, x.shape[0], x.shape[2], x.shape[3], anchor=g)

    def _grid(self, B: int, H: int, W: int) -> Tuple[int, int]:
        th, tw = self.tile
        if min(B, H, W) < 1 or max(B, H, W) > 65535:
            raise ValueError(f"batch and image size must lie in [1, 65535], got {B}x{H}x{W}")
        oy, ox = tile_grid(H, W, self.tile, self.overlap)
        if len(oy) * len(ox) > MAX_TILES:
            raise ValueError(f"{H}x{W} needs {len(oy)} x {len(ox)} tiles of {th}x{tw}; at most {MAX_TILES} per image")
        return len(oy), len(ox)

    def tile_predictions(self, x: torch.Tensor) -> torch.Tensor:
        """`model` on the tiles of x (row-major per image, images in order), as fp32 [B*T, C, th, tw]."""
        model, (th, tw) = self.model, self.tile
        check_inference_input("TiledPredictor", model, x)
        B, _, H, W = x.shape
        ny, nx = self._grid(B, H, W)
        n, C = B * ny * nx, model.num_channels
        with torch.no_grad():
            x = x.detach().float().contiguous()
            tiles = torch.empty(n, 3, th, tw, device=x.device)
            ops.tile_gather(x, tiles, self.tile, self.overlap)
            pred = torch.empty(n, C, th, tw, device=x.device)
            chunked_forward(model, tiles, self.max_batch, pred)
        return pred

    def anchor_prediction(self, x: torch.Tensor) -> torch.Tensor:
        """The anchor of x float [B,3,H,W]: x resized to the anchor size, run through `model` in chunks of at most
        `max_batch` images, the prediction resized back to H x W; fp32 [B,H,W]."""
        if self.anchor is None:
            raise ValueError("this TiledPredictor has no anchor size")
        model, (ah, aw) = self.model, self.anchor
        B, _, H, W = x.shape
        with torch.no_grad():
            x = x.detach().float().contiguous()
            small = torch.empty(B, 3, ah, aw, device=x.device)
            ops.resize_bilinear(x, small)
            g_small = torch.empty(B, 1, ah, aw, device=x.device)
            chunked_forward(model, small, self.max_batch, g_small)
            g = torch.empty(B, H, W, device=x.device)
            ops.resize_bilinear(g_small.view(B, ah, aw), g)
        return g

    def merge(self, pred: torch.Tensor, B: int, H: int, W: int, anchor: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Aligns (one channel: depth) and blends tile predictions fp32 [B*T, C, th, tw] into the [B,(C,)H,W] output.
        With `anchor` (fp32 [B,H,W], `anchor_prediction`) the alignment fits the tiles to it instead of the ridge."""
        (th, tw), ov = self.tile, self.overlap
        ny, nx = self._grid(B, H, W)
        T, C = ny * nx, pred.shape[1]
        st = None
        if anchor is not None and C != 1:
            raise ValueError("an anchor applies to one-channel (depth) predictions only")
        if C == 1:
            st = torch.empty(B, T, 2, device=pred.device, dtype=torch.float64)
            moments = None
            if T > 1:
                moments = torch.empty(B, ops.tile_pairs(ny, nx), 6, device=pred.device, dtype=torch.float64)
                ops.tile_overlap_moments(pred.view(B * T, th, tw), moments, (H, W), self.tile, ov)
            if anchor is None:
                ops.tile_align_solve(moments, st, (ny, nx))
            else:
                am = torch.empty(B, T, 5, device=pred.device, dtype=torch.float64)
                ops.tile_anchor_moments(pred.view(B * T, th, tw), anchor, am, self.tile, ov)
                ops.tile_align_solve_anchored(moments, am, st, (ny, nx))
        out = torch.empty(B, C, H, W, device=pred.device)
        ops.tile_blend(pred, st, out, self.tile, ov)
        return out.squeeze(1) if C == 1 else out
