"""Test-time ensembles of depth and surface-normal predictions: several predictions of one image (mirrored, and at
several input sizes) put in one frame and merged per pixel on the device.

    from omnidata_b200.ensemble import EnsemblePredictor
    ens = EnsemblePredictor(model, sizes=[None, (512, 768)], flip=True, max_batch=32)
    out = ens(x)                                  # x fp32 [B,3,H,W] -> [B,H,W] (depth) or [B,3,H,W] (normals)
    out, spread = ens(x, return_spread=True)      # + a per-pixel spread map [B,H,W]

`predictor` is a `DPTDepthModel` in eval() mode or a `TiledPredictor` (multi-scale tiled ensembles); anything with the
same call contract and a `num_channels` attribute works too.  Members, in order: for each entry of `sizes` (None: the
input's own size) the prediction of the input resized to that size (`ops.resize_bilinear`, skipped at equal size), then,
with `flip`, the prediction of its horizontal mirror; each is resized back to H x W.  Member 0 is the reference frame.
K = len(sizes) * (1 + flip) members, 1 <= K <= 16; K = 1 returns `predictor(x)` unchanged.  Members are stored as
predicted, still mirrored: the merge kernels read them un-mirrored (csrc/ensemble.cu).

- depth (`num_channels == 1`): each member carries its own scale and shift (the models are affine-invariant), so per
  image one least-squares problem puts all members in member 0's frame (s_0 = 1, t_0 = 0; include/omnidata_b200.h
  odb_ensemble_align_solve), and the output is the per-pixel median of s_k a_k + t_k; spread = the median absolute
  deviation from it.  A pixel where any member is not finite gets member 0's value and spread NaN.  Not clamped;
- normals (`num_channels == 3`): the members are clamped to [0, 1] and decoded (2c - 1), the x component of a mirrored
  member negated; the output is the normalised mean vector re-encoded, spread = the members' mean angle to it in
  degrees.

Inference only.  The merge is deterministic, independent of the batch, and neither synchronises nor allocates beyond
its outputs after its first call at a shape (its scratch buffers are kept per shape).  Whether ensembling lowers task
error has not been evaluated: there is no trained checkpoint or dataset here.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _capi, ops
from .tiled import TiledPredictor, check_inference_input, check_predictor_size, chunked_forward

MAX_MEMBERS = _capi.ENSEMBLE_MAX_MEMBERS


class EnsemblePredictor:
    """Predicts each image K times (sizes x mirror) through `predictor` and merges the predictions (module docstring)."""

    def __init__(self, predictor, sizes: Optional[Sequence[Optional[Tuple[int, int]]]] = None, flip: bool = True,
                 max_batch: int = 32):
        sizes = [None] if sizes is None else [None if s is None else (int(s[0]), int(s[1])) for s in sizes]
        if not sizes:
            raise ValueError("sizes must name at least one input size (None: the input's own)")
        k = len(sizes) * (2 if flip else 1)
        if k > MAX_MEMBERS:
            raise ValueError(f"{len(sizes)} sizes{' x 2 (flip)' if flip else ''} make {k} members; at most {MAX_MEMBERS}")
        if max_batch < 1:
            raise ValueError(f"max_batch must be at least 1, got {max_batch}")
        channels = predictor.model.num_channels if isinstance(predictor, TiledPredictor) else predictor.num_channels
        if channels not in (1, 3):
            raise ValueError(f"ensembles merge depth (1 channel) or normals (3 channels), got {channels} channels")
        for s in sizes:
            if s is not None:
                check_predictor_size(predictor, *s)
        self.predictor = predictor
        self.sizes: List[Optional[Tuple[int, int]]] = sizes
        self.flip = bool(flip)
        self.max_batch = int(max_batch)
        self.num_channels = channels
        self.members = [(s, f) for s in sizes for f in ((False, True) if flip else (False,))]
        self.flips = sum(1 << i for i, (_, f) in enumerate(self.members) if f)      # member i mirrored: bit i
        self._buffers: Dict[tuple, dict] = {}

    def _check_input(self, x: torch.Tensor):
        p = self.predictor
        check_inference_input("EnsemblePredictor", p.model if isinstance(p, TiledPredictor) else p, x)
        B, _, H, W = x.shape
        if not 1 <= B <= 65535:
            raise ValueError(f"batch must lie in [1, 65535], got {B}")
        for s in self.sizes:
            check_predictor_size(p, *(s or (H, W)))

    def __call__(self, x: torch.Tensor, return_spread: bool = False):
        """The merged prediction of x float [B,3,H,W]: [B,H,W] for depth, [B,3,H,W] for normals; with
        `return_spread`, also the spread fp32 [B,H,W]."""
        self._check_input(x)
        if len(self.members) == 1:
            with torch.no_grad():
                out = self.predictor(x)
            if not return_spread:
                return out
            B, _, H, W = x.shape                  # one member: no spread (NaN where a depth is not finite)
            spread = torch.zeros(B, H, W, device=x.device)
            if self.num_channels == 1:
                spread.masked_fill_(~torch.isfinite(out.view(B, H, W)), float("nan"))
            return out, spread
        return self.merge(self.member_predictions(x), return_spread)

    def _buffer(self, B: int, H: int, W: int, device) -> dict:
        key = (B, H, W, device)
        buf = self._buffers.get(key)
        if buf is None:
            K, C = len(self.members), self.num_channels
            buf = {"members": torch.empty(K, B, C, H, W, device=device)}
            if C == 1:
                buf["gram"] = torch.empty(B, (K + 1) * (K + 2) // 2, device=device, dtype=torch.float64)
                buf["workspace"] = torch.empty(ops.ensemble_gram_workspace_bytes(K, B, H, W) // 8, device=device,
                                               dtype=torch.float64)
                buf["scale_shift"] = torch.empty(B, K, 2, device=device, dtype=torch.float64)
            self._buffers[key] = buf
        return buf

    def member_predictions(self, x: torch.Tensor) -> torch.Tensor:
        """The K members of x float [B,3,H,W] at H x W, mirrored ones still mirrored: fp32 [K, B, C, H, W].  The
        buffer is kept for the next call at this shape, which overwrites it."""
        self._check_input(x)
        B, _, H, W = x.shape
        with torch.no_grad():
            x = x.detach().float().contiguous()
            members = self._buffer(B, H, W, x.device)["members"]
            k = 0
            for size in self.sizes:
                h, w = size or (H, W)
                xs = x
                if (h, w) != (H, W):
                    xs = torch.empty(B, 3, h, w, device=x.device)
                    ops.resize_bilinear(x, xs)
                for flipped in ((False, True) if self.flip else (False,)):
                    xin = torch.flip(xs, dims=(3,)) if flipped else xs
                    chunked_forward(self.predictor, xin, self.max_batch, members[k])
                    k += 1
        return members

    def merge(self, members: torch.Tensor, return_spread: bool = False):
        """Merges members fp32 [K, B, C, H, W] (`member_predictions`) into the output (and the spread)."""
        K, B, C, H, W = members.shape
        if K != len(self.members) or C != self.num_channels:
            raise ValueError(f"expected {len(self.members)} members of {self.num_channels} channels, got "
                             f"{tuple(members.shape)}")
        spread = torch.empty(B, H, W, device=members.device) if return_spread else None
        if C == 1:
            buf = self._buffer(B, H, W, members.device)
            ops.ensemble_gram(members, self.flips, buf["gram"], buf["workspace"])
            ops.ensemble_align_solve(buf["gram"], buf["scale_shift"])
            out = torch.empty(B, H, W, device=members.device)
            ops.ensemble_merge_depth(members, self.flips, buf["scale_shift"], out, spread)
        else:
            out = torch.empty(B, 3, H, W, device=members.device)
            ops.ensemble_merge_normal(members, self.flips, out, spread)
        return (out, spread) if return_spread else out
