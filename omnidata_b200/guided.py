"""Full-resolution depth and normals from one low-resolution forward: guided upsampling with the fast guided filter (He &
Sun, "Fast Guided Image Filtering", 2015), steered by the input image, on the device.

    from omnidata_b200.guided import GuidedPredictor
    gp = GuidedPredictor(model, size=(768, 1024), radius=4, eps=1e-3, max_batch=32)
    out = gp(x)                     # x fp32 [B,3,H,W], any H, W -> [B,H,W] (depth) or [B,3,H,W] (normals)

`predictor` is a `DPTDepthModel` in eval() mode, a `TiledPredictor`, or anything with the same call contract and a
`num_channels` attribute; a `GuidedPredictor` has one too, so it can be a member predictor of an `EnsemblePredictor`.
A call:

1. g = x resized to size = h x w (`ops.resize_bilinear`; skipped when h x w is the input's own size);
2. p = predictor(g), in chunks of at most `max_batch` images;
3. per low-resolution pixel, the local linear model p_c ~ a_c . g + b_c fitted over the (2 radius + 1)^2 window around
   it (ridge eps), then a_c, b_c averaged over the same windows (fp64, csrc/guided.cu);
4. those coefficients resampled to H x W and applied to x itself: out_c = a_c . x + b_c (fp32).

The guide is x exactly as the predictor receives it, so `eps` is in squared units of x: the depth model's input lies in
[-1, 1], the normal model's in [0, 1].  `radius` is in low-resolution pixels.  The defaults (radius 4, eps 1e-3) are
not tuned: there is no checkpoint or dataset here to tune them on.  The filter is linear in the prediction, so filtering
s p + t gives s out + t: the output keeps the prediction's own scale and shift.  It is not clamped, and normals are
filtered per channel and not renormalised.

Inference only.  Deterministic and independent of the batch; after the first call at a batch size `refine` neither
synchronises nor allocates beyond its output (its scratch buffers are kept per shape), so a call can be captured in a
CUDA graph.  Whether guided output has lower task error than tiled output has not been evaluated: there is no trained
checkpoint or dataset here (`evaluate.py --mode guided` measures it on a dataset).
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import torch

from . import _capi, ops
from .tiled import TiledPredictor, check_inference_input, check_predictor_size, chunked_forward

MAX_RADIUS = _capi.GUIDED_MAX_RADIUS


class GuidedPredictor:
    """Predicts at `size` through `predictor` and upsamples the prediction with the input image as the guide (module
    docstring)."""

    def __init__(self, predictor, size: Tuple[int, int], radius: int = 4, eps: float = 1e-3, max_batch: int = 32):
        channels = predictor.model.num_channels if isinstance(predictor, TiledPredictor) else predictor.num_channels
        if channels not in (1, 3):
            raise ValueError(f"guided upsampling takes depth (1 channel) or normals (3 channels), got {channels} "
                             "channels")
        if isinstance(radius, bool) or int(radius) != radius or not 1 <= radius <= MAX_RADIUS:
            raise ValueError(f"radius must be an integer in [1, {MAX_RADIUS}], got {radius}")
        eps = float(eps)
        if not (math.isfinite(eps) and eps > 0):
            raise ValueError(f"eps must be finite and > 0, got {eps}")
        if max_batch < 1:
            raise ValueError(f"max_batch must be at least 1, got {max_batch}")
        h, w = int(size[0]), int(size[1])
        check_predictor_size(predictor, h, w)
        self.predictor = predictor
        self.size = (h, w)
        self.radius = int(radius)
        self.eps = eps
        self.max_batch = int(max_batch)
        self.num_channels = channels
        self._buffers: Dict[tuple, dict] = {}

    def _check_input(self, x: torch.Tensor):
        p = self.predictor
        check_inference_input("GuidedPredictor", p.model if isinstance(p, TiledPredictor) else p, x)
        B, _, H, W = x.shape
        if not (1 <= B <= 65535 and 1 <= H <= 65535 and 1 <= W <= 65535):
            raise ValueError(f"batch and image size must lie in [1, 65535], got {B}x{H}x{W}")

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        """The guided prediction of x fp32 [B,3,H,W]: [B,H,W] for depth, [B,3,H,W] for normals."""
        g, p = self.low_res_prediction(x)
        return self.refine(x, g, p)

    def _buffer(self, B: int, device) -> dict:
        key = (B, device)
        buf = self._buffers.get(key)
        if buf is None:
            (h, w), C = self.size, self.num_channels
            buf = {"guide": torch.empty(B, 3, h, w, device=device), "pred": torch.empty(B, C, h, w, device=device),
                   "coef": torch.empty(B, 4 * C, h, w, device=device),
                   "workspace": torch.empty(ops.guided_workspace_bytes(B, C, h, w) // 8, device=device,
                                            dtype=torch.float64)}
            self._buffers[key] = buf
        return buf

    def low_res_prediction(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """(g, p): x resized to `size` (x itself at its own size) and `predictor`'s prediction of it, fp32 [B,3,h,w] and
        [B,C,h,w].  The buffers are kept for the next call at this batch size, which overwrites them."""
        self._check_input(x)
        B, _, H, W = x.shape
        with torch.no_grad():
            x = x.detach().float().contiguous()
            buf = self._buffer(B, x.device)
            g = x
            if self.size != (H, W):
                g = buf["guide"]
                ops.resize_bilinear(x, g)
            chunked_forward(self.predictor, g, self.max_batch, buf["pred"])
        return g, buf["pred"]

    def refine(self, x: torch.Tensor, g: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
        """The guided filter of p fp32 [B,C,h,w] against g fp32 [B,3,h,w] (`low_res_prediction`), applied to x fp32
        [B,3,H,W]: [B,H,W] for depth, [B,3,H,W] for normals."""
        self._check_input(x)
        B, _, H, W = x.shape
        if tuple(g.shape) != (B, 3, *self.size) or tuple(p.shape) != (B, self.num_channels, *self.size):
            raise ValueError(f"expected g [{B},3,{self.size[0]},{self.size[1]}] and p [{B},{self.num_channels},"
                             f"{self.size[0]},{self.size[1]}], got {tuple(g.shape)} and {tuple(p.shape)}")
        with torch.no_grad():
            x = x.detach().float().contiguous()
            buf = self._buffer(B, x.device)
            ops.guided_coefficients(g, p, self.radius, self.eps, buf["workspace"], buf["coef"])
            out = torch.empty(B, self.num_channels, H, W, device=x.device)
            ops.guided_apply(x, buf["coef"], out)
        return out.squeeze(1) if self.num_channels == 1 else out
