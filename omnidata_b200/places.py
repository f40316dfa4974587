"""Recognise places by appearance on the device (csrc/places.cu): randomized-fern codes of frames and a nearest-code
lookup over a database of keyframes (Glocker et al., "Real-time RGB-D camera relocalization via randomized ferns",
2015; the keyframe encoding ElasticFusion uses).  LoopClosure (omnidata_b200/loop.py) uses it to find loops beyond
the pose radius and to relocalise lost frames.

    from omnidata_b200.places import FernDatabase
    db = FernDatabase((h, w), ferns=500, seed=0)
    db.add(db.encode(metres, rgb))                     # one code per keyframe
    index, distance = db.query(db.encode(pred, rgb)[0], k=3)
    db.dissimilarity(distance)                         # distance / ferns, in [0, 1]

A code is computed from a 60 x 80 thumbnail of the frame: each cell's mean depth, R, G and B over its usable samples
(finite, depth also > 0).  Each channel is normalised per frame by its lower median m and the lower median s of
|v - m| over the cells, so a depth map in metres and a relative prediction of the same view (any positive scale and
shift) give the same code, and so does an image under any gain and bias per colour channel (the exposure and white
balance changes of real video).  Fern f looks at one cell p_f and sets bit c of its 4-bit code when (v_c - m_c) >
theta_f,c s_c.  The table (cells uniform over the 4800, thresholds uniform in [-1, 1]) is drawn once from
numpy.random.default_rng(seed); these ranges and the default of 500 ferns are untuned.  The distance of two codes is
the number of ferns whose codes differ, an integer, so lookups are exact: the k nearest entries, ties to the lower
index, padded with -1.

depth fp32 [B,H,W] or [H,W] (metres or a relative prediction; NaN and <= 0: no depth), rgb fp32 [B,3,H,W] or [3,H,W];
H >= 60 and W >= 80.  Codes are uint8 [B,F] on the device.  Definition: DESIGN.md §3 "Place recognition and
relocalisation" and include/omnidata_b200.h; oracle/places_oracle.py restates it in float64.  Bit-reproducible; after
the first call at a shape `encode` and `query` neither synchronise nor allocate beyond the outputs they keep, so they
can be captured in a CUDA graph.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch

from . import _capi, ops
from .losses import _StepBuffers
from .track import _value_error

GRID = _capi.FERN_GRID
CELLS = GRID[0] * GRID[1]


def fern_table(ferns: int, seed: int) -> Tuple[np.ndarray, np.ndarray]:
    """(cells int32 [F] uniform over the 4800 thumbnail cells, thresholds float64 [F,4] uniform in [-1, 1]), drawn in
    that order from numpy.random.default_rng(seed)."""
    rng = np.random.default_rng(seed)
    cells = rng.integers(0, CELLS, size=ferns).astype(np.int32)
    thresholds = rng.uniform(-1.0, 1.0, size=(ferns, 4))
    return cells, thresholds


class FernDatabase(_StepBuffers):
    """Fern codes of frames of one size and a growing database of them (module docstring)."""

    def __init__(self, size: Tuple[int, int], ferns: int = 500, seed: int = 0, device=None):
        h, w = (int(v) for v in size)
        _value_error(ops.check_fern_frames, "FernDatabase", 1, h, w)
        if isinstance(ferns, bool) or not isinstance(ferns, int) or not 1 <= ferns <= _capi.FERN_MAX_FERNS:
            raise ValueError(f"FernDatabase: ferns must be an integer in [1, {_capi.FERN_MAX_FERNS}], got {ferns!r}")
        if isinstance(seed, bool) or not isinstance(seed, int) or seed < 0:
            raise ValueError(f"FernDatabase: seed must be an integer >= 0, got {seed!r}")
        self.size, self.ferns, self.seed = (h, w), ferns, seed
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        cells, thresholds = fern_table(ferns, seed)
        self.cells = torch.from_numpy(cells).to(self.device)
        self.thresholds = torch.from_numpy(thresholds).to(self.device)
        self._codes = torch.zeros((16, ferns), dtype=torch.uint8, device=self.device)   # [capacity,F]
        self.count = 0
        self._bufs = {}

    @property
    def codes(self) -> torch.Tensor:
        """The stored codes, uint8 [count,F] (a view of the database's buffer)."""
        return self._codes[:self.count]

    @torch.no_grad()
    def encode(self, depth: torch.Tensor, rgb: torch.Tensor) -> torch.Tensor:
        """uint8 [B,F] codes on the device; kept for the next call with B frames, which overwrites them."""
        name = "FernDatabase.encode"
        h, w = self.size
        if depth.dim() == 2:
            depth = depth.unsqueeze(0)
        if rgb.dim() == 3:
            rgb = rgb.unsqueeze(0)
        if depth.dim() != 3 or tuple(depth.shape[1:]) != (h, w):
            raise ValueError(f"{name}: depth must be [B, {h}, {w}] or [{h}, {w}], got {tuple(depth.shape)}")
        b = depth.shape[0]
        if tuple(rgb.shape) != (b, 3, h, w):
            raise ValueError(f"{name}: rgb must be [{b}, 3, {h}, {w}] (or [3, {h}, {w}] with one frame), got "
                             f"{tuple(rgb.shape)}")
        for what, t in (("depth", depth), ("rgb", rgb)):
            if t.dtype != torch.float32 or t.device != self.device or not t.is_contiguous():
                raise ValueError(f"{name}: {what} must be contiguous fp32 on {self.device}, got {t.dtype} on "
                                 f"{t.device}")
        _value_error(ops.check_fern_frames, name, b, h, w)
        ws = self._buf(f"encode_ws{b}", (-(-ops.fern_encode_workspace_bytes(b) // 8),), torch.float64, self.device)
        codes = self._buf(f"codes{b}", (b, self.ferns), torch.uint8, self.device)
        with torch.cuda.device(self.device):
            _value_error(ops.fern_encode, depth, rgb, self.cells, self.thresholds, codes, ws)
        return codes

    @torch.no_grad()
    def add(self, codes: torch.Tensor):
        """Appends codes uint8 [B,F] or [F] (on the device) as entries count .. count + B - 1; the buffer grows by
        doubling."""
        if codes.dim() == 1:
            codes = codes.unsqueeze(0)
        if codes.dim() != 2 or codes.shape[1] != self.ferns or codes.dtype != torch.uint8 or \
                codes.device != self.device:
            raise ValueError(f"FernDatabase.add: codes must be uint8 [B, {self.ferns}] or [{self.ferns}] on "
                             f"{self.device}, got {codes.dtype} {tuple(codes.shape)} on {codes.device}")
        need = self.count + codes.shape[0]
        if need > self._codes.shape[0]:
            cap = self._codes.shape[0]
            while cap < need:
                cap *= 2
            grown = torch.zeros((cap, self.ferns), dtype=torch.uint8, device=self.device)
            grown[:self.count].copy_(self._codes[:self.count])
            self._codes = grown
        self._codes[self.count:need].copy_(codes)
        self.count = need

    @torch.no_grad()
    def query(self, code: torch.Tensor, k: int, limit: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """(indices int32 [k], distances int32 [k]) on the device: the k entries i < limit (default: every entry)
        nearest to code uint8 [F], in (distance, index) order, padded with -1.  Kept for the next call with this k,
        which overwrites them."""
        name = "FernDatabase.query"
        limit = self.count if limit is None else limit
        if isinstance(limit, bool) or not isinstance(limit, (int, np.integer)) or not 0 <= limit <= self.count:
            raise ValueError(f"{name}: limit must be an integer in [0, {self.count}], got {limit!r}")
        if code.dim() == 2 and code.shape[0] == 1:
            code = code[0]
        if tuple(code.shape) != (self.ferns,) or code.dtype != torch.uint8 or code.device != self.device:
            raise ValueError(f"{name}: code must be uint8 [{self.ferns}] on {self.device}, got {code.dtype} "
                             f"{tuple(code.shape)} on {code.device}")
        if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= _capi.FERN_MAX_K:
            raise ValueError(f"{name}: k must be an integer in [1, {_capi.FERN_MAX_K}], got {k!r}")
        n_db = self._codes.shape[0]
        ws = self._buf("query_ws", (-(-ops.fern_query_workspace_bytes(n_db) // 8),), torch.float64, self.device)
        index = self._buf(f"index{k}", (k,), torch.int32, self.device)
        distance = self._buf(f"distance{k}", (k,), torch.int32, self.device)
        with torch.cuda.device(self.device):
            _value_error(ops.fern_query, self._codes, code.contiguous(), int(limit), int(k), index, distance, ws)
        return index, distance

    def dissimilarity(self, distance):
        """distance / ferns: the fraction of ferns whose codes differ (tensor or number)."""
        return distance / self.ferns
