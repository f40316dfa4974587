"""Optimizer step of the depth train step (train_depth.py:381-383 `torch.optim.Adam(self.parameters(), lr)`,
:425 `gradient_clip_val=10`) on flat fp32 buffers: two kernel launches per step, no host synchronisation.

    opt = FlatAdam(flat_params, lr=1e-5)           # flat_params: one fp32 CUDA tensor holding every parameter
    norm = opt.step(flat_grads, max_norm=10.0)     # clip_grad_norm_ + Adam update; returns the norm tensor

`flatten_parameters(module)` re-points a module's parameters into such a buffer (views), which is also the
layout the bucketed gradient all-reduce of `train.DepthTrainStep` wants (train.TrainEngine writes the network's
gradients straight into the matching flat gradient buffer).  The step is checked against torch.optim.Adam in the tests.

    opt = FlatAdam(flat_params, lr=1e-5, segments=[(0, 4096), (8192, 9000)])

restricts the norm and the update to those [start, end) ranges of the flat buffers (the trainable parameters of a
partly frozen model): elements outside them, and their moments, are never read or written.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

from . import _capi
from ._capi import check, lib


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def flatten_parameters(module: torch.nn.Module) -> torch.Tensor:
    """One contiguous fp32 buffer for all parameters of `module` (16-byte aligned slices); every parameter
    becomes a view into it.  Returns the buffer."""
    params = [p for p in module.parameters()]
    sizes = [(p.numel() + 3) // 4 * 4 for p in params]
    flat = torch.zeros(sum(sizes), device=params[0].device, dtype=torch.float32)
    off = 0
    for p, n in zip(params, sizes):
        flat[off:off + p.numel()].copy_(p.data.reshape(-1).float())
        p.data = flat[off:off + p.numel()].view_as(p.data)
        off += n
    return flat


MAX_SEGMENTS = 1024     # optim.cu kMaxSegments


def check_segments(segments: Sequence[Tuple[int, int]], n: int) -> int:
    """Validates a segment list for the _segments kernels: ascending, disjoint, non-empty [start, end) ranges inside
    [0, n), every start a multiple of 4 and every length but the last a multiple of 4.  -> total element count."""
    if not 1 <= len(segments) <= MAX_SEGMENTS:
        raise ValueError(f"FlatAdam: 1..{MAX_SEGMENTS} segments required, got {len(segments)}")
    prev, total = 0, 0
    for k, (s, e) in enumerate(segments):
        if not prev <= s < e <= n or s % 4 or (k + 1 < len(segments) and (e - s) % 4):
            raise ValueError(f"FlatAdam: bad segment {k} [{s}, {e}) (ascending, disjoint, inside [0, {n}), starts and "
                             "all lengths but the last multiples of 4)")
        prev, total = e, total + e - s
    return total


class FlatAdam:
    def __init__(self, flat_params: torch.Tensor, lr: float = 1e-5, betas=(0.9, 0.999), eps: float = 1e-8,
                 segments: Optional[Sequence[Tuple[int, int]]] = None):
        if not flat_params.is_cuda or flat_params.dtype != torch.float32 or flat_params.dim() != 1:
            raise _capi.OdbError("FlatAdam: a flat fp32 CUDA tensor is required (no CPU path)")
        self.params = flat_params
        # optional [start, end) ranges the step is restricted to: a device table read by the _segments kernels
        self.segments = None if segments is None else [(int(s), int(e)) for s, e in segments]
        self._seg_table, self._seg_total = None, 0
        if self.segments is not None:
            self._seg_total = check_segments(self.segments, flat_params.numel())
            self._seg_table = torch.tensor(self.segments, dtype=torch.int64).to(flat_params.device)
        self.lr, self.betas, self.eps = lr, betas, eps
        self.exp_avg = torch.zeros_like(flat_params)
        self.exp_avg_sq = torch.zeros_like(flat_params)
        self.step_count = 0
        self._ws = torch.zeros(int(lib().odb_grad_norm_workspace_bytes()), device=flat_params.device, dtype=torch.uint8)
        self._clip = torch.zeros(2, device=flat_params.device, dtype=torch.float32)
        # CUDA-graph replay: the step-dependent scalars live in device memory and are refreshed before each replay
        self._scalars_dev = torch.zeros(2, device=flat_params.device, dtype=torch.float32)

    def stage_step_scalars(self, host2: torch.Tensor) -> None:
        """Advance the step counter and copy this step's (lr / (1 - beta1^t), sqrt(1 - beta2^t)) through the pinned
        fp32[2] tensor `host2` (which must stay untouched until the copy has run) to the device buffer that
        `step(..., scalars_on_device=True)` reads; call once before each replay of a captured step."""
        self.step_count += 1
        check(lib().odb_adam_step_scalars(self.lr, self.betas[0], self.betas[1], self.step_count, host2.data_ptr()),
              "odb_adam_step_scalars")
        self._scalars_dev.copy_(host2, non_blocking=True)

    @_capi.on_tensor_device
    def step(self, flat_grads: torch.Tensor, max_norm: Optional[float] = 10.0,
             scalars_on_device: bool = False) -> Optional[torch.Tensor]:
        """scalars_on_device: the launch reads the step scalars staged by `stage_step_scalars` (the form a CUDA graph
        captures); otherwise they are computed here from the step counter."""
        g = flat_grads
        if not g.is_cuda or g.dtype != torch.float32 or g.shape != self.params.shape or not g.is_contiguous():
            raise _capi.OdbError("FlatAdam.step: gradients must match the flat parameter buffer")
        if not scalars_on_device:
            self.step_count += 1
        clip_ptr = None
        scal = self._scalars_dev.data_ptr() if scalars_on_device else None
        if self._seg_table is None:
            if max_norm is not None:
                check(lib().odb_clip_grad_norm(g.data_ptr(), g.numel(), float(max_norm), self._ws.data_ptr(),
                                               self._clip.data_ptr(), _stream()), "odb_clip_grad_norm")
                clip_ptr = self._clip.data_ptr()
            check(lib().odb_adam_step(self.params.data_ptr(), g.data_ptr(), self.exp_avg.data_ptr(),
                                      self.exp_avg_sq.data_ptr(), g.numel(), clip_ptr, self.lr, self.betas[0],
                                      self.betas[1], self.eps, max(self.step_count, 1), scal, _stream()), "odb_adam_step")
        else:
            tab, nseg, total = self._seg_table.data_ptr(), len(self.segments), self._seg_total
            if max_norm is not None:
                check(lib().odb_clip_grad_norm_segments(g.data_ptr(), tab, nseg, total, float(max_norm), self._ws.data_ptr(),
                                                        self._clip.data_ptr(), _stream()), "odb_clip_grad_norm_segments")
                clip_ptr = self._clip.data_ptr()
            check(lib().odb_adam_step_segments(self.params.data_ptr(), g.data_ptr(), self.exp_avg.data_ptr(),
                                               self.exp_avg_sq.data_ptr(), tab, nseg, total, clip_ptr, self.lr,
                                               self.betas[0], self.betas[1], self.eps, max(self.step_count, 1), scal,
                                               _stream()), "odb_adam_step_segments")
        return self._clip[0] if max_norm is not None else None
