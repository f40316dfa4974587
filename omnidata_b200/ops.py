"""Thin torch-tensor front end of the C-ABI kernels (pointers + sizes only cross the boundary).

Every function enqueues on torch's current CUDA stream and returns immediately.  Activations are
channels-last bf16 tensors ([B, H, W, C] or [rows, C]); strides are taken from the tensors, so
sliced / strided views (parity planes, token windows) are passed without copies.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _capi
from ._capi import ACT_GELU, ACT_NONE, ACT_RELU, DTYPE_BF16, DTYPE_E4M3, DTYPE_F32, ConvGemmDesc, View, check, lib

__all__ = [
    "ACT_NONE", "ACT_RELU", "ACT_GELU", "conv_gemm", "linear", "conv1x1", "conv3x3", "conv3x3_s2",
    "linear_fp8", "layernorm_e4m3", "rowquant_e4m3",
    "layernorm", "attention", "groupnorm_stats", "groupnorm_apply", "stem_gn_relu_maxpool",
    "stem_im2col", "patchify", "upsample2x_add", "write_cls_row", "readout_cls_bias", "pack_conv_weight",
    "cast_f32_bf16", "head_tail_f32", "tile_gather", "tile_overlap_moments", "tile_align_solve", "tile_blend",
    "resize_bilinear", "tile_anchor_moments", "tile_align_solve_anchored",
    "metrics_workspace_bytes", "depth_metrics_update", "normal_metrics_update", "normal_metrics_median",
    "ensemble_gram_workspace_bytes", "ensemble_gram", "ensemble_align_solve", "ensemble_merge_depth",
    "ensemble_merge_normal", "guided_workspace_bytes", "guided_coefficients", "guided_apply",
    "boundary_workspace_bytes", "depth_edges", "edge_hysteresis", "edge_distance2", "boundary_metrics_update",
    "sparse_align_workspace_bytes", "sparse_align_fit", "sparse_align_apply",
    "fusion_workspace_bytes", "depth_normals_workspace_bytes", "depth_normal_fusion", "depth_normals",
    "tsdf_mesh_workspace_bytes", "tsdf_integrate", "tsdf_raycast", "tsdf_raycast_color", "tsdf_mesh_count", "tsdf_mesh_emit",
]

_DTYPES = {torch.bfloat16: DTYPE_BF16, torch.float32: DTYPE_F32}


def _dt(t: torch.Tensor, name: str = "tensor") -> int:
    """odb_dtype of an activation tensor (bf16 in production, fp32 for the residual stream / correctness mode)."""
    if not t.is_cuda:
        raise _capi.OdbError(f"{name}: tensor must live on a CUDA device (no CPU path exists)")
    try:
        return _DTYPES[t.dtype]
    except KeyError:
        raise _capi.OdbError(f"{name}: expected bfloat16 or float32 storage, got {t.dtype}") from None


def _same_device(*ts):
    dev = None
    for t in ts:
        if t is None:
            continue
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise _capi.OdbError(f"tensors live on different devices ({dev} and {t.device})")
    return dev


class LaunchTimer:
    """Optional per-launch device timing (bench.py roofline pass): every C-ABI call made while the
    timer is active is bracketed by CUDA events on torch's current stream — the stream the kernel is
    launched on.  Not used on the normal path."""

    active: "Optional[LaunchTimer]" = None

    def __init__(self):
        self.records = []          # (name, info dict, start event, end event)

    def __enter__(self):
        LaunchTimer.active = self
        return self

    def __exit__(self, *exc):
        LaunchTimer.active = None

    def results(self):
        torch.cuda.synchronize()
        return [(n, i, s.elapsed_time(e)) for n, i, s, e in self.records]


def _call(name: str, info: dict, fn, dev, *args):
    """Enqueue one C-ABI call on the current stream of `dev` — the device the tensors live on, made current for the
    duration of the call (kernel attributes, SM counts and TMA descriptors are per device).  The stream is appended
    as the last argument."""
    if dev is None or dev.type != "cuda":
        raise _capi.OdbError(f"{name}: tensors must live on a CUDA device (no CPU path exists)")
    if dev.index is not None and dev.index != torch.cuda.current_device():
        with torch.cuda.device(dev):
            return _call(name, info, fn, dev, *args)
    stream = torch.cuda.current_stream(dev).cuda_stream
    t = LaunchTimer.active
    if t is None:
        check(fn(*args, stream), name)
        return
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    check(fn(*args, stream), name)
    e.record()
    t.records.append((name, info, s, e))


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise _capi.OdbError(f"{name}: tensor must live on a CUDA device (no CPU path exists)")
    if t.dtype != dtype:
        raise _capi.OdbError(f"{name}: expected {dtype}, got {t.dtype}")


def _view4(t: torch.Tensor, name: str, dtype=torch.bfloat16) -> View:
    """[B,H,W,C] (or [rows,C] -> B=H=1) tensor with unit channel stride -> odb_view."""
    _need(t, dtype, name)
    if t.dim() == 2:
        t = t.unsqueeze(0).unsqueeze(0)
    if t.dim() != 4 or t.stride(3) != 1:
        raise _capi.OdbError(f"{name}: need a channels-last [B,H,W,C] view with unit channel stride")
    b, h, w, c = t.shape
    return View(t.data_ptr(), c, w, h, b, t.stride(2), t.stride(1), t.stride(0))


def conv_gemm(views: Sequence[torch.Tensor], taps: Sequence[Tuple[int, int, int]], weight: torch.Tensor,
              out: Optional[torch.Tensor], *, bias: Optional[torch.Tensor] = None,
              bias_per_image: bool = False, residual: Optional[torch.Tensor] = None, act: int = ACT_NONE,
              out2: Optional[torch.Tensor] = None, tile: Optional[Tuple[int, int]] = None, block_n: int = 0,
              cta_pair: int = 0, halo: int = 0, epilogue: int = 0, gn_stats: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
              gn_groups: int = 32, gn_eps: float = 1e-5, out2_act: int = ACT_RELU,
              head: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor, bool]] = None,
              out_extent: Optional[Tuple[int, int, int]] = None) -> None:
    """taps: (view index, dx, dy).  head = (w[head_c,32] f32, b[head_c] f32, out[B,head_c,H,W] f32, relu).
    out2_act: activation of the out2 copy (ACT_RELU, or ACT_GELU: `out` keeps the pre-activation)."""
    d = ConvGemmDesc()
    dev = _same_device(*views, weight, out, out2, bias, residual)
    in_t = views[0].dtype
    d.in_dtype = _dt(views[0], "view0")
    d.num_views = len(views)
    for i, v in enumerate(views):
        d.views[i] = _view4(v, f"view{i}", in_t)
    d.num_taps = len(taps)
    for i, (vi, dx, dy) in enumerate(taps):
        d.tap_view[i], d.tap_dx[i], d.tap_dy[i] = vi, dx, dy
    _need(weight, in_t, "weight")
    if not weight.is_contiguous():
        raise _capi.OdbError("weight must be contiguous [n][taps*C]")
    d.weight = weight.data_ptr()
    d.n = weight.shape[0]
    out_t = in_t if out is None else out.dtype
    d.out_dtype = _DTYPES.get(out_t, -1)
    if out is not None:
        d.out = _view4(out, "out", out_t)
    if out2 is not None:
        d.out2 = _view4(out2, "out2", out_t)
        d.out2_act = out2_act
    if bias is not None:
        _need(bias, torch.float32, "bias")
        d.bias = bias.data_ptr()
        d.bias_sb = d.n if bias_per_image else 0
    if residual is not None:
        r = residual
        if r.dim() == 3:  # [rows_per_image, C] broadcast over batch is passed as [1,H,W,C] with sb=0
            r = r.unsqueeze(0)
        rv = _view4(r, "residual", out_t)
        if residual.dim() == 4 and residual.shape[0] == 1 and out is not None and out.dim() == 4 and out.shape[0] > 1:
            rv.sb = 0
        d.residual = rv
    d.act = act
    if tile is not None:
        d.tile_w, d.tile_h = tile
    d.block_n = block_n
    d.cta_pair = cta_pair
    d.halo = halo
    d.epilogue = epilogue
    if head is not None:
        hw, hb, hout, hrelu = head
        _need(hw, torch.float32, "head_w"); _need(hb, torch.float32, "head_b"); _need(hout, torch.float32, "head_out")
        d.head_w, d.head_b, d.head_out = hw.data_ptr(), hb.data_ptr(), hout.data_ptr()
        d.head_c = hw.shape[0]
        d.head_relu = 1 if hrelu else 0
        b, _, h, w = hout.shape
        d.out = View(None, 32, w, h, b, 0, 0, 0)
    rows = d.out.w * d.out.h * d.out.b
    info = {"m": rows, "n": d.n, "k": d.num_taps * d.views[0].c, "taps": d.num_taps, "w": d.out.w, "h": d.out.h,
            "f32": d.in_dtype == DTYPE_F32}
    if gn_stats is None:
        _call("odb_conv_gemm", info, lib().odb_conv_gemm, dev, C.byref(d))
        return
    # fused GroupNorm statistics: the epilogue writes per-warp partial sums, a tiny kernel reduces them
    partial, stats = gn_stats
    _need(partial, torch.float32, "gn partial"); _need(stats, torch.float32, "gn stats")
    plan = (C.c_int32 * 4)()
    check(lib().odb_conv_gemm_plan(C.byref(d), plan), "odb_conv_gemm_plan")
    part_rows = plan[0] * plan[1] * 4
    if partial.numel() < d.out.b * part_rows * gn_groups * 2:
        raise _capi.OdbError("conv_gemm: gn partial buffer too small")
    d.gn_partial = partial.data_ptr()
    d.gn_groups = gn_groups
    _call("odb_conv_gemm", info, lib().odb_conv_gemm, dev, C.byref(d))
    count = float(d.out.w) * float(d.out.h) * (d.n // gn_groups)
    _call("odb_groupnorm_finalize", {}, lib().odb_groupnorm_finalize, dev, partial.data_ptr(), stats.data_ptr(),
          d.out.b, part_rows, gn_groups, count, gn_eps)


E4M3 = torch.float8_e4m3fn


def _rows_operand(t: torch.Tensor, dtype, name: str, cols: Optional[int] = None) -> Tuple[int, int]:
    """(rows, cols) of a contiguous 2-D [rows, cols] operand of `dtype`, 16-byte aligned; raises otherwise."""
    _need(t, dtype, name)
    if t.dim() != 2 or not t.is_contiguous() or t.data_ptr() % 16 != 0:
        raise _capi.OdbError(f"{name}: need a contiguous, 16-byte aligned [rows, cols] tensor, got {tuple(t.shape)}")
    if cols is not None and t.shape[1] != cols:
        raise _capi.OdbError(f"{name}: expected {cols} columns, got {t.shape[1]}")
    return t.shape[0], t.shape[1]


def _row_scale(s: torch.Tensor, rows: int, name: str = "row_scale"):
    _need(s, torch.float32, name)
    if s.dim() != 1 or s.shape[0] != rows or not s.is_contiguous():
        raise _capi.OdbError(f"{name}: need a contiguous fp32 [{rows}] tensor, got {tuple(s.shape)}")


def linear_fp8(x, row_scale, weight, col_scale, out, *, bias, residual=None, act: int = ACT_NONE,
               block_n: int = 0) -> None:
    """The fp8 mode's linear layer: out = epilogue((x @ weight^T) * (row_scale[r] * col_scale[c]) + bias[c]).
    x e4m3 [rows, K] with row_scale fp32 [rows]; weight e4m3 [N, K] with col_scale fp32 [N]; bias fp32 [N].
    out bf16 [rows, N] (act ACT_NONE or ACT_GELU), or fp32 [rows, N] = residual (fp32 [rows, N]) + the value."""
    rows, k = _rows_operand(x, E4M3, "x")
    n, _ = _rows_operand(weight, E4M3, "weight", k)
    _row_scale(row_scale, rows)
    _row_scale(col_scale, n, "col_scale")
    _need(bias, torch.float32, "bias")
    if bias.numel() != n or not bias.is_contiguous() or col_scale.data_ptr() % 16 != 0:
        raise _capi.OdbError("linear_fp8: bias [N] contiguous and col_scale 16-byte aligned required")
    f32 = out.dtype == torch.float32
    _rows_operand(out, torch.float32 if f32 else torch.bfloat16, "out", n)
    if out.shape[0] != rows:
        raise _capi.OdbError("linear_fp8: out must have x's rows")
    if f32 != (residual is not None) or (f32 and act != ACT_NONE) or act not in (ACT_NONE, ACT_GELU):
        raise _capi.OdbError("linear_fp8: bf16 out with bias [+ GELU], or fp32 out with an fp32 residual")
    d = ConvGemmDesc()
    d.in_dtype = DTYPE_E4M3
    d.num_views = 1
    d.views[0] = View(x.data_ptr(), k, rows, 1, 1, k, 0, 0)
    d.num_taps = 1
    d.weight = weight.data_ptr()
    d.n = n
    d.out_dtype = DTYPE_F32 if f32 else DTYPE_BF16
    d.out = _view4(out, "out", out.dtype)
    d.bias = bias.data_ptr()
    if residual is not None:
        _rows_operand(residual, torch.float32, "residual", n)
        d.residual = _view4(residual, "residual", torch.float32)
    d.act = act
    d.block_n = block_n
    info = {"m": rows, "n": n, "k": k, "taps": 1, "w": rows, "h": 1, "f32": False, "fp8": True}
    _call("odb_conv_gemm_scaled", info, lib().odb_conv_gemm_scaled, _same_device(x, weight, out, bias, residual),
          C.byref(d), row_scale.data_ptr(), col_scale.data_ptr())


def layernorm_e4m3(x, gamma, beta, out, row_scale, eps: float = 1e-6):
    """LayerNorm of x (fp32 or bf16 [.., cols]) quantised per row to e4m3 `out` with its fp32 row scales."""
    _need(gamma, torch.float32, "gamma"); _need(beta, torch.float32, "beta")
    _need(out, E4M3, "out")
    if not (x.is_contiguous() and out.is_contiguous()) or out.shape != x.shape:
        raise _capi.OdbError("layernorm_e4m3: contiguous x and out of one shape required")
    rows = x.numel() // x.shape[-1]
    _row_scale(row_scale, rows)
    _call("odb_layernorm_e4m3", {"bytes": x.element_size() * x.numel() + out.numel() + 4 * rows},
          lib().odb_layernorm_e4m3, _same_device(x, gamma, beta, out, row_scale), x.data_ptr(), gamma.data_ptr(),
          beta.data_ptr(), out.data_ptr(), row_scale.data_ptr(), rows, x.shape[-1], eps, _dt(x, "x"))


def rowquant_e4m3(x, out, row_scale):
    """Per-row e4m3 quantisation of x bf16 [rows, cols] into out e4m3 [rows, cols] and row_scale fp32 [rows]."""
    rows, cols = _rows_operand(x, torch.bfloat16, "x")
    _rows_operand(out, E4M3, "out", cols)
    if out.shape[0] != rows:
        raise _capi.OdbError("rowquant_e4m3: out must have x's shape")
    _row_scale(row_scale, rows)
    _call("odb_rowquant_e4m3", {"bytes": 3 * x.numel() + 4 * rows, "cols": cols}, lib().odb_rowquant_e4m3,
          _same_device(x, out, row_scale), x.data_ptr(), out.data_ptr(), row_scale.data_ptr(), rows, cols)


TAPS_1 = [(0, 0, 0)]
TAPS_3X3 = [(0, kx - 1, ky - 1) for ky in range(3) for kx in range(3)]


def pack_conv_weight(w: torch.Tensor, dtype=torch.bfloat16) -> torch.Tensor:
    """[N, Cin, kh, kw] (any float dtype) -> `dtype` [N, kh*kw*Cin], tap-major / channel-minor."""
    n = w.shape[0]
    return w.permute(0, 2, 3, 1).reshape(n, -1).to(dtype).contiguous()


def linear(x, weight, out, **kw):
    conv_gemm([x], TAPS_1, weight, out, **kw)


def conv1x1(x, weight, out, **kw):
    conv_gemm([x], TAPS_1, weight, out, **kw)


def conv3x3(x, weight, out, **kw):
    conv_gemm([x], TAPS_3X3, weight, out, **kw)


def _parity_taps(mode: str):
    # input index = 2*o + k - pad_before ; parity plane p, plane coordinate o + d
    taps = []
    for ky in range(3):
        for kx in range(3):
            if mode == "same":      # TF-SAME for even sizes: pad (0,1)
                py, dy = (ky & 1), (1 if ky == 2 else 0)
                px, dx = (kx & 1), (1 if kx == 2 else 0)
            elif mode == "sym1":    # padding=1 both sides
                py, dy = ((ky + 1) & 1), (-1 if ky == 0 else 0)
                px, dx = ((kx + 1) & 1), (-1 if kx == 0 else 0)
            else:
                raise ValueError(mode)
            taps.append((py * 2 + px, dx, dy))
    return taps


def conv3x3_s2(x, weight, out, mode: str, **kw):
    """Stride-2 3x3 conv through four parity-plane views of x (no im2col, no copies)."""
    planes = [x[:, py::2, px::2, :] for py in range(2) for px in range(2)]
    conv_gemm(planes, _parity_taps(mode), weight, out, **kw)


def layernorm(x, gamma, beta, out, eps: float = 1e-6):
    """x bf16 or fp32 (the fp32 residual stream), out bf16 (fp32 only together with an fp32 x)."""
    _need(gamma, torch.float32, "gamma"); _need(beta, torch.float32, "beta")
    if not (x.is_contiguous() and out.is_contiguous()):
        raise _capi.OdbError("layernorm: contiguous tensors required")
    rows = x.numel() // x.shape[-1]
    _call("odb_layernorm", {"bytes": x.element_size() * x.numel() + out.element_size() * out.numel()},
          lib().odb_layernorm, _same_device(x, gamma, beta, out), x.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
          out.data_ptr(), rows, x.shape[-1], eps, _dt(x, "x"), _dt(out, "out"))


def attention(qkv, out, heads: int = 12, scale: float = 0.125, lse=None):
    b, n, c3 = qkv.shape
    if not (qkv.is_contiguous() and out.is_contiguous()) or c3 != 3 * heads * 64:
        raise _capi.OdbError("attention: qkv must be contiguous [B, tokens, 3*heads*64]")
    info = {"flops": 4.0 * b * heads * n * n * 64, "bytes": qkv.element_size() * (qkv.numel() + out.numel())}
    if qkv.dtype == torch.float32:
        _need(out, torch.float32, "out")
        _call("odb_attention_f32", info, lib().odb_attention_f32, _same_device(qkv, out), qkv.data_ptr(), out.data_ptr(),
              b, n, heads, scale)
        return
    _need(qkv, torch.bfloat16, "qkv"); _need(out, torch.bfloat16, "out")
    if lse is not None:
        _need(lse, torch.float32, "lse")
    _call("odb_attention", info, lib().odb_attention, _same_device(qkv, out, lse), qkv.data_ptr(), out.data_ptr(),
          _ptr(lse), b, n, heads, scale)


_GN_SCRATCH = {}


def groupnorm_scratch(device, nbytes: int) -> torch.Tensor:
    """Zero-initialised scratch shared by all GroupNorm statistics launches of one device/stream."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    t = _GN_SCRATCH.get(key)
    if t is None or t.numel() < nbytes:
        t = torch.zeros(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _GN_SCRATCH[key] = t
    return t


def groupnorm_stats(x, stats, groups: int = 32, eps: float = 1e-5, scratch: Optional[torch.Tensor] = None):
    """stats[b, g] = (mean, rstd).  Deterministic; `scratch` must stay zeroed between calls (it does)."""
    _need(stats, torch.float32, "stats")
    b, c = x.shape[0], x.shape[-1]
    hw = x.numel() // (b * c)
    need = int(lib().odb_groupnorm_scratch_bytes(b, hw, c, groups))
    if need < 0:
        raise _capi.OdbError("groupnorm_stats: unsupported shape")
    if scratch is None:
        scratch = groupnorm_scratch(x.device, need)
    _call("odb_groupnorm_stats", {"bytes": x.element_size() * x.numel()}, lib().odb_groupnorm_stats,
          _same_device(x, stats, scratch), x.data_ptr(), stats.data_ptr(), scratch.data_ptr(), scratch.numel(), b, hw, c,
          groups, eps, _dt(x, "x"))


def groupnorm_apply(x, stats, gamma, beta, out, *, relu: bool, res=None, res_stats=None, res_gamma=None,
                    res_beta=None, groups: int = 32):
    b, c = x.shape[0], x.shape[-1]
    hw = x.numel() // (b * c)
    if out.dtype != x.dtype or (res is not None and res.dtype != x.dtype):
        raise _capi.OdbError("groupnorm_apply: x, res and out must share one storage type")
    _call("odb_groupnorm_apply", {"bytes": x.element_size() * x.numel() * (2 + (res is not None))},
          lib().odb_groupnorm_apply, _same_device(x, stats, gamma, beta, res, out),
          x.data_ptr(), stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), _ptr(res), _ptr(res_stats),
          _ptr(res_gamma), _ptr(res_beta), out.data_ptr(), b, hw, c, groups, 1 if relu else 0, _dt(x, "x"))


def stem_gn_relu_maxpool(x, stats, gamma, beta, out, groups: int = 32):
    b, h, w, c = x.shape
    if out.dtype != x.dtype:
        raise _capi.OdbError("stem_gn_relu_maxpool: x and out must share one storage type")
    _call("odb_stem_gn_relu_maxpool", {"bytes": int(1.25 * x.element_size() * x.numel())}, lib().odb_stem_gn_relu_maxpool,
          _same_device(x, stats, gamma, beta, out), x.data_ptr(), stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
          out.data_ptr(), b, h, w, c, groups, _dt(x, "x"))


def stem_im2col(x, cols):
    _need(x, torch.float32, "x")
    b, ch, h, w = x.shape
    if ch != 3 or not x.is_contiguous():
        raise _capi.OdbError("stem_im2col: contiguous [B,3,H,W] fp32 input required")
    _call("odb_stem_im2col", {}, lib().odb_stem_im2col, _same_device(x, cols), x.data_ptr(), cols.data_ptr(), b, h, w,
          cols.shape[-1], _dt(cols, "cols"))


def patchify(x, cols, patch: int = 16):
    """x fp32 [B,3,H,W] -> cols [B*(H/p)*(W/p), 3*p*p] (the im2col of a stride-p, kernel-p convolution)."""
    _need(x, torch.float32, "x")
    b, c, h, w = x.shape
    if c != 3 or not x.is_contiguous() or not cols.is_contiguous() or cols.numel() != b * (h // patch) * (w // patch) * 3 * patch * patch:
        raise _capi.OdbError("patchify: x [B,3,H,W] contiguous, cols [B*gh*gw, 3*p*p]")
    _call("odb_patchify", {"bytes": x.numel() * 4 + cols.numel() * cols.element_size()}, lib().odb_patchify,
          _same_device(x, cols), x.data_ptr(), cols.data_ptr(), b, h, w, patch, _dt(cols, "cols"))


def upsample2x_add(z, out, res=None, out_relu=None):
    b, h, w, c = z.shape
    for t in (out, res, out_relu):
        if t is not None and t.dtype != z.dtype:
            raise _capi.OdbError("upsample2x_add: all tensors must share one storage type")
    n_in = b * h * w * c * z.element_size()
    info = {"bytes": n_in + 4 * n_in * (1 + (res is not None) + (out_relu is not None)), "h": h, "c": c}
    _call("odb_upsample2x_add", info, lib().odb_upsample2x_add, _same_device(z, out, res, out_relu), z.data_ptr(),
          _ptr(res), out.data_ptr(), _ptr(out_relu), b, h, w, c, _dt(z, "z"))


def write_cls_row(tokens, cls, pos0):
    b, n, c = tokens.shape
    _call("odb_write_cls_row", {}, lib().odb_write_cls_row, _same_device(tokens, cls, pos0), tokens.data_ptr(),
          cls.data_ptr(), pos0.data_ptr(), b, n, c, _dt(tokens, "tokens"))


def readout_cls_bias(w, bias, tokens, out):
    b, n, c = tokens.shape
    if w.dtype != tokens.dtype:
        raise _capi.OdbError("readout_cls_bias: w and tokens must share one storage type")
    _call("odb_readout_cls_bias", {}, lib().odb_readout_cls_bias, _same_device(w, bias, tokens, out), w.data_ptr(),
          bias.data_ptr(), tokens.data_ptr(), out.data_ptr(), b, n, c, _dt(tokens, "tokens"))


def cast_f32_bf16(src, dst):
    """dst (bf16) = round(src (fp32)); contiguous, numel a multiple of 8."""
    _need(src, torch.float32, "src"); _need(dst, torch.bfloat16, "dst")
    if not (src.is_contiguous() and dst.is_contiguous()) or src.numel() != dst.numel():
        raise _capi.OdbError("cast_f32_bf16: contiguous tensors of equal size required")
    _call("odb_cast_f32_bf16", {"bytes": 6 * src.numel()}, lib().odb_cast_f32_bf16, _same_device(src, dst),
          src.data_ptr(), dst.data_ptr(), src.numel())


def head_tail_f32(x, w, bias, out, relu: bool, pre=None):
    """fp32 correctness mode: out[b,k,y,x] = relu?(bias[k] + sum_j w[k,j] x[b,y,x,j]), x fp32 [B,H,W,32]."""
    for t_, n_ in ((x, "x"), (w, "w"), (bias, "bias"), (out, "out")):
        _need(t_, torch.float32, n_)
    b, h, wd, c = x.shape
    if c != 32 or not x.is_contiguous() or not out.is_contiguous():
        raise _capi.OdbError("head_tail_f32: x must be contiguous [B,H,W,32]")
    _call("odb_head_tail_f32", {}, lib().odb_head_tail_f32, _same_device(x, w, bias, out, pre), x.data_ptr(),
          w.data_ptr(), bias.data_ptr(), out.data_ptr(), _ptr(pre), b, h, wd, w.shape[0], 1 if relu else 0)


def _check_planes(name: str, *sizes: int, what: str = "batch and image size"):
    """OdbError unless every size (images as a grid dimension, plane height and width) lies in [1, 65535]."""
    if not all(1 <= s <= 65535 for s in sizes):
        raise _capi.OdbError(f"{name}: {what} must lie in [1, 65535], got {'x'.join(str(s) for s in sizes)}")


def _check_workspace(name: str, ws: torch.Tensor, nbytes: int):
    _need(ws, torch.float64, "workspace")
    if ws.numel() * 8 < nbytes or not ws.is_contiguous():
        raise _capi.OdbError(f"{name}: workspace needs {nbytes} contiguous bytes")


# ---------------------------------------------------------------- tiled inference merge (csrc/tiled.cu)
def _tile_shapes(name, b, h, w, tile, overlap):
    from .tiled import tile_grid
    _check_planes(name, b, h, w)
    th, tw = tile
    if th < 32 or tw < 32 or th % 32 or tw % 32 or overlap < 0 or 2 * overlap >= min(th, tw):
        raise _capi.OdbError(f"{name}: tile {th}x{tw} (multiples of 32) with 0 <= 2 overlap < min(tile), got {overlap}")
    oy, ox = tile_grid(h, w, tile, overlap)
    if len(oy) * len(ox) > _capi.TILE_MAX_TILES:
        raise _capi.OdbError(f"{name}: {len(oy)} x {len(ox)} tiles, at most {_capi.TILE_MAX_TILES} per image")
    return len(oy), len(ox)


def _need_shape(t, shape, dtype, name):
    _need(t, dtype, name)
    if tuple(t.shape) != tuple(shape) or not t.is_contiguous():
        raise _capi.OdbError(f"{name}: expected a contiguous {dtype} tensor {tuple(shape)}, got {tuple(t.shape)}")


def tile_gather(x, tiles, tile: Tuple[int, int], overlap: int):
    """tiles fp32 [B*T, 3, th, tw] = the tiles of x fp32 [B, 3, H, W], edge-replicated where x is smaller."""
    _need(x, torch.float32, "x")
    if x.dim() != 4 or x.shape[1] != 3 or not x.is_contiguous():
        raise _capi.OdbError("tile_gather: x must be a contiguous fp32 [B,3,H,W] tensor")
    b, _, h, w = x.shape
    ny, nx = _tile_shapes("tile_gather", b, h, w, tile, overlap)
    _need_shape(tiles, (b * ny * nx, 3, tile[0], tile[1]), torch.float32, "tiles")
    if tiles.data_ptr() % 16:
        raise _capi.OdbError("tile_gather: tiles must be 16-byte aligned")
    _call("odb_tile_gather", {"bytes": 8 * tiles.numel()}, lib().odb_tile_gather, _same_device(x, tiles), x.data_ptr(),
          b, h, w, tile[0], tile[1], overlap, tiles.data_ptr())


def tile_pairs(ny: int, nx: int) -> int:
    return ny * (nx - 1) + (ny - 1) * nx


def tile_overlap_moments(pred, moments, image_hw: Tuple[int, int], tile: Tuple[int, int], overlap: int):
    """moments fp64 [B, pairs, 6] = (n, Sa, Sb, Saa, Sbb, Sab) over each neighbour pair's overlap; pred fp32
    [B*T, th, tw] (a depth model's tile predictions)."""
    h, w = image_hw
    b = moments.shape[0] if moments.dim() == 3 else 0
    ny, nx = _tile_shapes("tile_overlap_moments", b, h, w, tile, overlap)
    _need_shape(pred, (b * ny * nx, tile[0], tile[1]), torch.float32, "pred")
    _need_shape(moments, (b, tile_pairs(ny, nx), 6), torch.float64, "moments")
    _call("odb_tile_overlap_moments", {"bytes": 4 * pred.numel()}, lib().odb_tile_overlap_moments,
          _same_device(pred, moments), pred.data_ptr(), b, h, w, tile[0], tile[1], overlap, moments.data_ptr())


def _align_solve_args(name, moments, scale_shift, grid: Tuple[int, int]):
    ny, nx = grid
    b = scale_shift.shape[0] if scale_shift.dim() == 3 else 0
    if ny < 1 or nx < 1 or ny * nx > _capi.TILE_MAX_TILES:
        raise _capi.OdbError(f"{name}: grid {ny}x{nx}, at most {_capi.TILE_MAX_TILES} tiles")
    _check_planes(name, b, what="batch")
    _need_shape(scale_shift, (b, ny * nx, 2), torch.float64, "scale_shift")
    if moments is not None:
        _need_shape(moments, (b, tile_pairs(ny, nx), 6), torch.float64, "moments")
    elif ny * nx > 1:
        raise _capi.OdbError(f"{name}: moments are required for more than one tile")
    nbytes = int(lib().odb_tile_align_workspace_bytes(b, ny, nx))
    ws = torch.empty(nbytes, device=scale_shift.device, dtype=torch.uint8) if nbytes > 0 else None
    return b, ws


def tile_align_solve(moments, scale_shift, grid: Tuple[int, int]):
    """scale_shift fp64 [B, T, 2] = per-tile (s, t) of the alignment least squares (csrc/tiled.cu) for a ny x nx grid."""
    b, ws = _align_solve_args("tile_align_solve", moments, scale_shift, grid)
    _call("odb_tile_align_solve", {}, lib().odb_tile_align_solve, _same_device(moments, scale_shift, ws),
          _ptr(moments), b, grid[0], grid[1], _ptr(ws), scale_shift.data_ptr())


def tile_anchor_moments(pred, anchor, moments, tile: Tuple[int, int], overlap: int):
    """moments fp64 [B, T, 5] = (n, Sa, Saa, Sg, Sag) over each tile's pixels inside the image; pred fp32 [B*T, th, tw]
    (a depth model's tile predictions), anchor fp32 [B, H, W] (the whole-image prediction at the image's size)."""
    _need(anchor, torch.float32, "anchor")
    if anchor.dim() != 3 or not anchor.is_contiguous():
        raise _capi.OdbError("tile_anchor_moments: anchor must be a contiguous fp32 [B,H,W] tensor")
    b, h, w = anchor.shape
    ny, nx = _tile_shapes("tile_anchor_moments", b, h, w, tile, overlap)
    _need_shape(pred, (b * ny * nx, tile[0], tile[1]), torch.float32, "pred")
    _need_shape(moments, (b, ny * nx, 5), torch.float64, "moments")
    _call("odb_tile_anchor_moments", {"bytes": 4 * (pred.numel() + anchor.numel())}, lib().odb_tile_anchor_moments,
          _same_device(pred, anchor, moments), pred.data_ptr(), anchor.data_ptr(), b, h, w, tile[0], tile[1], overlap,
          moments.data_ptr())


def tile_align_solve_anchored(moments, anchor_moments, scale_shift, grid: Tuple[int, int]):
    """scale_shift fp64 [B, T, 2] = per-tile (s, t) of the alignment least squares with every tile anchored to a
    whole-image prediction (anchor_moments fp64 [B, T, 5] from tile_anchor_moments) instead of the ridge to (1, 0)."""
    b, ws = _align_solve_args("tile_align_solve_anchored", moments, scale_shift, grid)
    _need_shape(anchor_moments, (b, grid[0] * grid[1], 5), torch.float64, "anchor_moments")
    _call("odb_tile_align_solve_anchored", {}, lib().odb_tile_align_solve_anchored,
          _same_device(moments, anchor_moments, scale_shift, ws), _ptr(moments), anchor_moments.data_ptr(), b,
          grid[0], grid[1], _ptr(ws), scale_shift.data_ptr())


def resize_bilinear(x, out):
    """out fp32 [..., oh, ow] = F.interpolate(x, (oh, ow), mode="bilinear", align_corners=False, antialias=True) of x
    fp32 [..., ih, iw] (the same leading dimensions), two passes with cached per-axis tables
    (imageproc.resample_tables)."""
    from .imageproc import resample_tables
    _need(x, torch.float32, "x")
    _need(out, torch.float32, "out")
    if x.dim() < 2 or out.dim() != x.dim() or x.shape[:-2] != out.shape[:-2] or not x.is_contiguous() \
            or not out.is_contiguous():
        raise _capi.OdbError(f"resize_bilinear: contiguous fp32 [..., h, w] tensors with the same leading dimensions "
                             f"expected, got {tuple(x.shape)} -> {tuple(out.shape)}")
    (ih, iw), (oh, ow) = x.shape[-2:], out.shape[-2:]
    planes = x.numel() // (ih * iw) if x.numel() else 0
    if not 1 <= planes <= 65535 or min(ih, iw, oh, ow) < 1 or max(ih, iw, oh, ow) > 65535:
        raise _capi.OdbError(f"resize_bilinear: planes and sizes must lie in [1, 65535], got {planes} planes "
                             f"{ih}x{iw} -> {oh}x{ow}")
    dev = _same_device(x, out)
    bh, wh, kh = resample_tables(iw, ow, dev)
    bv, wv, kv = resample_tables(ih, oh, dev)
    tmp = torch.empty(planes * ih * ow, device=dev, dtype=torch.float32)
    _call("odb_resize_bilinear_f32", {"bytes": 4 * (x.numel() + 2 * tmp.numel() + out.numel())},
          lib().odb_resize_bilinear_f32, dev, x.data_ptr(), planes, ih, iw, oh, ow, bh.data_ptr(), wh.data_ptr(), kh,
          bv.data_ptr(), wv.data_ptr(), kv, tmp.data_ptr(), out.data_ptr())


def tile_blend(pred, scale_shift, out, tile: Tuple[int, int], overlap: int):
    """out fp32 [B, C, H, W] = the weighted blend of the tile predictions pred fp32 [B*T, C, th, tw], each mapped by its
    (s, t) from scale_shift fp64 [B, T, 2] (None: s = 1, t = 0)."""
    if out.dim() != 4:
        raise _capi.OdbError("tile_blend: out must be [B,C,H,W]")
    b, c, h, w = out.shape
    ny, nx = _tile_shapes("tile_blend", b, h, w, tile, overlap)
    _need_shape(out, (b, c, h, w), torch.float32, "out")
    _need_shape(pred, (b * ny * nx, c, tile[0], tile[1]), torch.float32, "pred")
    if scale_shift is not None:
        _need_shape(scale_shift, (b, ny * nx, 2), torch.float64, "scale_shift")
    _call("odb_tile_blend", {}, lib().odb_tile_blend, _same_device(pred, scale_shift, out), pred.data_ptr(),
          _ptr(scale_shift), b, c, h, w, tile[0], tile[1], overlap, out.data_ptr())


# ---------------------------------------------------------------- evaluation metrics (csrc/metrics.cu)
_MASK_KINDS = {torch.uint8: _capi.MASK_U8, torch.bool: _capi.MASK_U8, torch.float32: _capi.MASK_F32}


def metrics_plane_shape(pred: torch.Tensor, channels: int, name: str = "pred") -> Tuple[int, int, int]:
    """(B, H, W) of a metrics input: [B,H,W] or [B,1,H,W] for one channel, [B,C,H,W] otherwise."""
    if channels == 1 and pred.dim() == 3:
        return tuple(pred.shape)
    if pred.dim() == 4 and pred.shape[1] == channels:
        return pred.shape[0], pred.shape[2], pred.shape[3]
    want = "[B,H,W] or [B,1,H,W]" if channels == 1 else f"[B,{channels},H,W]"
    raise _capi.OdbError(f"{name}: expected {want}, got {tuple(pred.shape)}")


def check_metric_inputs(name, pred, gt, mask, channels):
    """Checks pred / gt (fp32, contiguous, one shape) and the optional mask (uint8 / bool / fp32, contiguous,
    [B,H,W] or [B,1,H,W]); returns (b, h, w, mask pointer, ODB_MASK_*).  Nothing is copied."""
    b, h, w = metrics_plane_shape(pred, channels)
    _check_planes(name, b, h, w)
    for t, n in ((pred, "pred"), (gt, "gt")):
        _need(t, torch.float32, n)
        if metrics_plane_shape(t, channels, n) != (b, h, w) or not t.is_contiguous():
            raise _capi.OdbError(f"{name}: {n} must be a contiguous fp32 tensor of {b}x{h}x{w} planes, "
                                 f"got {tuple(t.shape)}")
    if mask is None:
        return b, h, w, None, _capi.MASK_NONE
    if not mask.is_cuda:
        raise _capi.OdbError(f"{name}: mask must live on a CUDA device (no CPU path exists)")
    if mask.dtype not in _MASK_KINDS:
        raise _capi.OdbError(f"{name}: mask must be uint8, bool or float32, got {mask.dtype}")
    if tuple(mask.shape) not in ((b, h, w), (b, 1, h, w)) or not mask.is_contiguous():
        raise _capi.OdbError(f"{name}: mask must be a contiguous [B,H,W] or [B,1,H,W] tensor for {b}x{h}x{w}, "
                             f"got {tuple(mask.shape)}")
    return b, h, w, mask.data_ptr(), _MASK_KINDS[mask.dtype]


def metrics_workspace_bytes(b: int, h: int, w: int) -> int:
    n = int(lib().odb_metrics_workspace_bytes(b, h, w))
    if n < 0:
        raise _capi.OdbError(f"metrics workspace: batch and image size must lie in [1, 65535], got {b}x{h}x{w}")
    return n


def depth_metrics_update(pred, gt, mask, space: int, min_depth: float, max_depth: float, workspace, records, sums,
                         counts, align: bool = True):
    """Adds the depth metrics of pred / gt fp32 [B,(1,)H,W] (mask: None or [B,(1,)H,W] uint8 / bool / fp32, nonzero =
    valid) to the state sums fp64 [7], counts int64 [4]; records fp64 [B, 12] receives the per-image results
    (include/omnidata_b200.h odb_depth_metrics_update).  max_depth = inf: none.  align=False: pred is already metric
    and is only clamped (odb_depth_metrics_update_metric; depth space only)."""
    b, h, w, mptr, mkind = check_metric_inputs("depth_metrics_update", pred, gt, mask, 1)
    if space not in (_capi.SPACE_DEPTH, _capi.SPACE_DISPARITY):
        raise _capi.OdbError(f"depth_metrics_update: unknown space {space}")
    if not align and space != _capi.SPACE_DEPTH:
        raise _capi.OdbError("depth_metrics_update: align=False takes depth space only")
    if not (math.isfinite(min_depth) and 0 <= min_depth < max_depth) or \
            (space == _capi.SPACE_DISPARITY and not math.isfinite(max_depth)):
        raise _capi.OdbError(f"depth_metrics_update: need 0 <= min_depth < max_depth (finite in disparity space), got "
                             f"{min_depth}, {max_depth}")
    _check_workspace("depth_metrics_update", workspace, metrics_workspace_bytes(b, h, w))
    _need_shape(records, (b, _capi.DEPTH_RECORD), torch.float64, "records")
    _need_shape(sums, (7,), torch.float64, "sums")
    _need_shape(counts, (4,), torch.int64, "counts")
    dev = _same_device(pred, gt, mask, workspace, records, sums, counts)
    tail = (float(min_depth), float(max_depth), workspace.data_ptr(), records.data_ptr(), sums.data_ptr(),
            counts.data_ptr())
    if align:
        _call("odb_depth_metrics_update", {"bytes": 2 * 2 * 4 * b * h * w}, lib().odb_depth_metrics_update, dev,
              pred.data_ptr(), gt.data_ptr(), mptr, mkind, b, h, w, space, *tail)
    else:
        _call("odb_depth_metrics_update_metric", {"bytes": 2 * 2 * 4 * b * h * w},
              lib().odb_depth_metrics_update_metric, dev, pred.data_ptr(), gt.data_ptr(), mptr, mkind, b, h, w, *tail)


def normal_metrics_update(pred, gt, mask, workspace, sums, counts, hist):
    """Adds the angular errors of pred / gt fp32 [B,3,H,W] (model encoding [0, 1]; mask as for depth) to the state
    sums fp64 [2], counts int64 [5] and hist int64 [NORMAL_HIST_BINS] (odb_normal_metrics_update)."""
    b, h, w, mptr, mkind = check_metric_inputs("normal_metrics_update", pred, gt, mask, 3)
    _check_workspace("normal_metrics_update", workspace, metrics_workspace_bytes(b, h, w))
    _need_shape(sums, (2,), torch.float64, "sums")
    _need_shape(counts, (5,), torch.int64, "counts")
    _need_shape(hist, (_capi.NORMAL_HIST_BINS,), torch.int64, "hist")
    _call("odb_normal_metrics_update", {"bytes": 2 * 3 * 4 * b * h * w}, lib().odb_normal_metrics_update,
          _same_device(pred, gt, mask, workspace, sums, counts, hist), pred.data_ptr(), gt.data_ptr(), mptr, mkind, b,
          h, w, workspace.data_ptr(), sums.data_ptr(), counts.data_ptr(), hist.data_ptr())


def normal_metrics_median(hist, out):
    """out fp64 [2] = (bin, its centre in degrees) of the lower median of the angles counted in hist; (-1, NaN) if none."""
    _need_shape(hist, (_capi.NORMAL_HIST_BINS,), torch.int64, "hist")
    _need_shape(out, (2,), torch.float64, "out")
    _call("odb_normal_metrics_median", {}, lib().odb_normal_metrics_median, _same_device(hist, out), hist.data_ptr(),
          out.data_ptr())


# ---------------------------------------------------------------- depth-boundary errors (csrc/boundary.cu)
def boundary_workspace_bytes(b: int, h: int, w: int) -> int:
    n = int(lib().odb_boundary_workspace_bytes(b, h, w))
    if n < 0:
        raise _capi.OdbError(f"boundary workspace: batch and image size must lie in [1, 65535], got {b}x{h}x{w}")
    return n


def check_edge_params(name: str, sigma: float, low: float, high: float, min_depth: float, max_depth: float):
    """OdbError unless 0 < sigma <= 4, low and high are finite with 0 <= low <= high, and 0 <= min_depth < max_depth
    (max_depth = inf: none)."""
    if not (0.0 < sigma <= 4.0):
        raise _capi.OdbError(f"{name}: sigma must lie in (0, 4], got {sigma}")
    if not (math.isfinite(low) and math.isfinite(high) and 0.0 <= low <= high):
        raise _capi.OdbError(f"{name}: need finite 0 <= low <= high, got low={low}, high={high}")
    if not (math.isfinite(min_depth) and 0.0 <= min_depth < max_depth):
        raise _capi.OdbError(f"{name}: need 0 <= min_depth < max_depth, got {min_depth}, {max_depth}")


def _edge_map(name: str, t: torch.Tensor, b: int, h: int, w: int, what: str):
    """Checks a uint8 / bool [B,H,W] or [B,1,H,W] map for b x h x w planes."""
    if not t.is_cuda:
        raise _capi.OdbError(f"{name}: {what} must live on a CUDA device (no CPU path exists)")
    if t.dtype not in (torch.uint8, torch.bool):
        raise _capi.OdbError(f"{name}: {what} must be uint8 or bool, got {t.dtype}")
    if tuple(t.shape) not in ((b, h, w), (b, 1, h, w)) or not t.is_contiguous():
        raise _capi.OdbError(f"{name}: {what} must be a contiguous [B,H,W] or [B,1,H,W] tensor for {b}x{h}x{w}, "
                             f"got {tuple(t.shape)}")


def depth_edges(depth, mask, sigma: float, low: float, high: float, min_depth: float, max_depth: float, workspace,
                edges):
    """edges uint8 [B,H,W] = the edge map E(depth, V) of depth fp32 [B,(1,)H,W], V from depth itself and the mask
    (include/omnidata_b200.h odb_depth_edges).  workspace: fp64, boundary_workspace_bytes of them."""
    b, h, w, mptr, mkind = check_metric_inputs("depth_edges", depth, depth, mask, 1)
    check_edge_params("depth_edges", sigma, low, high, min_depth, max_depth)
    _check_workspace("depth_edges", workspace, boundary_workspace_bytes(b, h, w))
    _need_shape(edges, (b, h, w), torch.uint8, "edges")
    _call("odb_depth_edges", {"bytes": 4 * b * h * w}, lib().odb_depth_edges,
          _same_device(depth, mask, workspace, edges), depth.data_ptr(), mptr, mkind, b, h, w, float(sigma),
          float(low), float(high), float(min_depth), float(max_depth), workspace.data_ptr(), edges.data_ptr())


def edge_hysteresis(weak_strong, workspace, edges):
    """edges uint8 [B,H,W] = the weak pixels of weak_strong uint8 [B,H,W] (bit 0 weak, bit 1 strong) whose 8-connected
    weak component holds a strong pixel (odb_edge_hysteresis)."""
    _need(weak_strong, torch.uint8, "weak_strong")
    if weak_strong.dim() != 3:
        raise _capi.OdbError(f"edge_hysteresis: weak_strong must be [B,H,W], got {tuple(weak_strong.shape)}")
    b, h, w = weak_strong.shape
    _check_planes("edge_hysteresis", b, h, w)
    _edge_map("edge_hysteresis", weak_strong, b, h, w, "weak_strong")
    _check_workspace("edge_hysteresis", workspace, boundary_workspace_bytes(b, h, w))
    _need_shape(edges, (b, h, w), torch.uint8, "edges")
    _call("odb_edge_hysteresis", {"bytes": 2 * b * h * w}, lib().odb_edge_hysteresis,
          _same_device(weak_strong, workspace, edges), weak_strong.data_ptr(), b, h, w, workspace.data_ptr(),
          edges.data_ptr())


def edge_distance2(edges, workspace, dist2):
    """dist2 int64 [B,H,W] = the exact squared Euclidean distance to the nearest nonzero pixel of edges uint8 / bool
    [B,H,W]; -1 (all bits set) throughout an image without one (odb_edge_distance2)."""
    if edges.dim() != 3:
        raise _capi.OdbError(f"edge_distance2: edges must be [B,H,W], got {tuple(edges.shape)}")
    b, h, w = edges.shape
    _check_planes("edge_distance2", b, h, w)
    _edge_map("edge_distance2", edges, b, h, w, "edges")
    _check_workspace("edge_distance2", workspace, boundary_workspace_bytes(b, h, w))
    _need_shape(dist2, (b, h, w), torch.int64, "dist2")
    _call("odb_edge_distance2", {"bytes": 9 * b * h * w}, lib().odb_edge_distance2,
          _same_device(edges, workspace, dist2), edges.data_ptr(), b, h, w, workspace.data_ptr(), dist2.data_ptr())


def boundary_metrics_update(pred, gt, mask, gt_edges, sigma: float, low: float, high: float, max_dist: float,
                            min_depth: float, max_depth: float, workspace, records, sums, counts):
    """Adds the depth-boundary errors of pred / gt fp32 [B,(1,)H,W] (mask as for depth_metrics_update; gt_edges None
    or uint8 / bool [B,(1,)H,W], nonzero = edge) to the state sums fp64 [2], counts int64 [5]; records fp64
    [B, BOUNDARY_RECORD] receives the per-image results (include/omnidata_b200.h odb_boundary_metrics_update)."""
    b, h, w, mptr, mkind = check_metric_inputs("boundary_metrics_update", pred, gt, mask, 1)
    if gt_edges is not None:
        _edge_map("boundary_metrics_update", gt_edges, b, h, w, "gt_edges")
    check_edge_params("boundary_metrics_update", sigma, low, high, min_depth, max_depth)
    if not (math.isfinite(max_dist) and max_dist > 0.0):
        raise _capi.OdbError(f"boundary_metrics_update: max_dist must be finite and > 0, got {max_dist}")
    _check_workspace("boundary_metrics_update", workspace, boundary_workspace_bytes(b, h, w))
    _need_shape(records, (b, _capi.BOUNDARY_RECORD), torch.float64, "records")
    _need_shape(sums, (2,), torch.float64, "sums")
    _need_shape(counts, (5,), torch.int64, "counts")
    _call("odb_boundary_metrics_update", {"bytes": 2 * 4 * b * h * w}, lib().odb_boundary_metrics_update,
          _same_device(pred, gt, mask, gt_edges, workspace, records, sums, counts), pred.data_ptr(), gt.data_ptr(),
          mptr, mkind, _ptr(gt_edges), b, h, w, float(sigma), float(low), float(high), float(max_dist),
          float(min_depth), float(max_depth), workspace.data_ptr(), records.data_ptr(), sums.data_ptr(),
          counts.data_ptr())


# ---------------------------------------------------------------- test-time ensembles (csrc/ensemble.cu)
def _ensemble_members(name, members, flips: int, channels: int):
    """Checks members fp32 [K, B, C, H, W] (contiguous; C = channels) and the mirror bits; returns (K, B, H, W)."""
    _need(members, torch.float32, "members")
    if members.dim() != 5 or members.shape[2] != channels or not members.is_contiguous():
        raise _capi.OdbError(f"{name}: members must be a contiguous fp32 [K,B,{channels},H,W] tensor, got "
                             f"{tuple(members.shape)}")
    k, b, _, h, w = members.shape
    if not 1 <= k <= _capi.ENSEMBLE_MAX_MEMBERS:
        raise _capi.OdbError(f"{name}: need 1 <= K <= {_capi.ENSEMBLE_MAX_MEMBERS} members, got {k}")
    _check_planes(name, b, h, w)
    if not 0 <= flips < (1 << k) or flips & 1:
        raise _capi.OdbError(f"{name}: flips must be a bit mask of the K members with member 0 unmirrored, got {flips}")
    return k, b, h, w


def _ensemble_spread(spread, b, h, w):
    if spread is not None:
        _need_shape(spread, (b, h, w), torch.float32, "spread")


def ensemble_gram_workspace_bytes(k: int, b: int, h: int, w: int) -> int:
    n = int(lib().odb_ensemble_gram_workspace_bytes(k, b, h, w))
    if n < 0:
        raise _capi.OdbError(f"ensemble gram workspace: refused {k} members, {b}x{h}x{w}")
    return n


def ensemble_gram(members, flips: int, gram, workspace):
    """gram fp64 [B, (K+1)(K+2)/2] = the packed upper triangle of the Gram matrix of (a_0, .., a_{K-1}, 1) over the
    pixels where all members are finite; members fp32 [K, B, 1, H, W], member k mirrored where bit k of flips is set
    (include/omnidata_b200.h odb_ensemble_gram).  workspace: fp64, ensemble_gram_workspace_bytes of them."""
    k, b, h, w = _ensemble_members("ensemble_gram", members, flips, 1)
    _need_shape(gram, (b, (k + 1) * (k + 2) // 2), torch.float64, "gram")
    _check_workspace("ensemble_gram", workspace, ensemble_gram_workspace_bytes(k, b, h, w))
    _call("odb_ensemble_gram", {"bytes": 4 * members.numel()}, lib().odb_ensemble_gram,
          _same_device(members, gram, workspace), members.data_ptr(), k, flips, b, h, w, workspace.data_ptr(),
          gram.data_ptr())


def ensemble_align_solve(gram, scale_shift):
    """scale_shift fp64 [B, K, 2] = the (s_k, t_k) that put every member in member 0's frame, from gram fp64
    [B, (K+1)(K+2)/2] (odb_ensemble_align_solve)."""
    b = scale_shift.shape[0] if scale_shift.dim() == 3 else 0
    k = scale_shift.shape[1] if scale_shift.dim() == 3 else 0
    if not 1 <= k <= _capi.ENSEMBLE_MAX_MEMBERS:
        raise _capi.OdbError(f"ensemble_align_solve: scale_shift must be [B, K, 2] with 1 <= K <= "
                             f"{_capi.ENSEMBLE_MAX_MEMBERS}, got {tuple(scale_shift.shape)}")
    _check_planes("ensemble_align_solve", b, what="batch")
    _need_shape(scale_shift, (b, k, 2), torch.float64, "scale_shift")
    _need_shape(gram, (b, (k + 1) * (k + 2) // 2), torch.float64, "gram")
    _call("odb_ensemble_align_solve", {}, lib().odb_ensemble_align_solve, _same_device(gram, scale_shift),
          gram.data_ptr(), k, b, scale_shift.data_ptr())


def ensemble_merge_depth(members, flips: int, scale_shift, out, spread=None):
    """out fp32 [B, H, W] = the per-pixel median of s_k a_k + t_k over the members fp32 [K, B, 1, H, W]; spread fp32
    [B, H, W] (optional) = the median absolute deviation from it (odb_ensemble_merge_depth)."""
    k, b, h, w = _ensemble_members("ensemble_merge_depth", members, flips, 1)
    _need_shape(scale_shift, (b, k, 2), torch.float64, "scale_shift")
    _need_shape(out, (b, h, w), torch.float32, "out")
    _ensemble_spread(spread, b, h, w)
    _call("odb_ensemble_merge_depth", {"bytes": 4 * (members.numel() + out.numel() * (1 + (spread is not None)))},
          lib().odb_ensemble_merge_depth, _same_device(members, scale_shift, out, spread), members.data_ptr(),
          scale_shift.data_ptr(), k, flips, b, h, w, out.data_ptr(), _ptr(spread))


def ensemble_merge_normal(members, flips: int, out, spread=None):
    """out fp32 [B, 3, H, W] = the re-encoded normalised mean of the decoded, un-mirrored members fp32 [K, B, 3, H, W];
    spread fp32 [B, H, W] (optional) = the members' mean angle to it in degrees (odb_ensemble_merge_normal)."""
    k, b, h, w = _ensemble_members("ensemble_merge_normal", members, flips, 3)
    _need_shape(out, (b, 3, h, w), torch.float32, "out")
    _ensemble_spread(spread, b, h, w)
    _call("odb_ensemble_merge_normal", {"bytes": 4 * (members.numel() + out.numel() + (0 if spread is None else
                                                                                      members.numel() + spread.numel()))},
          lib().odb_ensemble_merge_normal, _same_device(members, out, spread), members.data_ptr(), k, flips, b, h, w,
          out.data_ptr(), _ptr(spread))


# ---------------------------------------------------------------- guided upsampling (csrc/guided.cu)
def _guided_planes(name, t, channels, tname):
    """Checks t fp32 [B, channels, h, w] (contiguous); returns (B, h, w)."""
    _need(t, torch.float32, tname)
    if t.dim() != 4 or t.shape[1] != channels or not t.is_contiguous():
        raise _capi.OdbError(f"{name}: {tname} must be a contiguous fp32 [B,{channels},h,w] tensor, got "
                             f"{tuple(t.shape)}")
    b, _, h, w = t.shape
    _check_planes(name, b, h, w)
    return b, h, w


def _guided_channels(name, c):
    if c not in (1, 3):
        raise _capi.OdbError(f"{name}: 1 (depth) or 3 (normal) prediction channels, got {c}")


def guided_workspace_bytes(b: int, c: int, h: int, w: int) -> int:
    n = int(lib().odb_guided_workspace_bytes(b, c, h, w))
    if n < 0:
        raise _capi.OdbError(f"guided workspace: refused {b}x{c}x{h}x{w}")
    return n


def guided_coefficients(guide, pred, radius: int, eps: float, workspace, coef):
    """coef fp32 [B, 4C, h, w] = the box-averaged local linear coefficients (plane 4c + k: a_ck for k < 3, b_c for
    k = 3) of pred fp32 [B, C, h, w] against guide fp32 [B, 3, h, w] over (2 radius + 1)^2 windows, ridge eps
    (include/omnidata_b200.h odb_guided_coefficients).  workspace: fp64, guided_workspace_bytes of them."""
    b, h, w = _guided_planes("guided_coefficients", guide, 3, "guide")
    c = pred.shape[1] if pred.dim() == 4 else 0
    _guided_channels("guided_coefficients", c)
    if _guided_planes("guided_coefficients", pred, c, "pred") != (b, h, w):
        raise _capi.OdbError(f"guided_coefficients: pred {tuple(pred.shape)} does not match guide {tuple(guide.shape)}")
    if not 1 <= radius <= _capi.GUIDED_MAX_RADIUS:
        raise _capi.OdbError(f"guided_coefficients: radius must lie in [1, {_capi.GUIDED_MAX_RADIUS}], got {radius}")
    if not (math.isfinite(eps) and eps > 0):
        raise _capi.OdbError(f"guided_coefficients: eps must be finite and > 0, got {eps}")
    _need_shape(coef, (b, 4 * c, h, w), torch.float32, "coef")
    _check_workspace("guided_coefficients", workspace, guided_workspace_bytes(b, c, h, w))
    _call("odb_guided_coefficients", {"bytes": 4 * (guide.numel() + pred.numel() + coef.numel())},
          lib().odb_guided_coefficients, _same_device(guide, pred, workspace, coef), guide.data_ptr(), pred.data_ptr(),
          b, c, h, w, int(radius), float(eps), workspace.data_ptr(), coef.data_ptr())


def guided_apply(image, coef, out):
    """out fp32 [B, C, H, W] = B_c + A_c . x per pixel, x = image fp32 [B, 3, H, W] and (A_c, B_c) = coef fp32
    [B, 4C, h, w] resampled to H x W as resize_bilinear resamples (odb_guided_apply)."""
    b, H, W = _guided_planes("guided_apply", image, 3, "image")
    c4 = coef.shape[1] if coef.dim() == 4 else 0
    _guided_channels("guided_apply", c4 // 4 if c4 % 4 == 0 else 0)
    bc, h, w = _guided_planes("guided_apply", coef, c4, "coef")
    if bc != b:
        raise _capi.OdbError(f"guided_apply: coef {tuple(coef.shape)} and image {tuple(image.shape)} differ in batch")
    _need_shape(out, (b, c4 // 4, H, W), torch.float32, "out")
    from .imageproc import resample_tables
    dev = _same_device(image, coef, out)
    bh, wh, kh = resample_tables(w, W, dev)
    bv, wv, kv = resample_tables(h, H, dev)
    _call("odb_guided_apply", {"bytes": 4 * (image.numel() + out.numel())}, lib().odb_guided_apply, dev,
          image.data_ptr(), coef.data_ptr(), b, c4 // 4, h, w, H, W, bh.data_ptr(), wh.data_ptr(), kh, bv.data_ptr(),
          wv.data_ptr(), kv, out.data_ptr())


# ---------------------------------------------------------------- sparse metric alignment (csrc/sparse.cu)
def check_sparse_grid(name: str, grid: Tuple[int, int], h: int, w: int):
    """OdbError unless 1 <= gy <= h, 1 <= gx <= w and gy gx <= SPARSE_MAX_NODES."""
    gy, gx = grid
    if not (1 <= gy <= h and 1 <= gx <= w and gy * gx <= _capi.SPARSE_MAX_NODES):
        raise _capi.OdbError(f"{name}: grid {gy}x{gx} for {h}x{w} images: need 1 <= gy <= h, 1 <= gx <= w and at "
                             f"most {_capi.SPARSE_MAX_NODES} nodes")


def _check_depth_range(name: str, space: int, min_depth: float, max_depth: float):
    if space not in (_capi.SPACE_DEPTH, _capi.SPACE_DISPARITY):
        raise _capi.OdbError(f"{name}: unknown space {space}")
    if not (math.isfinite(min_depth) and 0 <= min_depth < max_depth) or \
            (space == _capi.SPACE_DISPARITY and not math.isfinite(max_depth)):
        raise _capi.OdbError(f"{name}: need 0 <= min_depth < max_depth (finite in disparity space), got "
                             f"{min_depth}, {max_depth}")


def sparse_align_workspace_bytes(b: int, h: int, w: int, grid: Tuple[int, int]) -> int:
    _check_planes("sparse_align_workspace_bytes", b, h, w)
    check_sparse_grid("sparse_align_workspace_bytes", grid, h, w)
    return int(lib().odb_sparse_align_workspace_bytes(b, h, w, grid[0], grid[1]))


def sparse_align_fit(pred, sparse, mask, grid: Tuple[int, int], space: int, min_depth: float, max_depth: float,
                     smooth: float, robust: float, iterations: int, workspace, nodes, records):
    """nodes fp64 [B, gy, gx, 2] = the scale / shift nodes fitted to the sparse depths sparse fp32 [B,(1,)H,W] (metres;
    mask: None or [B,(1,)H,W] uint8 / bool / fp32, nonzero = valid) from pred fp32 [B,(1,)H,W]; records fp64
    [B, SPARSE_RECORD] (include/omnidata_b200.h odb_sparse_align_fit).  robust = 0: one least-squares solve
    (iterations 1); robust = delta > 0: iterations in [2, 32] Huber IRLS solves.  max_depth = inf: none."""
    name = "sparse_align_fit"
    b, h, w, mptr, mkind = check_metric_inputs(name, pred, sparse, mask, 1)
    check_sparse_grid(name, grid, h, w)
    _check_depth_range(name, space, min_depth, max_depth)
    if not (math.isfinite(smooth) and smooth >= 0 and (smooth > 0 or grid[0] * grid[1] == 1)):
        raise _capi.OdbError(f"{name}: smooth must be finite, >= 0, and > 0 for more than one node, got {smooth}")
    if not (math.isfinite(robust) and robust >= 0) or \
            not (2 <= iterations <= 32 if robust > 0 else iterations == 1):
        raise _capi.OdbError(f"{name}: need robust = 0 with 1 iteration or robust > 0 with 2..32 iterations, got "
                             f"robust={robust}, iterations={iterations}")
    _check_workspace(name, workspace, sparse_align_workspace_bytes(b, h, w, grid))
    _need_shape(nodes, (b, grid[0], grid[1], 2), torch.float64, "nodes")
    _need_shape(records, (b, _capi.SPARSE_RECORD), torch.float64, "records")
    _call("odb_sparse_align_fit", {"bytes": 2 * 4 * b * h * w * (iterations + 1)}, lib().odb_sparse_align_fit,
          _same_device(pred, sparse, mask, workspace, nodes, records), pred.data_ptr(), sparse.data_ptr(), mptr, mkind,
          b, h, w, grid[0], grid[1], space, float(min_depth), float(max_depth), float(smooth), float(robust),
          int(iterations), workspace.data_ptr(), nodes.data_ptr(), records.data_ptr())


def sparse_align_apply(pred, nodes, out, space: int, min_depth: float, max_depth: float):
    """out fp32 [B,H,W] = the metric depth of pred fp32 [B,(1,)H,W] under the nodes fp64 [B, gy, gx, 2]
    (odb_sparse_align_apply)."""
    name = "sparse_align_apply"
    b, h, w = metrics_plane_shape(pred, 1)
    _check_planes(name, b, h, w)
    _need(pred, torch.float32, "pred")
    if not pred.is_contiguous():
        raise _capi.OdbError(f"{name}: pred must be contiguous")
    _need(nodes, torch.float64, "nodes")
    if nodes.dim() != 4 or nodes.shape[0] != b or nodes.shape[3] != 2:
        raise _capi.OdbError(f"{name}: nodes must be fp64 [{b}, gy, gx, 2], got {tuple(nodes.shape)}")
    grid = (nodes.shape[1], nodes.shape[2])
    check_sparse_grid(name, grid, h, w)
    _need_shape(nodes, (b, grid[0], grid[1], 2), torch.float64, "nodes")
    _check_depth_range(name, space, min_depth, max_depth)
    _need_shape(out, (b, h, w), torch.float32, "out")
    _call("odb_sparse_align_apply", {"bytes": 2 * 4 * b * h * w}, lib().odb_sparse_align_apply,
          _same_device(pred, nodes, out), pred.data_ptr(), nodes.data_ptr(), b, h, w, grid[0], grid[1], space,
          float(min_depth), float(max_depth), out.data_ptr())


# ---------------------------------------------------------------- depth-normal fusion (csrc/fusion.cu)
def check_intrinsics(name: str, intrinsics) -> Tuple[float, float, float, float]:
    """(fx, fy, cx, cy) as floats; OdbError unless fx, fy > 0 and all four are finite."""
    try:
        fx, fy, cx, cy = (float(v) for v in intrinsics)
    except (TypeError, ValueError):
        raise _capi.OdbError(f"{name}: intrinsics must be (fx, fy, cx, cy), got {intrinsics!r}") from None
    if not all(math.isfinite(v) for v in (fx, fy, cx, cy)) or fx <= 0 or fy <= 0:
        raise _capi.OdbError(f"{name}: intrinsics need finite fx, fy > 0 and finite cx, cy, got {intrinsics!r}")
    return fx, fy, cx, cy


def _check_axes_jump(name: str, axes, jump: float):
    if len(tuple(axes)) != 3 or any(v not in (1, -1) for v in axes):
        raise _capi.OdbError(f"{name}: axes must be three signs +-1, got {axes!r}")
    if not (math.isfinite(jump) and jump > 0):
        raise _capi.OdbError(f"{name}: jump must be finite and > 0, got {jump}")


def fusion_workspace_bytes(b: int, h: int, w: int) -> int:
    _check_planes("fusion_workspace_bytes", b, h, w)
    return int(lib().odb_fusion_workspace_bytes(b, h, w))


def depth_normals_workspace_bytes(b: int, h: int, w: int) -> int:
    _check_planes("depth_normals_workspace_bytes", b, h, w)
    return int(lib().odb_depth_normals_workspace_bytes(b, h, w))


def depth_normal_fusion(depth, normals, mask, intrinsics, axes, jump: float, weight: float, shift: bool,
                        iterations: int, tol: float, workspace, out, records):
    """out fp32 [B,H,W] = depth fp32 [B,(1,)H,W] fused with normals fp32 [B,3,H,W] (the normal model's [0, 1] encoding;
    mask: None or [B,(1,)H,W] uint8 / bool / fp32, nonzero = valid); records fp64 [B, FUSION_RECORD]
    (include/omnidata_b200.h odb_depth_normal_fusion)."""
    name = "depth_normal_fusion"
    b, h, w, mptr, mkind = check_metric_inputs(name, depth, depth, mask, 1)
    _need(normals, torch.float32, "normals")
    if tuple(normals.shape) != (b, 3, h, w) or not normals.is_contiguous():
        raise _capi.OdbError(f"{name}: normals must be a contiguous fp32 [{b}, 3, {h}, {w}] tensor, got "
                             f"{tuple(normals.shape)}")
    fx, fy, cx, cy = check_intrinsics(name, intrinsics)
    _check_axes_jump(name, axes, jump)
    if not (math.isfinite(weight) and weight > 0) or not (math.isfinite(tol) and tol > 0) or \
            not 1 <= iterations <= 10000:
        raise _capi.OdbError(f"{name}: need weight > 0, tol > 0 (finite) and iterations in [1, 10000], got "
                             f"{weight}, {tol}, {iterations}")
    _check_workspace(name, workspace, fusion_workspace_bytes(b, h, w))
    if workspace.data_ptr() % 16:
        raise _capi.OdbError(f"{name}: workspace must be 16-byte aligned")
    _need_shape(out, (b, h, w), torch.float32, "out")
    _need_shape(records, (b, _capi.FUSION_RECORD), torch.float64, "records")
    _call("odb_depth_normal_fusion", {"bytes": 128 * b * h * w * iterations}, lib().odb_depth_normal_fusion,
          _same_device(depth, normals, mask, workspace, out, records), depth.data_ptr(), normals.data_ptr(), mptr,
          mkind, b, h, w, fx, fy, cx, cy, int(axes[0]), int(axes[1]), int(axes[2]), float(jump), float(weight),
          1 if shift else 0, int(iterations), float(tol), workspace.data_ptr(), out.data_ptr(), records.data_ptr())


def depth_normals(depth, mask, intrinsics, axes, jump: float, workspace, out):
    """out fp32 [B,3,H,W] = the normals of depth fp32 [B,(1,)H,W] in the normal model's encoding, NaN where undefined
    (include/omnidata_b200.h odb_depth_normals)."""
    name = "depth_normals"
    b, h, w, mptr, mkind = check_metric_inputs(name, depth, depth, mask, 1)
    fx, fy, cx, cy = check_intrinsics(name, intrinsics)
    _check_axes_jump(name, axes, jump)
    _check_workspace(name, workspace, depth_normals_workspace_bytes(b, h, w))
    _need_shape(out, (b, 3, h, w), torch.float32, "out")
    _call("odb_depth_normals", {"bytes": 16 * b * h * w}, lib().odb_depth_normals,
          _same_device(depth, mask, workspace, out), depth.data_ptr(), mptr, mkind, b, h, w, fx, fy, cx, cy,
          int(axes[0]), int(axes[1]), int(axes[2]), float(jump), workspace.data_ptr(), out.data_ptr())


# ---------------------------------------------------------------- TSDF volumes (csrc/volume.cu)
def check_volume_grid(name: str, dims, origin, voxel: float) -> Tuple[Tuple[int, int, int], Tuple[float, float, float]]:
    """((nx, ny, nz), origin) as ints / floats; OdbError unless each dimension lies in [2, TSDF_MAX_DIM], nx ny nz <=
    TSDF_MAX_POINTS, the origin is finite and voxel is finite and > 0."""
    try:
        nx, ny, nz = (int(v) for v in dims)
        ox, oy, oz = (float(v) for v in origin)
    except (TypeError, ValueError):
        raise _capi.OdbError(f"{name}: dims must be (nx, ny, nz) and origin (x, y, z), got {dims!r}, {origin!r}") \
            from None
    if tuple(dims) != (nx, ny, nz) or not all(2 <= d <= _capi.TSDF_MAX_DIM for d in (nx, ny, nz)) or \
            nx * ny * nz > _capi.TSDF_MAX_POINTS:
        raise _capi.OdbError(f"{name}: dims must lie in [2, {_capi.TSDF_MAX_DIM}] with nx ny nz <= "
                             f"{_capi.TSDF_MAX_POINTS}, got {dims!r}")
    if not all(math.isfinite(v) for v in (ox, oy, oz)) or not (math.isfinite(voxel) and voxel > 0):
        raise _capi.OdbError(f"{name}: need a finite origin and a finite voxel > 0, got {origin!r}, {voxel}")
    return (nx, ny, nz), (ox, oy, oz)


def check_poses(name: str, cam_to_world) -> np.ndarray:
    """Host float64 [B, 16] (row-major 4 x 4 camera-to-world matrices) from numpy or a CPU tensor, [B,4,4] or [4,4];
    OdbError unless every pose is finite with last row 0 0 0 1 and |R^T R - I| <= 1e-6 entrywise."""
    if isinstance(cam_to_world, torch.Tensor):
        if cam_to_world.device.type != "cpu":
            raise _capi.OdbError(f"{name}: poses are host data (numpy or a CPU tensor), got a {cam_to_world.device} "
                                 "tensor")
        cam_to_world = cam_to_world.numpy()
    T = np.asarray(cam_to_world, dtype=np.float64)
    if T.shape == (4, 4):
        T = T[None]
    if T.ndim != 3 or T.shape[1:] != (4, 4) or T.shape[0] < 1:
        raise _capi.OdbError(f"{name}: poses must be [B,4,4] or [4,4], got {T.shape}")
    if not np.isfinite(T).all():
        raise _capi.OdbError(f"{name}: poses must be finite")
    if not (T[:, 3] == np.array([0.0, 0.0, 0.0, 1.0])).all():
        raise _capi.OdbError(f"{name}: the last row of a pose must be 0 0 0 1")
    R = T[:, :3, :3]
    if np.abs(np.einsum("bki,bkj->bij", R, R) - np.eye(3)).max() > 1e-6:
        raise _capi.OdbError(f"{name}: the rotation of a pose is not orthonormal (|R^T R - I| > 1e-6)")
    return np.ascontiguousarray(T.reshape(-1, 16))


def _volume_planes(name: str, tsdf, weight, color, dims):
    nx, ny, nz = dims
    _need_shape(tsdf, (nz, ny, nx), torch.float32, "tsdf")
    _need_shape(weight, (nz, ny, nx), torch.float32, "weight")
    if color is not None:
        _need_shape(color, (3, nz, ny, nx), torch.float32, "color")


def tsdf_mesh_workspace_bytes(dims) -> int:
    nx, ny, nz = check_volume_grid("tsdf_mesh_workspace_bytes", dims, (0, 0, 0), 1.0)[0]
    return int(lib().odb_tsdf_mesh_workspace_bytes(nx, ny, nz))


def tsdf_integrate(tsdf, weight, color, dims, origin, voxel: float, trunc: float, depth, rgb, intrinsics,
                   cam_to_world):
    """Integrates depth fp32 [B,H,W] (metres; rgb fp32 [B,3,H,W] exactly when color is given) seen from cam_to_world
    (host, see check_poses) into tsdf, weight fp32 [nz,ny,nx] and color fp32 [3,nz,ny,nx] in place
    (include/omnidata_b200.h odb_tsdf_integrate)."""
    name = "tsdf_integrate"
    dims, origin = check_volume_grid(name, dims, origin, voxel)
    if not (math.isfinite(trunc) and trunc > 0):
        raise _capi.OdbError(f"{name}: trunc must be finite and > 0, got {trunc}")
    _volume_planes(name, tsdf, weight, color, dims)
    _need(depth, torch.float32, "depth")
    if depth.dim() != 3 or not depth.is_contiguous():
        raise _capi.OdbError(f"{name}: depth must be a contiguous fp32 [B,H,W] tensor, got {tuple(depth.shape)}")
    b, h, w = depth.shape
    _check_planes(name, b, h, w)
    if (color is None) != (rgb is None):
        raise _capi.OdbError(f"{name}: rgb is required exactly when the volume stores colour")
    if rgb is not None:
        _need_shape(rgb, (b, 3, h, w), torch.float32, "rgb")
    fx, fy, cx, cy = check_intrinsics(name, intrinsics)
    T = check_poses(name, cam_to_world)
    if T.shape[0] != b:
        raise _capi.OdbError(f"{name}: {b} depth frames but {T.shape[0]} poses")
    n = dims[0] * dims[1] * dims[2]
    _call(name, {"bytes": 8 * n + 4 * b * h * w}, lib().odb_tsdf_integrate,
          _same_device(tsdf, weight, color, depth, rgb), tsdf.data_ptr(), weight.data_ptr(), _ptr(color), *dims,
          *origin, float(voxel), float(trunc), depth.data_ptr(), _ptr(rgb), b, h, w, fx, fy, cx, cy, T.ctypes.data)


def tsdf_raycast(tsdf, weight, dims, origin, voxel: float, intrinsics, cam_to_world, step: float, out):
    """out fp32 [H,W] = the z-depth of the first surface seen from cam_to_world (host [4,4]), 0 where none
    (include/omnidata_b200.h odb_tsdf_raycast)."""
    _raycast("tsdf_raycast", tsdf, weight, None, dims, origin, voxel, intrinsics, cam_to_world, step, out, None)


def tsdf_raycast_color(tsdf, weight, color, dims, origin, voxel: float, intrinsics, cam_to_world, step: float, out,
                       rgb):
    """out fp32 [H,W] as tsdf_raycast, bit for bit, and rgb fp32 [3,H,W] = the colour of color fp32 [3,nz,ny,nx] at
    the hit, NaN where out = 0 (include/omnidata_b200.h odb_tsdf_raycast_color)."""
    name = "tsdf_raycast_color"
    if color is None or rgb is None:
        raise _capi.OdbError(f"{name}: needs the volume's colour planes and an rgb output")
    _raycast(name, tsdf, weight, color, dims, origin, voxel, intrinsics, cam_to_world, step, out, rgb)


def _raycast(name, tsdf, weight, color, dims, origin, voxel, intrinsics, cam_to_world, step, out, rgb):
    dims, origin = check_volume_grid(name, dims, origin, voxel)
    _volume_planes(name, tsdf, weight, color, dims)
    fx, fy, cx, cy = check_intrinsics(name, intrinsics)
    T = check_poses(name, cam_to_world)
    if T.shape[0] != 1:
        raise _capi.OdbError(f"{name}: one pose, got {T.shape[0]}")
    if not (math.isfinite(step) and voxel / 64 <= step <= voxel):
        raise _capi.OdbError(f"{name}: step must lie in [voxel / 64, voxel], got {step}")
    _need(out, torch.float32, "out")
    if out.dim() != 2 or not out.is_contiguous():
        raise _capi.OdbError(f"{name}: out must be a contiguous fp32 [H,W] tensor, got {tuple(out.shape)}")
    h, w = out.shape
    _check_planes(name, 1, h, w)
    if color is None:
        _call(name, {"bytes": 4 * h * w}, lib().odb_tsdf_raycast, _same_device(tsdf, weight, out), tsdf.data_ptr(),
              weight.data_ptr(), *dims, *origin, float(voxel), T.ctypes.data, h, w, fx, fy, cx, cy, float(step),
              out.data_ptr())
        return
    _need_shape(rgb, (3, h, w), torch.float32, "rgb")
    _call(name, {"bytes": 16 * h * w}, lib().odb_tsdf_raycast_color, _same_device(tsdf, weight, color, out, rgb),
          tsdf.data_ptr(), weight.data_ptr(), color.data_ptr(), *dims, *origin, float(voxel), T.ctypes.data, h, w, fx,
          fy, cx, cy, float(step), out.data_ptr(), rgb.data_ptr())


def tsdf_mesh_count(tsdf, weight, dims, workspace, counts):
    """counts int64 [2] = (vertices, faces) of the mesh of tsdf / weight; fills workspace for tsdf_mesh_emit
    (include/omnidata_b200.h odb_tsdf_mesh_count)."""
    name = "tsdf_mesh_count"
    dims = check_volume_grid(name, dims, (0, 0, 0), 1.0)[0]
    _volume_planes(name, tsdf, weight, None, dims)
    _check_workspace(name, workspace, tsdf_mesh_workspace_bytes(dims))
    _need_shape(counts, (2,), torch.int64, "counts")
    n = dims[0] * dims[1] * dims[2]
    _call(name, {"bytes": 14 * n}, lib().odb_tsdf_mesh_count, _same_device(tsdf, weight, workspace, counts),
          tsdf.data_ptr(), weight.data_ptr(), *dims, workspace.data_ptr(), counts.data_ptr())


def tsdf_mesh_emit(tsdf, weight, color, dims, origin, voxel: float, workspace, vertices, faces, colors):
    """vertices fp32 [V,3], faces int32 [F,3] and colors fp32 [V,3] (exactly when color is given), sized from the counts
    of tsdf_mesh_count on the same workspace (include/omnidata_b200.h odb_tsdf_mesh_emit)."""
    name = "tsdf_mesh_emit"
    dims, origin = check_volume_grid(name, dims, origin, voxel)
    _volume_planes(name, tsdf, weight, color, dims)
    _check_workspace(name, workspace, tsdf_mesh_workspace_bytes(dims))
    for t, dt, n in ((vertices, torch.float32, "vertices"), (faces, torch.int32, "faces")):
        _need(t, dt, n)
        if t.dim() != 2 or t.shape[1] != 3 or not t.is_contiguous():
            raise _capi.OdbError(f"{name}: {n} must be a contiguous [N, 3] tensor, got {tuple(t.shape)}")
    if (color is None) != (colors is None):
        raise _capi.OdbError(f"{name}: colors is required exactly when the volume stores colour")
    if colors is not None:
        _need_shape(colors, tuple(vertices.shape), torch.float32, "colors")
    n = dims[0] * dims[1] * dims[2]
    _call(name, {"bytes": 14 * n}, lib().odb_tsdf_mesh_emit,
          _same_device(tsdf, weight, color, workspace, vertices, faces, colors), tsdf.data_ptr(), weight.data_ptr(),
          _ptr(color), *dims, *origin, float(voxel), workspace.data_ptr(), vertices.data_ptr(), faces.data_ptr(),
          _ptr(colors))


# ---------------------------------------------------------------- sparse TSDF volumes (csrc/sparse_volume.cu)
def sparse_tsdf_desc(data, keys, birth, nbr, table_keys, table_ids, table_birth, bbox, scratch, blocks: int,
                     origin, voxel: float) -> _capi.SparseTSDF:
    """The odb_sparse_tsdf descriptor of one volume's device arrays (include/omnidata_b200.h): data fp32
    [capacity, 2 or 5, 512], keys int64 / birth int32 [capacity], nbr int32 [capacity, 8], the table int64 / int32 /
    int32 [table_size], bbox int32 [6], scratch int32 [2 + table_size]; OdbError on any mismatch."""
    name = "sparse_tsdf"
    _need(data, torch.float32, "data")
    if data.dim() != 3 or data.shape[1] not in (2, 5) or data.shape[2] != 512 or not data.is_contiguous():
        raise _capi.OdbError(f"{name}: data must be a contiguous fp32 [capacity, 2 or 5, 512], got {tuple(data.shape)}")
    cap, tsize = data.shape[0], table_keys.numel()
    for t, shape, dt, n in ((keys, (cap,), torch.int64, "keys"), (birth, (cap,), torch.int32, "birth"),
                            (nbr, (cap, 8), torch.int32, "nbr"), (table_keys, (tsize,), torch.int64, "table_keys"),
                            (table_ids, (tsize,), torch.int32, "table_ids"),
                            (table_birth, (tsize,), torch.int32, "table_birth"), (bbox, (6,), torch.int32, "bbox"),
                            (scratch, (2 + tsize,), torch.int32, "scratch")):
        _need_shape(t, shape, dt, n)
    _same_device(data, keys, birth, nbr, table_keys, table_ids, table_birth, bbox, scratch)
    if not 0 <= blocks <= cap or cap > _capi.SPARSE_TSDF_MAX_BLOCKS or tsize < 1024 or tsize & (tsize - 1) or \
            blocks > tsize // 2:
        raise _capi.OdbError(f"{name}: {blocks} blocks do not fit capacity {cap} and table size {tsize}")
    ox, oy, oz = (float(v) for v in origin)
    if not all(math.isfinite(v) for v in (ox, oy, oz)) or not (math.isfinite(voxel) and voxel > 0):
        raise _capi.OdbError(f"{name}: need a finite origin and a finite voxel > 0, got {origin!r}, {voxel}")
    return _capi.SparseTSDF(data.data_ptr(), keys.data_ptr(), birth.data_ptr(), nbr.data_ptr(), table_keys.data_ptr(),
                            table_ids.data_ptr(), table_birth.data_ptr(), bbox.data_ptr(), scratch.data_ptr(),
                            int(blocks), int(cap), int(tsize), int(data.shape[1]), ox, oy, oz, float(voxel))


def _sparse_frames(name, depth, rgb, channels, intrinsics, cam_to_world):
    _need(depth, torch.float32, "depth")
    if depth.dim() != 3 or not depth.is_contiguous():
        raise _capi.OdbError(f"{name}: depth must be a contiguous fp32 [B,H,W] tensor, got {tuple(depth.shape)}")
    b, h, w = depth.shape
    _check_planes(name, b, h, w)
    if (channels == 5) != (rgb is not None):
        raise _capi.OdbError(f"{name}: rgb is required exactly when the volume stores colour")
    if rgb is not None:
        _need_shape(rgb, (b, 3, h, w), torch.float32, "rgb")
    k = check_intrinsics(name, intrinsics)
    T = check_poses(name, cam_to_world)
    if T.shape[0] != b:
        raise _capi.OdbError(f"{name}: {b} depth frames but {T.shape[0]} poses")
    return b, h, w, k, T


def sparse_tsdf_rebuild(desc: _capi.SparseTSDF, device):
    """Clears the hash table and inserts the allocated blocks with their ids (odb_sparse_tsdf_rebuild)."""
    _call("sparse_tsdf_rebuild", {}, lib().odb_sparse_tsdf_rebuild, device, C.byref(desc))


def sparse_tsdf_mark(desc: _capi.SparseTSDF, device, trunc: float, max_depth: float, depth, intrinsics, cam_to_world,
                     frame0: int):
    """Inserts the blocks covered by depth fp32 [B,H,W] seen from cam_to_world into the table; scratch[0:2] = (new
    blocks, table half full) (odb_sparse_tsdf_mark)."""
    name = "sparse_tsdf_mark"
    b, h, w, (fx, fy, cx, cy), T = _sparse_frames(name, depth, None, 2, intrinsics, cam_to_world)
    if not (math.isfinite(trunc) and trunc > 0 and math.isfinite(max_depth) and max_depth > 0):
        raise _capi.OdbError(f"{name}: trunc and max_depth must be finite and > 0, got {trunc}, {max_depth}")
    _call(name, {"bytes": 4 * b * h * w}, lib().odb_sparse_tsdf_mark, _same_device(depth), C.byref(desc),
          float(trunc), float(max_depth), depth.data_ptr(), b, h, w, fx, fy, cx, cy, T.ctypes.data, int(frame0))


def sparse_tsdf_commit_workspace_bytes(n_new: int) -> int:
    return int(lib().odb_sparse_tsdf_commit_workspace_bytes(int(n_new)))


def sparse_tsdf_commit(desc: _capi.SparseTSDF, device, n_new: int, workspace):
    """Gives the n_new marked blocks their ids (odb_sparse_tsdf_commit)."""
    name = "sparse_tsdf_commit"
    _check_workspace(name, workspace, sparse_tsdf_commit_workspace_bytes(n_new))
    _call(name, {}, lib().odb_sparse_tsdf_commit, device, C.byref(desc), int(n_new), workspace.data_ptr())


def sparse_tsdf_integrate(desc: _capi.SparseTSDF, device, trunc: float, depth, rgb, intrinsics, cam_to_world,
                          frame0: int):
    """Integrates depth fp32 [B,H,W] (rgb fp32 [B,3,H,W] exactly when the volume stores colour), frames numbered
    frame0.., into the allocated blocks (odb_sparse_tsdf_integrate)."""
    name = "sparse_tsdf_integrate"
    b, h, w, (fx, fy, cx, cy), T = _sparse_frames(name, depth, rgb, desc.channels, intrinsics, cam_to_world)
    if not (math.isfinite(trunc) and trunc > 0):
        raise _capi.OdbError(f"{name}: trunc must be finite and > 0, got {trunc}")
    _call(name, {"bytes": 4 * desc.channels * 512 * desc.blocks + 4 * b * h * w}, lib().odb_sparse_tsdf_integrate,
          _same_device(depth, rgb), C.byref(desc), float(trunc), depth.data_ptr(), _ptr(rgb), b, h, w, fx, fy, cx, cy,
          T.ctypes.data, int(frame0))


def sparse_tsdf_raycast(desc: _capi.SparseTSDF, device, intrinsics, cam_to_world, step: float, out, rgb=None):
    """out fp32 [H,W] (and rgb fp32 [3,H,W] for a colour volume) as tsdf_raycast / tsdf_raycast_color over the
    allocated blocks' bounding box (odb_sparse_tsdf_raycast)."""
    name = "sparse_tsdf_raycast"
    fx, fy, cx, cy = check_intrinsics(name, intrinsics)
    T = check_poses(name, cam_to_world)
    if T.shape[0] != 1:
        raise _capi.OdbError(f"{name}: one pose, got {T.shape[0]}")
    if not (math.isfinite(step) and desc.voxel / 64 <= step <= desc.voxel):
        raise _capi.OdbError(f"{name}: step must lie in [voxel / 64, voxel], got {step}")
    _need(out, torch.float32, "out")
    if out.dim() != 2 or not out.is_contiguous():
        raise _capi.OdbError(f"{name}: out must be a contiguous fp32 [H,W] tensor, got {tuple(out.shape)}")
    h, w = out.shape
    _check_planes(name, 1, h, w)
    if rgb is not None:
        if desc.channels != 5:
            raise _capi.OdbError(f"{name}: rgb needs a volume that stores colour")
        _need_shape(rgb, (3, h, w), torch.float32, "rgb")
    _call(name, {"bytes": (16 if rgb is not None else 4) * h * w}, lib().odb_sparse_tsdf_raycast,
          _same_device(out, rgb), C.byref(desc), T.ctypes.data, h, w, fx, fy, cx, cy, float(step), out.data_ptr(),
          _ptr(rgb))


def sparse_tsdf_mesh_workspace_bytes(blocks: int) -> int:
    return int(lib().odb_sparse_tsdf_mesh_workspace_bytes(int(blocks)))


def sparse_tsdf_mesh_count(desc: _capi.SparseTSDF, device, workspace, counts):
    """counts int64 [2] = (vertices, faces) of the volume's mesh; fills workspace (odb_sparse_tsdf_mesh_count)."""
    name = "sparse_tsdf_mesh_count"
    _check_workspace(name, workspace, sparse_tsdf_mesh_workspace_bytes(desc.blocks))
    _need_shape(counts, (2,), torch.int64, "counts")
    _call(name, {"bytes": 10 * 512 * desc.blocks}, lib().odb_sparse_tsdf_mesh_count,
          _same_device(workspace, counts), C.byref(desc), workspace.data_ptr(), counts.data_ptr())


def sparse_tsdf_mesh_emit(desc: _capi.SparseTSDF, device, workspace, vertices, faces, colors):
    """vertices fp32 [V,3], faces int32 [F,3] and colors fp32 [V,3] (exactly for a colour volume), sized from
    sparse_tsdf_mesh_count on the same workspace (odb_sparse_tsdf_mesh_emit)."""
    name = "sparse_tsdf_mesh_emit"
    _check_workspace(name, workspace, sparse_tsdf_mesh_workspace_bytes(desc.blocks))
    for t, dt, n in ((vertices, torch.float32, "vertices"), (faces, torch.int32, "faces")):
        _need(t, dt, n)
        if t.dim() != 2 or t.shape[1] != 3 or not t.is_contiguous():
            raise _capi.OdbError(f"{name}: {n} must be a contiguous [N, 3] tensor, got {tuple(t.shape)}")
    if (desc.channels == 5) != (colors is not None):
        raise _capi.OdbError(f"{name}: colors is required exactly when the volume stores colour")
    if colors is not None:
        _need_shape(colors, tuple(vertices.shape), torch.float32, "colors")
    _call(name, {"bytes": 10 * 512 * desc.blocks}, lib().odb_sparse_tsdf_mesh_emit,
          _same_device(workspace, vertices, faces, colors), C.byref(desc), workspace.data_ptr(), vertices.data_ptr(),
          faces.data_ptr(), _ptr(colors))


# ---------------------------------------------------------------- camera tracking (csrc/track.cu)
TRACK_MAX_ITERATIONS = 100


def track_workspace_bytes(h: int, w: int) -> int:
    _check_planes("track_workspace_bytes", 1, h, w)
    return int(lib().odb_track_workspace_bytes(h, w))


def check_track_params(name: str, affine, iterations, tol: float, robust: float, max_dist: float, min_overlap: float):
    """OdbError unless affine is a bool, iterations an integer in [1, 100], tol, robust and max_dist finite and > 0, and
    min_overlap in (0, 1]."""
    if not isinstance(affine, bool):
        raise _capi.OdbError(f"{name}: affine must be a bool, got {affine!r}")
    if isinstance(iterations, bool) or not isinstance(iterations, (int, np.integer)) or \
            not 1 <= iterations <= TRACK_MAX_ITERATIONS:
        raise _capi.OdbError(f"{name}: iterations must be an integer in [1, {TRACK_MAX_ITERATIONS}], got "
                             f"{iterations!r}")
    for what, v in (("tol", tol), ("robust", robust), ("max_dist", max_dist)):
        if isinstance(v, bool) or not (isinstance(v, numbers.Real) and math.isfinite(v) and v > 0):
            raise _capi.OdbError(f"{name}: {what} must be finite and > 0, got {v!r}")
    if isinstance(min_overlap, bool) or not (isinstance(min_overlap, numbers.Real) and 0 < min_overlap <= 1):
        raise _capi.OdbError(f"{name}: min_overlap must lie in (0, 1], got {min_overlap!r}")


def check_photometric(name: str, photometric, photometric_robust):
    """OdbError unless photometric (lambda) is finite and >= 0 and photometric_robust is finite and > 0."""
    for what, v in (("photometric", photometric), ("photometric_robust", photometric_robust)):
        if isinstance(v, bool) or not (isinstance(v, numbers.Real) and math.isfinite(v)):
            raise _capi.OdbError(f"{name}: {what} must be a finite number, got {v!r}")
    if photometric < 0 or photometric_robust <= 0:
        raise _capi.OdbError(f"{name}: need photometric >= 0 and photometric_robust > 0, got {photometric!r}, "
                             f"{photometric_robust!r}")


def track_frame(pred, ref_depth, ref_normals, intrinsics, ref_pose, init_pose, init_nodes, affine: bool,
                iterations: int, tol: float, robust: float, max_dist: float, min_overlap: float, workspace, pose,
                nodes, record, rgb=None, ref_rgb=None, ref_intensity=None, photometric: float = 0.0,
                photometric_robust: float = 0.1):
    """pose fp64 [4,4], nodes fp64 [1,1,1,2] and record fp64 [TRACK_RECORD] of pred fp32 [(1,)H,W] tracked against
    ref_depth fp32 [H,W] and its normals ref_normals fp32 [(1,)3,H,W] (depth_normals with axes (1, 1, 1)) rendered at
    ref_pose, from init_pose (both host [4,4]) and init_nodes fp64 [1,1,1,2] (exactly when affine)
    (include/omnidata_b200.h odb_track_frame).  With photometric > 0: also rgb fp32 [3,H,W] (the frame's image),
    ref_rgb fp32 [3,H,W] (the model's colour at ref_pose), the scratch ref_intensity fp32 [3,H,W], and record fp64
    [TRACK_RGBD_RECORD] (odb_track_frame_rgbd)."""
    name = "track_frame"
    _need(pred, torch.float32, "pred")
    if pred.dim() == 3 and pred.shape[0] == 1:
        pred = pred[0]
    if pred.dim() != 2 or not pred.is_contiguous():
        raise _capi.OdbError(f"{name}: pred must be a contiguous fp32 [H,W] or [1,H,W] tensor, got "
                             f"{tuple(pred.shape)}")
    h, w = pred.shape
    _check_planes(name, 1, h, w)
    _need_shape(ref_depth, (h, w), torch.float32, "ref_depth")
    _need(ref_normals, torch.float32, "ref_normals")
    if tuple(ref_normals.shape) not in ((3, h, w), (1, 3, h, w)) or not ref_normals.is_contiguous():
        raise _capi.OdbError(f"{name}: ref_normals must be a contiguous fp32 [3, {h}, {w}] tensor, got "
                             f"{tuple(ref_normals.shape)}")
    fx, fy, cx, cy = check_intrinsics(name, intrinsics)
    poses = []
    for what, T in (("ref_pose", ref_pose), ("init_pose", init_pose)):
        T = check_poses(f"{name} {what}", T)
        if T.shape[0] != 1:
            raise _capi.OdbError(f"{name}: {what} must be one [4,4] pose, got {T.shape[0]}")
        poses.append(T)
    check_track_params(name, affine, iterations, tol, robust, max_dist, min_overlap)
    if affine != (init_nodes is not None):
        raise _capi.OdbError(f"{name}: init_nodes is required exactly when affine (the initial scale and shift)")
    if init_nodes is not None:
        _need_shape(init_nodes, (1, 1, 1, 2), torch.float64, "init_nodes")
    _check_workspace(name, workspace, track_workspace_bytes(h, w))
    _need_shape(pose, (4, 4), torch.float64, "pose")
    _need_shape(nodes, (1, 1, 1, 2), torch.float64, "nodes")
    check_photometric(name, photometric, photometric_robust)
    photo = photometric > 0
    if any((t is None) == photo for t in (rgb, ref_rgb, ref_intensity)):
        raise _capi.OdbError(f"{name}: rgb, ref_rgb and ref_intensity are required exactly when photometric > 0")
    _need_shape(record, (_capi.TRACK_RGBD_RECORD if photo else _capi.TRACK_RECORD,), torch.float64, "record")
    if photo:
        for what, t in (("rgb", rgb), ("ref_rgb", ref_rgb), ("ref_intensity", ref_intensity)):
            _need_shape(t, (3, h, w), torch.float32, what)
        _call("track_frame_rgbd", {"bytes": 44 * h * w * iterations}, lib().odb_track_frame_rgbd,
              _same_device(pred, rgb, ref_depth, ref_rgb, ref_normals, ref_intensity, init_nodes, workspace, pose,
                           nodes, record), pred.data_ptr(), rgb.data_ptr(), ref_depth.data_ptr(), ref_rgb.data_ptr(),
              ref_normals.data_ptr(), ref_intensity.data_ptr(), h, w, fx, fy, cx, cy, poses[0].ctypes.data,
              poses[1].ctypes.data, _ptr(init_nodes), 1 if affine else 0, int(iterations), float(tol), float(robust),
              float(max_dist), float(min_overlap), float(photometric), float(photometric_robust),
              workspace.data_ptr(), pose.data_ptr(), nodes.data_ptr(), record.data_ptr())
        return
    _call(name, {"bytes": 20 * h * w * iterations}, lib().odb_track_frame,
          _same_device(pred, ref_depth, ref_normals, init_nodes, workspace, pose, nodes, record), pred.data_ptr(),
          ref_depth.data_ptr(), ref_normals.data_ptr(), h, w, fx, fy, cx, cy, poses[0].ctypes.data,
          poses[1].ctypes.data, _ptr(init_nodes), 1 if affine else 0, int(iterations), float(tol), float(robust),
          float(max_dist), float(min_overlap), workspace.data_ptr(), pose.data_ptr(), nodes.data_ptr(),
          record.data_ptr())


def track_information(workspace, h: int, w: int, unknowns: int, info):
    """info fp64 [n,n] (n = unknowns, 6 or 8) = the normal matrix of the last step of the last track_frame call on
    workspace at h x w (include/omnidata_b200.h odb_track_information)."""
    name = "track_information"
    if unknowns not in (6, 8):
        raise _capi.OdbError(f"{name}: unknowns must be 6 or 8, got {unknowns!r}")
    _check_workspace(name, workspace, track_workspace_bytes(h, w))
    _need_shape(info, (unknowns, unknowns), torch.float64, "info")
    _call(name, {"bytes": 8 * unknowns * unknowns}, lib().odb_track_information, _same_device(workspace, info),
          workspace.data_ptr(), h, w, unknowns, info.data_ptr())


# ---------------------------------------------------------------- pose graphs (csrc/posegraph.cu)
POSEGRAPH_MAX_ITERATIONS = 100


def check_posegraph_sizes(name: str, n_nodes: int, n_edges: int):
    """OdbError unless 2 <= n_nodes <= POSEGRAPH_MAX_NODES and 1 <= n_edges <= 8 n_nodes."""
    if not 2 <= n_nodes <= _capi.POSEGRAPH_MAX_NODES or not 1 <= n_edges <= 8 * n_nodes:
        raise _capi.OdbError(f"{name}: need 2 <= N <= {_capi.POSEGRAPH_MAX_NODES} nodes and 1 <= E <= 8 N edges, got "
                             f"N = {n_nodes}, E = {n_edges}")


def posegraph_workspace_bytes(n_nodes: int, n_edges: int) -> int:
    check_posegraph_sizes("posegraph_workspace_bytes", n_nodes, n_edges)
    return int(lib().odb_posegraph_workspace_bytes(n_nodes, n_edges))


def check_posegraph(name: str, poses, edges, measurements, information):
    """Host (poses float64 [N,16], edges int32 [E,2], measurements float64 [E,16], information float64 [E,36]) from
    numpy or CPU tensors; OdbError unless the poses pass check_poses, every edge (i, j) has 0 <= i, j < N and i != j,
    every measurement is rigid (check_poses) and every information matrix is a finite symmetric 6 x 6 matrix."""
    T = check_poses(f"{name} poses", poses)
    n = T.shape[0]
    E = np.asarray(edges.numpy() if isinstance(edges, torch.Tensor) else edges)
    if E.ndim != 2 or E.shape[1] != 2 or not np.issubdtype(E.dtype, np.integer):
        raise _capi.OdbError(f"{name}: edges must be an integer [E,2] array, got {E.dtype} {E.shape}")
    check_posegraph_sizes(name, n, E.shape[0])
    if (E < 0).any() or (E >= n).any():
        raise _capi.OdbError(f"{name}: an edge index lies outside [0, {n})")
    if (E[:, 0] == E[:, 1]).any():
        raise _capi.OdbError(f"{name}: an edge joins a node to itself")
    Z = check_poses(f"{name} measurements", measurements)
    W = np.asarray(information.numpy() if isinstance(information, torch.Tensor) else information, np.float64)
    if Z.shape[0] != E.shape[0] or W.shape != (E.shape[0], 6, 6):
        raise _capi.OdbError(f"{name}: need [{E.shape[0]},4,4] measurements and [{E.shape[0]},6,6] information "
                             f"matrices, got {Z.shape[0]} and {W.shape}")
    if not np.isfinite(W).all():
        raise _capi.OdbError(f"{name}: information matrices must be finite")
    if not (W == W.transpose(0, 2, 1)).all():
        raise _capi.OdbError(f"{name}: information matrices must be symmetric")
    return T, np.ascontiguousarray(E, np.int32), Z, np.ascontiguousarray(W.reshape(-1, 36))


def posegraph_optimize(edges, poses, measurements, information, iterations: int, tol: float, workspace, poses_out,
                       record):
    """poses_out fp64 [N,4,4] and record fp64 [POSEGRAPH_RECORD] of the pose graph of device edges int32 [E,2], poses
    fp64 [N,4,4], measurements fp64 [E,4,4] and information fp64 [E,6,6], checked on the host by check_posegraph
    (include/omnidata_b200.h odb_posegraph_optimize)."""
    name = "posegraph_optimize"
    _need(edges, torch.int32, "edges")
    n, e = poses.shape[0], edges.shape[0]
    check_posegraph_sizes(name, n, e)
    _need_shape(edges, (e, 2), torch.int32, "edges")
    _need_shape(poses, (n, 4, 4), torch.float64, "poses")
    _need_shape(measurements, (e, 4, 4), torch.float64, "measurements")
    _need_shape(information, (e, 6, 6), torch.float64, "information")
    if isinstance(iterations, bool) or not isinstance(iterations, (int, np.integer)) or \
            not 1 <= iterations <= POSEGRAPH_MAX_ITERATIONS:
        raise _capi.OdbError(f"{name}: iterations must be an integer in [1, {POSEGRAPH_MAX_ITERATIONS}], got "
                             f"{iterations!r}")
    if isinstance(tol, bool) or not (isinstance(tol, numbers.Real) and math.isfinite(tol) and tol > 0):
        raise _capi.OdbError(f"{name}: tol must be finite and > 0, got {tol!r}")
    _check_workspace(name, workspace, posegraph_workspace_bytes(n, e))
    _need_shape(poses_out, (n, 4, 4), torch.float64, "poses_out")
    _need_shape(record, (_capi.POSEGRAPH_RECORD,), torch.float64, "record")
    m = 6 * (n - 1)
    _call(name, {"flops": iterations * m ** 3 / 3}, lib().odb_posegraph_optimize,
          _same_device(edges, poses, measurements, information, workspace, poses_out, record), n, e,
          edges.data_ptr(), poses.data_ptr(), measurements.data_ptr(), information.data_ptr(), int(iterations),
          float(tol), workspace.data_ptr(), poses_out.data_ptr(), record.data_ptr())


# ---------------------------------------------------------------- place recognition (csrc/places.cu)
def _check_fern_count(name: str, n_ferns):
    if isinstance(n_ferns, bool) or not isinstance(n_ferns, (int, np.integer)) or \
            not 1 <= n_ferns <= _capi.FERN_MAX_FERNS:
        raise _capi.OdbError(f"{name}: the number of ferns must be an integer in [1, {_capi.FERN_MAX_FERNS}], got "
                             f"{n_ferns!r}")


def check_fern_frames(name: str, n: int, h: int, w: int):
    """OdbError unless 1 <= n <= 65535 frames of h x w with FERN_GRID <= (h, w) <= 65535."""
    _check_planes(name, n, h, w)
    if h < _capi.FERN_GRID[0] or w < _capi.FERN_GRID[1]:
        raise _capi.OdbError(f"{name}: frames must be at least {_capi.FERN_GRID[0]}x{_capi.FERN_GRID[1]} (the "
                             f"thumbnail grid), got {h}x{w}")


def fern_encode_workspace_bytes(n: int) -> int:
    _check_planes("fern_encode_workspace_bytes", n, 1, 1)
    return int(lib().odb_fern_encode_workspace_bytes(n))


def fern_encode(depth, rgb, fern_cells, fern_thresholds, codes, workspace):
    """codes uint8 [n,F] of depth fp32 [n,H,W] and rgb fp32 [n,3,H,W] under the fern table fern_cells int32 [F] and
    fern_thresholds fp64 [F,4] (include/omnidata_b200.h odb_fern_encode).  Contiguous tensors on one device."""
    name = "fern_encode"
    _need(depth, torch.float32, "depth")
    if depth.dim() != 3:
        raise _capi.OdbError(f"{name}: depth must be [n,H,W], got {tuple(depth.shape)}")
    n, h, w = depth.shape
    check_fern_frames(name, n, h, w)
    f = fern_cells.shape[0] if fern_cells.dim() == 1 else -1
    _check_fern_count(name, f)
    _need_shape(rgb, (n, 3, h, w), torch.float32, "rgb")
    _need_shape(fern_cells, (f,), torch.int32, "fern_cells")
    _need_shape(fern_thresholds, (f, 4), torch.float64, "fern_thresholds")
    _need_shape(codes, (n, f), torch.uint8, "codes")
    if not depth.is_contiguous():
        raise _capi.OdbError(f"{name}: depth must be contiguous")
    _check_workspace(name, workspace, fern_encode_workspace_bytes(n))
    _call(name, {"bytes": 16 * n * h * w}, lib().odb_fern_encode,
          _same_device(depth, rgb, fern_cells, fern_thresholds, codes, workspace), n, h, w, depth.data_ptr(),
          rgb.data_ptr(), f, fern_cells.data_ptr(), fern_thresholds.data_ptr(), codes.data_ptr(), workspace.data_ptr())


def fern_query_workspace_bytes(n_db: int) -> int:
    if isinstance(n_db, bool) or not isinstance(n_db, (int, np.integer)) or not 1 <= n_db <= _capi.FERN_MAX_ENTRIES:
        raise _capi.OdbError(f"fern_query_workspace_bytes: need 1 <= n_db <= {_capi.FERN_MAX_ENTRIES}, got {n_db!r}")
    return int(lib().odb_fern_query_workspace_bytes(int(n_db)))


def fern_query(db_codes, code, limit: int, k: int, out_index, out_distance, workspace):
    """out_index and out_distance int32 [k]: the k entries i < limit of db_codes uint8 [n_db,F] nearest to code uint8
    [F] in the number of differing ferns, in (distance, index) order, padded with -1 (include/omnidata_b200.h
    odb_fern_query)."""
    name = "fern_query"
    _need(db_codes, torch.uint8, "db_codes")
    if db_codes.dim() != 2 or not db_codes.is_contiguous():
        raise _capi.OdbError(f"{name}: db_codes must be a contiguous [n_db,F] array, got {tuple(db_codes.shape)}")
    n_db, f = db_codes.shape
    _check_fern_count(name, f)
    ws_bytes = fern_query_workspace_bytes(n_db)
    _need_shape(code, (f,), torch.uint8, "code")
    for what, v, lo, hi in (("limit", limit, 0, n_db), ("k", k, 1, _capi.FERN_MAX_K)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= v <= hi:
            raise _capi.OdbError(f"{name}: {what} must be an integer in [{lo}, {hi}], got {v!r}")
    _need_shape(out_index, (k,), torch.int32, "out_index")
    _need_shape(out_distance, (k,), torch.int32, "out_distance")
    _check_workspace(name, workspace, ws_bytes)
    _call(name, {"bytes": int(limit) * f}, lib().odb_fern_query,
          _same_device(db_codes, code, out_index, out_distance, workspace), n_db, f, db_codes.data_ptr(),
          code.data_ptr(), int(limit), int(k), out_index.data_ptr(), out_distance.data_ptr(), workspace.data_ptr())


# ---------------------------------------------------------------- mesh metrics (csrc/mesh_metrics.cu)
def check_points(name: str, t, what: str = "points") -> int:
    """The point count of a contiguous fp32 [N,3] CUDA tensor; OdbError otherwise or beyond MESH_MAX_POINTS."""
    _need(t, torch.float32, what)
    if t.dim() != 2 or t.shape[1] != 3 or not t.is_contiguous():
        raise _capi.OdbError(f"{name}: {what} must be a contiguous fp32 [N,3] tensor, got {tuple(t.shape)}")
    if t.shape[0] > _capi.MESH_MAX_POINTS:
        raise _capi.OdbError(f"{name}: {t.shape[0]} {what}, at most {_capi.MESH_MAX_POINTS}")
    return int(t.shape[0])


def check_mesh(name: str, vertices, faces) -> Tuple[int, int]:
    """(V, F) of vertices fp32 [V,3] and faces int32 [F,3] (contiguous, on one CUDA device)."""
    _need(vertices, torch.float32, "vertices")
    _need(faces, torch.int32, "faces")
    for t, n in ((vertices, "vertices"), (faces, "faces")):
        if t.dim() != 2 or t.shape[1] != 3 or not t.is_contiguous():
            raise _capi.OdbError(f"{name}: {n} must be a contiguous [N,3] tensor, got {tuple(t.shape)}")
        if t.shape[0] >= 2 ** 31:
            raise _capi.OdbError(f"{name}: {t.shape[0]} {n}, at most 2^31 - 1")
    _same_device(vertices, faces)
    return int(vertices.shape[0]), int(faces.shape[0])


def _check_seed(name: str, seed: int, stream: int):
    if not (isinstance(seed, numbers.Integral) and isinstance(stream, numbers.Integral) and 0 <= seed < 2 ** 63 and
            0 <= stream < 2 ** 63):
        raise _capi.OdbError(f"{name}: seed and stream must be integers in [0, 2^63), got {seed!r}, {stream!r}")


def mesh_sample_workspace_bytes(nf: int) -> int:
    return int(lib().odb_mesh_sample_workspace_bytes(nf))


def mesh_sample_count(vertices, faces, density: float, seed: int, stream: int, workspace, info):
    """info int64 [2] = (samples, flags) of the surface sampling of the mesh; fills workspace for mesh_sample_emit
    (include/omnidata_b200.h odb_mesh_sample_count)."""
    name = "mesh_sample_count"
    nv, nf = check_mesh(name, vertices, faces)
    if not (math.isfinite(density) and density > 0):
        raise _capi.OdbError(f"{name}: density must be finite and > 0, got {density}")
    _check_seed(name, seed, stream)
    _check_workspace(name, workspace, mesh_sample_workspace_bytes(nf))
    _need_shape(info, (2,), torch.int64, "info")
    _call(name, {"bytes": 48 * nf}, lib().odb_mesh_sample_count, _same_device(vertices, faces, workspace, info),
          vertices.data_ptr(), nv, faces.data_ptr(), nf, float(density), int(seed), int(stream), workspace.data_ptr(),
          info.data_ptr())


def mesh_sample_emit(vertices, faces, seed: int, stream: int, workspace, out):
    """out fp32 [N,3] = the samples counted by mesh_sample_count on the same workspace (N its total)."""
    name = "mesh_sample_emit"
    nv, nf = check_mesh(name, vertices, faces)
    _check_seed(name, seed, stream)
    _check_workspace(name, workspace, mesh_sample_workspace_bytes(nf))
    n = check_points(name, out, "out")
    _call(name, {"bytes": 12 * n}, lib().odb_mesh_sample_emit, _same_device(vertices, faces, workspace, out),
          vertices.data_ptr(), nv, faces.data_ptr(), nf, int(seed), int(stream), workspace.data_ptr(), n,
          out.data_ptr())


def nn_bounds(reference, query, box):
    """box int32 [7] = the reference set's order-preserving min / max keys and the non-finite flags
    (include/omnidata_b200.h odb_nn_bounds)."""
    name = "nn_bounds"
    nr, nq = check_points(name, reference, "reference"), check_points(name, query, "query")
    _need_shape(box, (7,), torch.int32, "box")
    _call(name, {"bytes": 12 * (nr + nq)}, lib().odb_nn_bounds, _same_device(reference, query, box),
          reference.data_ptr(), nr, query.data_ptr(), nq, box.data_ptr())


def nn_grid_cells(grid) -> int:
    """The number of cells of the grid (lo[3], hi[3], h): prod over axes of floor((hi - lo) / h) + 1."""
    return math.prod(int(math.floor((grid[3 + a] - grid[a]) / grid[6])) + 1 for a in range(3))


def _nn_grid(name: str, grid) -> np.ndarray:
    g = np.ascontiguousarray(grid, dtype=np.float64)
    if g.shape != (7,) or not np.isfinite(g).all() or not (g[6] > 0) or not (g[:3] <= g[3:6]).all() or \
            nn_grid_cells(g) > _capi.NN_MAX_CELLS:
        raise _capi.OdbError(f"{name}: grid must be finite (lo[3], hi[3], h) with lo <= hi, h > 0 and at most "
                             f"{_capi.NN_MAX_CELLS} cells, got {grid!r}")
    return g


def nn_workspace_bytes(n_ref: int, grid) -> int:
    g = _nn_grid("nn_workspace_bytes", grid)
    return int(lib().odb_nn_workspace_bytes(n_ref, g.ctypes.data))


def nn_build(reference, grid, workspace):
    """Sorts reference fp32 [N,3] into the uniform grid (lo[3], hi[3], h) (host) in workspace
    (include/omnidata_b200.h odb_nn_build)."""
    name = "nn_build"
    nr = check_points(name, reference, "reference")
    g = _nn_grid(name, grid)
    _check_workspace(name, workspace, nn_workspace_bytes(nr, g))
    _call(name, {"bytes": 40 * nr}, lib().odb_nn_build, _same_device(reference, workspace), reference.data_ptr(), nr,
          g.ctypes.data, workspace.data_ptr())


def nn_query(query, n_ref: int, grid, workspace, distance, index):
    """distance fp64 [M] and index int32 [M] of each query's nearest reference point, from nn_build's workspace and
    grid (include/omnidata_b200.h odb_nn_query); n_ref = 0 needs neither."""
    name = "nn_query"
    nq = check_points(name, query, "query")
    g = None
    if n_ref:
        g = _nn_grid(name, grid)
        _check_workspace(name, workspace, nn_workspace_bytes(n_ref, g))
    _need_shape(distance, (nq,), torch.float64, "distance")
    _need_shape(index, (nq,), torch.int32, "index")
    _call(name, {"bytes": 24 * nq}, lib().odb_nn_query, _same_device(query, workspace, distance, index),
          query.data_ptr(), nq, int(n_ref), None if g is None else g.ctypes.data, _ptr(workspace),
          distance.data_ptr(), index.data_ptr())


def frustum_mask(points, intrinsics, size: Tuple[int, int], poses, max_depth: float, mask):
    """mask uint8 [N] = 1 where one of the cameras poses (a DEVICE fp64 [n,16] tensor of checked camera-to-world
    matrices, see check_poses) sees the point (include/omnidata_b200.h odb_frustum_mask)."""
    name = "frustum_mask"
    n = check_points(name, points)
    fx, fy, cx, cy = check_intrinsics(name, intrinsics)
    h, w = (int(v) for v in size)
    _check_planes(name, 1, h, w)
    if not (math.isfinite(max_depth) and max_depth > 0):
        raise _capi.OdbError(f"{name}: max_depth must be finite and > 0, got {max_depth}")
    _need(poses, torch.float64, "poses")
    if poses.dim() != 2 or poses.shape[1] != 16 or poses.shape[0] < 1 or poses.shape[0] >= 2 ** 31 or \
            not poses.is_contiguous():
        raise _capi.OdbError(f"{name}: poses must be a contiguous fp64 [n,16] tensor, got {tuple(poses.shape)}")
    _need_shape(mask, (n,), torch.uint8, "mask")
    _call(name, {"bytes": 13 * n}, lib().odb_frustum_mask, _same_device(points, poses, mask), points.data_ptr(), n,
          poses.data_ptr(), int(poses.shape[0]), h, w, fx, fy, cx, cy, float(max_depth), mask.data_ptr())


def compact_workspace_bytes(n: int) -> int:
    return int(lib().odb_compact_workspace_bytes(n))


def compact_points(points, mask, workspace, out, count):
    """out fp32 [>= K,3] starts with the K points of points fp32 [N,3] where mask uint8 [N] != 0, in order; count int64
    [1] = K on the device (include/omnidata_b200.h odb_compact_points)."""
    name = "compact_points"
    n = check_points(name, points)
    _need_shape(mask, (n,), torch.uint8, "mask")
    _check_workspace(name, workspace, compact_workspace_bytes(n))
    _need(out, torch.float32, "out")
    if out.dim() != 2 or out.shape[1] != 3 or out.shape[0] < n or not out.is_contiguous():
        raise _capi.OdbError(f"{name}: out must be a contiguous fp32 [>= {n}, 3] tensor, got {tuple(out.shape)}")
    _need_shape(count, (1,), torch.int64, "count")
    _call(name, {"bytes": 29 * n}, lib().odb_compact_points, _same_device(points, mask, workspace, out, count),
          points.data_ptr(), mask.data_ptr(), n, workspace.data_ptr(), out.data_ptr(), count.data_ptr())


def check_thresholds(name: str, thresholds) -> np.ndarray:
    try:
        t = np.asarray([float(v) for v in thresholds], dtype=np.float64)
    except (TypeError, ValueError):
        raise _capi.OdbError(f"{name}: thresholds must be a sequence of numbers, got {thresholds!r}") from None
    if not 1 <= len(t) <= _capi.MESH_MAX_THRESHOLDS or not (np.isfinite(t) & (t > 0)).all():
        raise _capi.OdbError(f"{name}: 1 to {_capi.MESH_MAX_THRESHOLDS} finite thresholds > 0, got {thresholds!r}")
    return t


def mesh_metrics_workspace_bytes(n_pred: int, n_gt: int) -> int:
    return int(lib().odb_mesh_metrics_workspace_bytes(n_pred, n_gt))


def mesh_metrics_update(dist_pred, dist_gt, thresholds, pred_culled: int, gt_culled: int, workspace, record, sums,
                        counts):
    """Folds one scene (dist_pred fp64 [N_p], dist_gt fp64 [N_g]) into sums fp64 [15] and counts int64 [7]; record
    fp64 [MESH_RECORD] (include/omnidata_b200.h odb_mesh_metrics_update)."""
    name = "mesh_metrics_update"
    t = check_thresholds(name, thresholds)
    for d, n in ((dist_pred, "dist_pred"), (dist_gt, "dist_gt")):
        _need(d, torch.float64, n)
        if d.dim() != 1 or not d.is_contiguous():
            raise _capi.OdbError(f"{name}: {n} must be a contiguous fp64 [N] tensor, got {tuple(d.shape)}")
    n_p, n_g = int(dist_pred.shape[0]), int(dist_gt.shape[0])
    _check_workspace(name, workspace, mesh_metrics_workspace_bytes(n_p, n_g))
    _need_shape(record, (_capi.MESH_RECORD,), torch.float64, "record")
    _need_shape(sums, (3 + 3 * _capi.MESH_MAX_THRESHOLDS,), torch.float64, "sums")
    _need_shape(counts, (7,), torch.int64, "counts")
    _call(name, {"bytes": 8 * (n_p + n_g)}, lib().odb_mesh_metrics_update,
          _same_device(dist_pred, dist_gt, workspace, record, sums, counts), dist_pred.data_ptr(), n_p,
          dist_gt.data_ptr(), n_g, t.ctypes.data, len(t), int(pred_culled), int(gt_culled), workspace.data_ptr(),
          record.data_ptr(), sums.data_ptr(), counts.data_ptr())
