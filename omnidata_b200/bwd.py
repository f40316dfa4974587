"""Torch-tensor front end of the backward kernels (include/omnidata_b200.h, "Backward of the network").

Same conventions as ops.py: pointers + sizes cross the C ABI, everything is enqueued on the current stream of the
tensors' device, activations / activation gradients are channels-last bf16 (production) or fp32 (correctness mode).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import _capi
from ._capi import WgradDesc, lib
from .ops import TAPS_1, TAPS_3X3, _call, _dt, _need, _ptr, _same_device, _view4


class Scratch:
    """One growing byte buffer per device for kernel workspaces (split partials, slab sums)."""

    def __init__(self):
        self.buf: Optional[torch.Tensor] = None

    def get(self, nbytes: int, device) -> torch.Tensor:
        nbytes = max(int(nbytes), 256)
        if self.buf is None or self.buf.numel() < nbytes or self.buf.device != device:
            self.buf = torch.empty(nbytes + (nbytes >> 2), dtype=torch.uint8, device=device)
        return self.buf


_SCRATCH = Scratch()


def _scratch(nbytes: int, device) -> torch.Tensor:
    return _SCRATCH.get(nbytes, device)


def mask_add(out, b, a=None, mask=None):
    """out = a + b * [mask > 0]  (a, mask optional)."""
    for t in (a, mask, out):
        if t is not None and (t.dtype != b.dtype or t.numel() != b.numel() or not t.is_contiguous()):
            raise _capi.OdbError("mask_add: contiguous tensors of one dtype / size required")
    _call("odb_mask_add", {"bytes": b.element_size() * b.numel() * (2 + (a is not None) + (mask is not None))},
          lib().odb_mask_add, _same_device(a, b, mask, out), _ptr(a), b.data_ptr(), _ptr(mask), out.data_ptr(), b.numel(),
          _dt(b))


def gelu_fwd(u, y):
    _call("odb_gelu_fwd", {"bytes": 2 * u.element_size() * u.numel()}, lib().odb_gelu_fwd, _same_device(u, y), u.data_ptr(),
          y.data_ptr(), u.numel(), _dt(u))


def gelu_bwd(dy, u, du):
    _call("odb_gelu_bwd", {"bytes": 3 * u.element_size() * u.numel()}, lib().odb_gelu_bwd, _same_device(dy, u, du),
          dy.data_ptr(), u.data_ptr(), du.data_ptr(), u.numel(), _dt(u))


def colsum(x, out, accumulate: bool = False, batches: int = 1):
    """out[bt, n] (+)= sum over the rows of x viewed as [batches, rows, n] (last dim contiguous, uniform row stride)."""
    _need(out, torch.float32, "out")
    n = x.shape[-1]
    if x.dim() == 2:
        rows, row_stride, batch_stride = x.shape[0] // batches, x.stride(0), (x.shape[0] // batches) * x.stride(0)
    elif x.dim() == 3:
        if batches != x.shape[0]:
            raise _capi.OdbError("colsum: batches must equal x.shape[0] for a 3-D input")
        rows, row_stride, batch_stride = x.shape[1], x.stride(1), x.stride(0)
    else:
        x = x.reshape(-1, n)
        rows, row_stride, batch_stride = x.shape[0] // batches, n, (x.shape[0] // batches) * n
    if x.stride(-1) != 1:
        raise _capi.OdbError("colsum: unit stride in the last dim required")
    ws = _scratch(lib().odb_colsum_workspace_bytes(batches, rows, n), x.device)
    _call("odb_colsum", {"bytes": x.element_size() * batches * rows * n}, lib().odb_colsum, _same_device(x, out), x.data_ptr(),
          out.data_ptr(), ws.data_ptr(), batches, rows, n, row_stride, batch_stride, 1 if accumulate else 0, _dt(x))


def layernorm_bwd(dy, x, gamma, ds_in, ds_out, ds_copy, dgamma, dbeta, eps: float = 1e-6, accumulate: bool = False,
                  dcolsum=None):
    """`dcolsum` (fp32 [cols], optional): column sums of ds_out, i.e. the bias gradient of the linear layer whose output
    gradient ds_out is — saves a separate pass over the fp32 stream.  dgamma = dbeta = None: a frozen norm (no affine
    gradients)."""
    _need(x, torch.float32, "x"); _need(ds_out, torch.float32, "ds_out")
    if dcolsum is not None:
        _need(dcolsum, torch.float32, "dcolsum")
    rows, cols = x.numel() // x.shape[-1], x.shape[-1]
    ws = _scratch(lib().odb_layernorm_bwd_workspace_bytes(cols), x.device)
    _call("odb_layernorm_bwd", {"bytes": x.numel() * (8 + dy.element_size() * 2)}, lib().odb_layernorm_bwd,
          _same_device(dy, x, gamma, ds_in, ds_out, ds_copy, dgamma, dbeta, dcolsum), dy.data_ptr(), x.data_ptr(),
          gamma.data_ptr(), _ptr(ds_in), ds_out.data_ptr(), _ptr(ds_copy), _ptr(dgamma), _ptr(dbeta), _ptr(dcolsum),
          ws.data_ptr(), rows, cols, eps,
          1 if accumulate else 0, _dt(dy))


def groupnorm_bwd(dy, x, stats, gamma, dx, dgamma, dbeta, mask=None, groups: int = 32, accumulate: bool = False):
    """dgamma = dbeta = None: dx only (a frozen norm)."""
    b, c = x.shape[0], x.shape[-1]
    hw = x.numel() // (b * c)
    need = lib().odb_groupnorm_bwd_workspace_bytes(b, hw, c, groups)
    if need < 0:
        raise _capi.OdbError("groupnorm_bwd: unsupported shape")
    ws = _scratch(need, x.device)
    _call("odb_groupnorm_bwd", {"bytes": x.element_size() * x.numel() * (5 + 2 * (mask is not None))}, lib().odb_groupnorm_bwd,
          _same_device(dy, mask, x, stats, gamma, dx, dgamma, dbeta), dy.data_ptr(), _ptr(mask), x.data_ptr(), stats.data_ptr(),
          gamma.data_ptr(), dx.data_ptr(), _ptr(dgamma), _ptr(dbeta), ws.data_ptr(), b, hw, c, groups,
          1 if accumulate else 0, _dt(x))


def upsample2x_bwd(dout, dz):
    b, h, w, c = dz.shape
    _call("odb_upsample2x_bwd", {"bytes": dout.element_size() * (dout.numel() + dz.numel())}, lib().odb_upsample2x_bwd,
          _same_device(dout, dz), dout.data_ptr(), dz.data_ptr(), b, h, w, c, _dt(dz))


def stem_pool_bwd(dt, s0, stats, gamma, beta, g_s0, groups: int = 32):
    b, h, w, c = s0.shape
    _call("odb_stem_pool_bwd", {}, lib().odb_stem_pool_bwd, _same_device(dt, s0, stats, gamma, beta, g_s0), dt.data_ptr(),
          s0.data_ptr(), stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), g_s0.data_ptr(), b, h, w, c, groups, _dt(s0))


def stem_input_grad(ds0, w, dx):
    """dx fp32 [B,3,H,W] = gradient w.r.t. the image of the 7x7 stride-2 TF-SAME stem convolution, from ds0 [B,H/2,W/2,64]
    (gradient w.r.t. its output) and w [64, kpad] (the packed operand the forward used, same dtype as ds0)."""
    _need(dx, torch.float32, "dx")
    if ds0.dim() != 4 or ds0.shape[-1] != 64 or not ds0.is_contiguous():
        raise _capi.OdbError("stem_input_grad: ds0 must be a contiguous [B,H/2,W/2,64] tensor")
    if w.dim() != 2 or w.shape[0] != 64 or w.dtype != ds0.dtype or not w.is_contiguous():
        raise _capi.OdbError("stem_input_grad: w must be a contiguous [64, kpad] tensor of ds0's dtype")
    b, h2, w2, _ = ds0.shape
    if tuple(dx.shape) != (b, 3, 2 * h2, 2 * w2) or not dx.is_contiguous():
        raise _capi.OdbError(f"stem_input_grad: dx must be a contiguous [{b},3,{2 * h2},{2 * w2}] tensor")
    info = {"flops": 2.0 * b * h2 * w2 * 64 * 147, "bytes": ds0.numel() * ds0.element_size() + dx.numel() * 4}
    _call("odb_stem_input_grad", info, lib().odb_stem_input_grad, _same_device(ds0, w, dx), ds0.data_ptr(), w.data_ptr(),
          dx.data_ptr(), b, 2 * h2, 2 * w2, w.shape[1], _dt(ds0))


def patch_input_grad(dcols, dx, patch: int = 16):
    """dx fp32 [B,3,H,W] = gradient w.r.t. the image of the plain-ViT patch embedding (the adjoint of ops.patchify), from
    dcols [B*(H/patch)*(W/patch), 3*patch*patch], the gradient w.r.t. the patch columns."""
    _need(dx, torch.float32, "dx")
    b, c, h, w = dx.shape
    if c != 3 or not dx.is_contiguous():
        raise _capi.OdbError("patch_input_grad: dx must be a contiguous [B,3,H,W] tensor")
    if (not dcols.is_contiguous() or h % patch or w % patch
            or dcols.numel() != b * (h // patch) * (w // patch) * 3 * patch * patch):
        raise _capi.OdbError(f"patch_input_grad: dcols must be a contiguous [{b}*(H/{patch})*(W/{patch}), "
                             f"{3 * patch * patch}] tensor")
    info = {"bytes": dcols.numel() * dcols.element_size() + dx.numel() * 4}
    _call("odb_patch_input_grad", info, lib().odb_patch_input_grad, _same_device(dcols, dx), dcols.data_ptr(),
          dx.data_ptr(), b, h, w, patch, _dt(dcols))


def pos_embed_resize_bwd(dgrid, gh: int, gw: int, dpos):
    """dpos fp32 [24*24, D] = gradient of the 24 x 24 position-embedding grid through its bilinear resize to gh x gw
    (F.interpolate(mode="bilinear", align_corners=False)), from dgrid fp32 [gh*gw, D], the gradient at the resized rows."""
    _need(dgrid, torch.float32, "dgrid")
    _need(dpos, torch.float32, "dpos")
    d = dgrid.shape[-1]
    if dgrid.numel() != gh * gw * d or not dgrid.is_contiguous():
        raise _capi.OdbError(f"pos_embed_resize_bwd: dgrid must be a contiguous [{gh}*{gw}, D] tensor")
    if dpos.numel() != 24 * 24 * d or not dpos.is_contiguous():
        raise _capi.OdbError(f"pos_embed_resize_bwd: dpos must be a contiguous [24*24, {d}] tensor")
    _call("odb_pos_embed_resize_bwd", {"bytes": 4 * (dgrid.numel() + dpos.numel())}, lib().odb_pos_embed_resize_bwd,
          _same_device(dgrid, dpos), dgrid.data_ptr(), dpos.data_ptr(), gh, gw, d)


def head_tail_fwd(a, w, bias, out, relu: bool):
    b, h, wd, cs = a.shape
    _call("odb_head_tail_fwd", {}, lib().odb_head_tail_fwd, _same_device(a, w, bias, out), a.data_ptr(), cs, w.data_ptr(),
          bias.data_ptr(), out.data_ptr(), b, h, wd, w.shape[0], 1 if relu else 0, _dt(a))


def head_tail_bwd(dout, out, a, w, da, dw, dbias, relu: bool, accumulate: bool = False):
    """dw = dbias = None: da only (a frozen head tail)."""
    b, h, wd, cs = a.shape
    ws = _scratch(lib().odb_head_tail_bwd_workspace_bytes(w.shape[0]), a.device)
    _call("odb_head_tail_bwd", {}, lib().odb_head_tail_bwd, _same_device(dout, out, a, w, da, dw, dbias), dout.data_ptr(),
          out.data_ptr(), a.data_ptr(), cs, w.data_ptr(), da.data_ptr(), _ptr(dw), _ptr(dbias), ws.data_ptr(), b, h,
          wd, w.shape[0], 1 if relu else 0, 1 if accumulate else 0, _dt(a))


def add_cast(ds_in, g, ds_out, copy=None):
    """ds_out (fp32) = ds_in (fp32 or None) + g; optional copy in g's dtype."""
    _need(ds_out, torch.float32, "ds_out")
    _call("odb_add_cast", {}, lib().odb_add_cast, _same_device(ds_in, g, ds_out, copy), _ptr(ds_in), g.data_ptr(),
          ds_out.data_ptr(), _ptr(copy), g.numel(), _dt(g))


def pack_weight(w, fwd, bwd, n: int, c: int, taps: int, n_pad: int, c_pad: int, standardize: bool, eps: float = 1e-8):
    """w fp32 [n][c][taps] -> fwd [n_pad][taps*c_pad] and bwd [c_pad][taps*n_pad] (either may be None)."""
    _need(w, torch.float32, "w")
    ref = fwd if fwd is not None else bwd
    _call("odb_pack_weight", {}, lib().odb_pack_weight, _same_device(w, fwd, bwd), w.data_ptr(), _ptr(fwd), _ptr(bwd), n, c,
          taps, n_pad, c_pad, 1 if standardize else 0, eps, _dt(ref))


def unpack_wgrad(gp, w, dw, n: int, c: int, taps: int, c_pad: int, standardize: bool, eps: float = 1e-8):
    _call("odb_unpack_wgrad", {}, lib().odb_unpack_wgrad, _same_device(gp, w, dw), gp.data_ptr(), _ptr(w), dw.data_ptr(), n, c,
          taps, c_pad, 1 if standardize else 0, eps)


def _item_table(items, device) -> torch.Tensor:
    """ctypes records -> one device byte tensor (the multi-tensor kernels' tables)."""
    import numpy as np
    raw = b"".join(bytes(it) for it in items)
    return torch.from_numpy(np.frombuffer(raw, dtype=np.uint8).copy()).to(device)


class PackTable:
    """One-launch weight packing of a fixed set of layers (pointers are captured: the buffers must stay alive)."""

    def __init__(self, layers, dtype):
        """layers: (w fp32 [n][c][taps], fwd, bwd, n, c, taps, n_pad, c_pad, standardize)."""
        items, rows, tiles = [], 0, 0
        keep = []
        for w, fwd, bwd_, n, c, taps, n_pad, c_pad, std in layers:
            items.append(_capi.PackItem(w.data_ptr(), fwd.data_ptr(), bwd_.data_ptr(), n, c, taps, n_pad, c_pad, 1 if std else 0,
                                        rows, tiles))
            rows += n_pad
            tiles += ((n_pad + 63) // 64) * ((c_pad + 63) // 64) * taps           # kPackTile (bwd_ops.cu)
            keep += [w, fwd, bwd_]
        self.keep, self.n, self.rows, self.tiles = keep, len(items), rows, tiles
        self.table = _item_table(items, layers[0][0].device)
        self.dtype = _capi.DTYPE_F32 if dtype == torch.float32 else _capi.DTYPE_BF16
        self.device = layers[0][0].device

    def run(self, eps: float = 1e-8):
        _call("odb_pack_weights_multi", {}, lib().odb_pack_weights_multi, self.device, self.table.data_ptr(), self.n, self.rows,
              self.tiles, eps, self.dtype)


class UnpackTable:
    """One-launch conversion of packed-layout weight gradients into parameter layout (+ weight-standardisation backward)."""

    def __init__(self, layers):
        """layers: (gp fp32 [n_pad][taps*c_pad], w fp32 param, dw fp32 grad, n, c, taps, c_pad, standardize)."""
        items, rows, mx, keep = [], 0, 1, []
        for gp, w, dw, n, c, taps, c_pad, std in layers:
            items.append(_capi.UnpackItem(gp.data_ptr(), w.data_ptr(), dw.data_ptr(), n, c, taps, c_pad, 1 if std else 0, rows, 0, 0))
            rows += n
            mx = max(mx, taps * c_pad)
            keep += [gp, w, dw]
        self.keep, self.n, self.rows, self.max_row = keep, len(items), rows, mx
        self.device = layers[0][0].device
        self.table = _item_table(items, self.device)

    def run(self, eps: float = 1e-8):
        _call("odb_unpack_wgrads_multi", {}, lib().odb_unpack_wgrads_multi, self.device, self.table.data_ptr(), self.n, self.rows,
              self.max_row, eps)


def conv_wgrad(views: Sequence[torch.Tensor], taps: Sequence[Tuple[int, int, int]], dy: torch.Tensor, out: torch.Tensor,
               accumulate: bool = False):
    """out fp32 [n][len(taps) * C] (+)= sum_pixels dy[pixel, n] * view_t[pixel + offset_t, c]."""
    _need(out, torch.float32, "out")
    d = WgradDesc()
    dt = views[0].dtype
    d.num_views = len(views)
    for i, v in enumerate(views):
        d.views[i] = _view4(v, f"view{i}", dt)
    d.num_taps = len(taps)
    for i, (vi, dx, dy_) in enumerate(taps):
        d.tap_view[i], d.tap_dx[i], d.tap_dy[i] = vi, dx, dy_
    d.dy = _view4(dy, "dy", dt)
    d.n = d.dy.c
    if out.numel() != d.n * len(taps) * d.views[0].c or not out.is_contiguous():
        raise _capi.OdbError("conv_wgrad: out must be contiguous [n][taps*C]")
    d.out = out.data_ptr()
    d.accumulate = 1 if accumulate else 0
    d.dtype = _dt(views[0])
    need = lib().odb_conv_wgrad_workspace_bytes(C.byref(d))
    if need < 0:
        raise _capi.OdbError("conv_wgrad: bad descriptor")
    ws = _scratch(need, dy.device)
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    rows = d.dy.w * d.dy.h * d.dy.b
    info = {"m": d.n, "n": len(taps) * d.views[0].c, "k": rows, "wgrad": True, "f32": d.dtype == _capi.DTYPE_F32}
    _call("odb_conv_wgrad", info, lib().odb_conv_wgrad, _same_device(*views, dy, out), C.byref(d))


def attention_bwd(qkv, o, d_o, lse, dqkv, heads: int = 12, scale: float = 0.125):
    """dqkv [b, T, 3*heads*64] = gradient w.r.t. qkv of o = attention(qkv), from d_o; lse fp32 [b, heads, T] (bf16 only):
    the log2-sum-exp ops.attention wrote.  The kernels address every tensor from (b, T, heads) alone, so the shapes
    are checked here."""
    if qkv.dim() != 3 or qkv.shape[-1] != 3 * heads * 64 or not qkv.is_contiguous():
        raise _capi.OdbError(f"attention_bwd: qkv must be a contiguous [b, T, {3 * heads * 64}] tensor")
    b, n, c3 = qkv.shape
    if n > 640:
        raise _capi.OdbError(f"attention_bwd: at most 640 tokens, got {n}")
    _dt(qkv)
    for name, t, shape in (("o", o, (b, n, heads * 64)), ("d_o", d_o, (b, n, heads * 64)), ("dqkv", dqkv, (b, n, c3))):
        if tuple(t.shape) != shape or t.dtype != qkv.dtype or not t.is_contiguous():
            raise _capi.OdbError(f"attention_bwd: {name} must be a contiguous {list(shape)} tensor of qkv's dtype")
    if qkv.dtype == torch.bfloat16:
        if lse is None or tuple(lse.shape) != (b, heads, n) or lse.dtype != torch.float32 or not lse.is_contiguous():
            raise _capi.OdbError(f"attention_bwd: lse must be a contiguous fp32 [{b}, {heads}, {n}] tensor")
    need = lib().odb_attention_bwd_workspace_bytes(b, n, heads, _dt(qkv))
    ws = _scratch(need, qkv.device)
    info = {"flops": 10.0 * b * heads * n * n * 64}
    _call("odb_attention_bwd", info, lib().odb_attention_bwd, _same_device(qkv, o, d_o, lse, dqkv), qkv.data_ptr(),
          o.data_ptr(), d_o.data_ptr(), _ptr(lse), dqkv.data_ptr(), ws.data_ptr(), ws.numel(), b, n, heads, scale, _dt(qkv))


__all__ = ["mask_add", "gelu_fwd", "gelu_bwd", "colsum", "layernorm_bwd", "groupnorm_bwd", "upsample2x_bwd", "stem_pool_bwd",
           "stem_input_grad", "patch_input_grad", "pos_embed_resize_bwd", "head_tail_fwd", "head_tail_bwd", "add_cast", "pack_weight", "unpack_wgrad", "conv_wgrad", "attention_bwd",
           "TAPS_1", "TAPS_3X3"]
