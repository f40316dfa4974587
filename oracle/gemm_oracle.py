"""Float64 restatement of the GEMM-shaped operations the forward and the backward of the DPTs launch: the implicit-GEMM
convolution (odb_conv_gemm with its epilogues: bias, activation, residual, out2 copy, fused GroupNorm statistics and
head tail; it also computes every input gradient), the attention (odb_attention, with its log-sum-exp), the weight
gradient (odb_conv_wgrad) and the attention backward (odb_attention_bwd).  Plain torch on any device; each function
follows the definition in
include/omnidata_b200.h, with views and taps exactly as the kernels take them:
  * a view is a channels-last [B, H, W, C] tensor, or [rows, C] meaning B = H = 1 (as ops._view4);
  * a tap (v, dx, dy) reads view v at (y + dy, x + dx), zero outside the view;
  * a packed weight is [N, taps * C], tap-major / channel-minor.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

# the attention kernels' exponent factor: fp32(0.125 * fp32(log2 e)), exact since 0.125 is a power of two
_LOG2E_F32 = float(torch.tensor(1.4426950408889634, dtype=torch.float32))


def as4(t: torch.Tensor) -> torch.Tensor:
    """[rows, C] -> [1, 1, rows, C]; a 4-D view is returned as is."""
    return t.unsqueeze(0).unsqueeze(0) if t.dim() == 2 else t


def _shifted(v: torch.Tensor, dx: int, dy: int, oh: int, ow: int) -> torch.Tensor:
    """v [B, H, W, C] read at (y + dy, x + dx) for y < oh, x < ow, zero outside v."""
    b, h, w, c = v.shape
    out = v.new_zeros(b, oh, ow, c)
    y0, y1 = max(0, -dy), min(oh, h - dy)
    x0, x1 = max(0, -dx), min(ow, w - dx)
    if y1 > y0 and x1 > x0:
        out[:, y0:y1, x0:x1] = v[:, y0 + dy:y1 + dy, x0 + dx:x1 + dx]
    return out


def im2col(views: Sequence[torch.Tensor], taps: Sequence[Tuple[int, int, int]], out_grid: Tuple[int, int, int]) -> torch.Tensor:
    """-> float64 [B, oh, ow, taps * C]: the GEMM operand the convolution of `views` / `taps` contracts over."""
    b, oh, ow = out_grid
    vs = [as4(v).double() for v in views]
    if any(v.shape[0] != b for v in vs):
        raise ValueError("views and output grid disagree on the batch")
    return torch.cat([_shifted(vs[vi], dx, dy, oh, ow) for vi, dx, dy in taps], dim=-1)


# float64 elements of im2col evaluated at once (1 GiB): a batch of 32 at 384 x 384 would otherwise need tens of GB
CHUNK_ELEMS = 1 << 27


def _image_chunks(views, taps, out_grid, max_elems):
    """(first, last) image ranges whose im2col holds at most max_elems elements (at least one image each)."""
    b, oh, ow = out_grid
    per_image = oh * ow * len(taps) * as4(views[0]).shape[-1]
    n = max(1, max_elems // max(per_image, 1))
    return [(i, min(b, i + n)) for i in range(0, b, n)]


def conv_acc_ref(views, taps, weight, out_grid, absolute: bool = False, max_elems: int = CHUNK_ELEMS) -> torch.Tensor:
    """The contraction alone, float64 [B, oh, ow, n]: sum_t sum_c view_t[b, y + dy_t, x + dx_t, c] * weight[n, t*C + c],
    evaluated over chunks of images.  absolute=True: the same of |view| and |weight|, the scale an fp32-accumulated
    element's rounding error is proportional to."""
    w = weight.double().abs() if absolute else weight.double()
    parts = []
    for i0, i1 in _image_chunks(views, taps, out_grid, max_elems):
        cols = im2col([as4(v)[i0:i1] for v in views], taps, (i1 - i0,) + tuple(out_grid[1:]))
        parts.append((cols.abs() if absolute else cols) @ w.t())
    return torch.cat(parts) if len(parts) > 1 else parts[0]


def _act(y: torch.Tensor, act: int) -> torch.Tensor:
    if act == 1:
        return torch.relu(y)
    if act == 2:
        return torch.nn.functional.gelu(y)
    if act != 0:
        raise ValueError(act)
    return y


def conv_gemm_ref(views, taps, weight, out_grid, bias=None, residual=None, act: int = 0, bias_per_image: bool = False,
                  out2_act: Optional[int] = None, max_elems: int = CHUNK_ELEMS):
    """odb_conv_gemm in float64: out[b, y, x, n] = residual + act(sum_t sum_c view_t[b, y + dy_t, x + dx_t, c] *
    weight[n, t * C + c] + bias[n]) over the output grid (B, oh, ow); act 0 none, 1 relu, 2 exact-erf gelu.
      * bias_per_image: bias is [B, n] and image b adds row b (bias_sb = n);
      * residual [1, H, W, n] (or [H, W, n]) is broadcast over the batch (residual sb = 0);
      * out2_act (1 relu, 2 gelu) also returns the out2 copy: out2_act(out) of the same unrounded value
        (conv_gemm.cu:737-744).  With a GELU copy the kernel's `out` keeps the pre-activation (act 0).
    The fp32-output epilogue (EPI_BIAS_RES_F32, conv_gemm.cu:549) is this definition with no rounding at all:
    out = residual + (acc + bias) in fp32.  The bf16 epilogues round `out` once, after the residual add
    (conv_gemm.cu:573 and 724), and the out2 copy once (conv_gemm.cu:744)."""
    y = conv_acc_ref(views, taps, weight, out_grid, max_elems=max_elems)
    if bias is not None:
        y = y + (bias.double()[:, None, None, :] if bias_per_image else bias.double())
    y = _act(y, act)
    if residual is not None:
        y = y + (residual.double().unsqueeze(0) if residual.dim() == 3 else as4(residual).double())
    if out2_act is None:
        return y
    return y, _act(y, out2_act)


def gn_stats_ref(y: torch.Tensor, groups: int = 32, eps: float = 1e-5) -> torch.Tensor:
    """Per image and group of the UNROUNDED conv result y [B, H, W, n] (float64): [B, groups, 2] = (mean, rstd =
    1 / sqrt(var + eps)) with the biased variance.  These are what the fused epilogue's partial sums (conv_gemm.cu:581,
    755) give after odb_groupnorm_finalize (ops.cu:211-215)."""
    b = y.shape[0]
    g = y.double().reshape(b, -1, groups, y.shape[-1] // groups).transpose(1, 2).reshape(b, groups, -1)
    mean = g.mean(-1)
    var = (g - mean[..., None]).pow(2).mean(-1)
    return torch.stack([mean, 1.0 / torch.sqrt(var + eps)], dim=-1)


def head_tail_ref(y: torch.Tensor, head_w: torch.Tensor, head_b: torch.Tensor, relu: bool) -> torch.Tensor:
    """The DPT head tail fused into the last 3x3 convolution (conv_gemm.cu:640-663): y [B, H, W, 32] is that
    convolution's conv + bias, unrounded; -> NCHW float64 [B, head_c, H, W] = relu?(relu(y) @ head_w^T + head_b), all
    in fp32 in the kernel (no rounding point)."""
    o = torch.relu(y.double()) @ head_w.double().t() + head_b.double()
    return (torch.relu(o) if relu else o).permute(0, 3, 1, 2)


def wgrad_ref(views, taps, dy, max_elems: int = CHUNK_ELEMS) -> torch.Tensor:
    """odb_conv_wgrad in float64: out[n, t * C + c] = sum_{b,y,x} dy[b, y, x, n] * view_t[b, y + dy_t, x + dx_t, c],
    over dy's grid -> [n, taps * C], summed over chunks of images."""
    d4 = as4(dy).double()
    b, oh, ow, n = d4.shape
    out = 0.0
    for i0, i1 in _image_chunks(views, taps, (b, oh, ow), max_elems):
        cols = im2col([as4(v)[i0:i1] for v in views], taps, (i1 - i0, oh, ow))
        out = out + d4[i0:i1].reshape(-1, n).t() @ cols.reshape(-1, cols.shape[-1])
    return out


def wgrad_abs_ref(views, taps, dy) -> torch.Tensor:
    """wgrad_ref of |views| and |dy|: the scale an fp32-accumulated element's rounding error is proportional to."""
    return wgrad_ref([as4(v).double().abs() for v in views], taps, as4(dy).double().abs())


def _bf16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(t.dtype)


def attention_bf16(q, k, v, scale: float = 0.125) -> torch.Tensor:
    """The wgmma attention kernel's arithmetic (csrc/attention_tc.cu) on q, k, v [..., T, 64], in their own dtype:
    exact two-pass softmax in the log2 domain, P = exp2(s * c - m * c) with c = fp32(scale * log2 e) and m the row
    maximum (attention_tc.cu:157-171); P is rounded to bf16 for the PV product (attention_tc.cu:177) while the row
    sum uses the unrounded values (attention_tc.cu:174); O = (bf16(P) V) / sum.  Equal to softmax(q k^T * scale) v
    in real arithmetic."""
    c = scale * _LOG2E_F32
    s = q @ k.transpose(-2, -1)
    m = s.amax(dim=-1, keepdim=True)
    p = torch.exp2(s * c - m * c)
    return (_bf16(p) @ v) / p.sum(dim=-1, keepdim=True)


def _qkv_heads(qkv, heads: int, head_dim: int = 64):
    b, t, _ = qkv.shape
    return qkv.double().view(b, t, 3, heads, head_dim).permute(2, 0, 3, 1, 4)           # q, k, v [b, heads, T, 64]


def attention_ref(qkv, heads: int, rounded: bool = False, scale: float = 0.125) -> torch.Tensor:
    """odb_attention / odb_attention_f32 of qkv [b, T, 3 * heads * 64] -> float64 [b, T, heads * 64].
    rounded=False: softmax(q k^T * scale) v exactly.  rounded=True: the bf16 kernel's P rounding (attention_bf16) in
    float64; its one remaining rounding, the bf16 store of O (attention_tc.cu:212), is left to the caller's bound."""
    q, k, v = _qkv_heads(qkv, heads)
    if rounded:
        o = attention_bf16(q, k, v, scale)
    else:
        o = torch.softmax(q @ k.transpose(-1, -2) * scale, -1) @ v
    b, t, _ = qkv.shape
    return o.transpose(1, 2).reshape(b, t, -1)


def lse_ref(qkv, heads: int, scale: float = 0.125) -> torch.Tensor:
    """The attention's `lse` output [b, heads, T]: log2 sum_j exp2(s_j * c), c = fp32(scale * log2 e)
    (attention_tc.cu:201, mc + log2(l)); attention_bwd_ref's P = exp2(s * c - lse) starts from it."""
    q, k, _ = _qkv_heads(qkv, heads)
    s = (q @ k.transpose(-1, -2)) * (scale * _LOG2E_F32)
    m = s.amax(-1, keepdim=True)
    return (m + torch.log2(torch.exp2(s - m).sum(-1, keepdim=True)))[..., 0]


def attention_bwd_ref(qkv, o, d_o, lse: Optional[torch.Tensor] = None, rounded: bool = False, scale: float = 0.125,
                      head_dim: int = 64) -> torch.Tensor:
    """Gradient w.r.t. qkv [b, T, 3 * heads * 64] of o = softmax(q k^T * scale) v (timm Attention), from d_o
    [b, T, heads * 64] -> float64 [b, T, 3 * heads * 64].

    rounded=False: the exact gradient (float64 autograd; `o` and `lse` are not used).
    rounded=True: the bf16 kernel's arithmetic (csrc/bgemm_tc.cu) in float64 between its rounding points —
      P = bf16(exp2(S * c - lse)) with c = fp32(scale * log2 e) and the forward kernel's log2-sum-exp `lse`
      [b, heads, T] (recomputed exactly when None); D = row dot of the bf16 o and d_o; dS = bf16(P * (dO V^T - D) *
      scale); dQ = bf16(dS K), dK = bf16(dS^T Q), dV = bf16(P^T dO)."""
    b, t, c3 = qkv.shape
    heads = c3 // (3 * head_dim)
    if not rounded:
        with torch.enable_grad():
            qd = qkv.detach().double().requires_grad_(True)
            q, k, v = qd.view(b, t, 3, heads, head_dim).permute(2, 0, 3, 1, 4)
            out = (torch.softmax(q @ k.transpose(-1, -2) * scale, -1) @ v).transpose(1, 2).reshape(b, t, heads * head_dim)
            g, = torch.autograd.grad(out, (qd,), d_o.double())
        return g
    q, k, v = qkv.double().view(b, t, 3, heads, head_dim).permute(2, 0, 3, 1, 4)        # [b, heads, T, 64]
    dO = d_o.double().view(b, t, heads, head_dim).transpose(1, 2)
    O = o.double().view(b, t, heads, head_dim).transpose(1, 2)
    c = scale * _LOG2E_F32
    s = q @ k.transpose(-1, -2)
    if lse is None:
        lse = torch.log2(torch.exp2(s * c).sum(-1))
    p = _bf16(torch.exp2(s * c - lse.double()[..., None]))
    dd = (O * dO).sum(-1, keepdim=True)
    ds = _bf16(p * (dO @ v.transpose(-1, -2) - dd) * scale)
    dq, dk, dv = _bf16(ds @ k), _bf16(ds.transpose(-1, -2) @ q), _bf16(p.transpose(-1, -2) @ dO)
    return torch.stack([dq, dk, dv]).permute(1, 3, 0, 2, 4).reshape(b, t, c3)
