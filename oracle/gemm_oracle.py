"""Float64 restatement of the three GEMM-shaped operations the backward of the train step launches: the implicit-GEMM
convolution (odb_conv_gemm, which also computes every input gradient), the weight gradient (odb_conv_wgrad) and the
attention backward (odb_attention_bwd).  Plain torch on any device; each function follows the definition in
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


def conv_gemm_ref(views, taps, weight, out_grid, bias=None, residual=None, act: int = 0) -> torch.Tensor:
    """odb_conv_gemm in float64: out[b, y, x, n] = residual + act(sum_t sum_c view_t[b, y + dy_t, x + dx_t, c] *
    weight[n, t * C + c] + bias[n]) over the output grid (B, oh, ow); act 0 none, 1 relu, 2 exact-erf gelu."""
    y = im2col(views, taps, out_grid) @ weight.double().t()
    if bias is not None:
        y = y + bias.double()
    if act == 1:
        y = torch.relu(y)
    elif act == 2:
        y = torch.nn.functional.gelu(y)
    elif act != 0:
        raise ValueError(act)
    if residual is not None:
        y = y + as4(residual).double()
    return y


def wgrad_ref(views, taps, dy) -> torch.Tensor:
    """odb_conv_wgrad in float64: out[n, t * C + c] = sum_{b,y,x} dy[b, y, x, n] * view_t[b, y + dy_t, x + dx_t, c],
    over dy's grid -> [n, taps * C]."""
    d4 = as4(dy).double()
    b, oh, ow, n = d4.shape
    cols = im2col(views, taps, (b, oh, ow))
    return d4.reshape(-1, n).t() @ cols.reshape(-1, cols.shape[-1])


def wgrad_abs_ref(views, taps, dy) -> torch.Tensor:
    """wgrad_ref of |views| and |dy|: the scale an fp32-accumulated element's rounding error is proportional to."""
    return wgrad_ref([as4(v).double().abs() for v in views], taps, as4(dy).double().abs())


def _bf16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(t.dtype)


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
