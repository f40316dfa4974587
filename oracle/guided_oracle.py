"""Guided upsampling restated in float64 torch (omnidata_b200/csrc/guided.cu, GuidedPredictor): clipped box means by
direct sums over the windows, the local linear model by a dense 3x3 solve, the second box mean with the single fp32
rounding of the coefficients, and the apply composed from imageproc.bilinear_aa_weights.  Works on the tensors' device.
Each definition names the kernel it mirrors."""
from __future__ import annotations

import torch

from omnidata_b200.imageproc import bilinear_aa_weights


def box_mean(f: torch.Tensor, r: int) -> torch.Tensor:
    """mean over W_i = {j : |j - i|_inf <= r} clipped at the border, of f [..., h, w] float64: every window's sum taken
    directly as 2r + 1 shifted rows, then 2r + 1 shifted columns (no cumulative sums), over the window's size."""
    f = f.double()
    h, w = f.shape[-2:]
    col = torch.zeros_like(f)
    for d in range(-r, r + 1):                      # col[y] += f[y + d] where y + d lies inside
        lo, hi = max(0, -d), min(h, h - d)
        if lo < hi:
            col[..., lo:hi, :] += f[..., lo + d:hi + d, :]
    s = torch.zeros_like(f)
    for d in range(-r, r + 1):
        lo, hi = max(0, -d), min(w, w - d)
        if lo < hi:
            s[..., :, lo:hi] += col[..., :, lo + d:hi + d]
    y = torch.arange(h, device=f.device)
    x = torch.arange(w, device=f.device)
    ny = (torch.clamp(y + r, max=h - 1) - torch.clamp(y - r, min=0) + 1).double()
    nx = (torch.clamp(x + r, max=w - 1) - torch.clamp(x - r, min=0) + 1).double()
    return s / (ny[:, None] * nx[None, :])


def linear_model(g: torch.Tensor, p: torch.Tensor, r: int, eps: float):
    """guided_box_v_products_kernel + guided_solve_kernel: (a [B, C, 3, h, w], b [B, C, h, w]) float64 with
    a_c = (Sigma + eps I)^-1 v_c and b_c = m_c - a_c . mu over the windows of radius r."""
    g, p = g.double(), p.double()
    mu = box_mean(g, r)                                                  # [B, 3, h, w]
    gg = box_mean(g[:, :, None] * g[:, None], r)                         # [B, 3, 3, h, w]
    sigma = gg - mu[:, :, None] * mu[:, None]
    m = box_mean(p, r)                                                   # [B, C, h, w]
    v = box_mean(g[:, None] * p[:, :, None], r) - mu[:, None] * m[:, :, None]      # [B, C, 3, h, w]
    A = sigma.permute(0, 3, 4, 1, 2) + eps * torch.eye(3, dtype=torch.float64, device=g.device)   # [B, h, w, 3, 3]
    rhs = v.permute(0, 3, 4, 2, 1)                                       # [B, h, w, 3, C]
    a = torch.linalg.solve(A, rhs).permute(0, 4, 3, 1, 2)               # [B, C, 3, h, w]
    b = m - (a * mu[:, None]).sum(2)
    return a, b


def coefficients(g: torch.Tensor, p: torch.Tensor, r: int, eps: float, round_fp32: bool = True) -> torch.Tensor:
    """odb_guided_coefficients: coef [B, 4C, h, w], plane 4c + k = box mean of a_ck (k < 3) or of b_c (k = 3), rounded
    to float32 once (float64 without `round_fp32`)."""
    a, b = linear_model(g, p, r, eps)
    B, C = b.shape[:2]
    ab = torch.cat([a, b[:, :, None]], 2).reshape(B, 4 * C, *b.shape[-2:])
    coef = box_mean(ab, r)
    return coef.float() if round_fp32 else coef


def resample(f: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """ops.resize_bilinear of f [..., h, w] to H x W in float64: the per-axis weights of bilinear_aa_weights as dense
    matrices."""
    h, w = f.shape[-2:]

    def dense(n_in, n_out):
        bounds, weights, _ = bilinear_aa_weights(n_in, n_out)
        M = torch.zeros(n_out, n_in, dtype=torch.float64)
        for o in range(n_out):
            x0, cnt = int(bounds[o, 0]), int(bounds[o, 1])
            M[o, x0:x0 + cnt] = torch.from_numpy(weights[o, :cnt])
        return M.to(f.device)
    return dense(h, H) @ f.double() @ dense(w, W).T


def apply(x: torch.Tensor, coef: torch.Tensor) -> torch.Tensor:
    """odb_guided_apply in float64: out [B, C, H, W] = B_c + sum_k A_ck x_k, (A, B) = coef resampled to x's size."""
    x = x.double()
    B, _, H, W = x.shape
    C = coef.shape[1] // 4
    out = torch.empty(B, C, H, W, dtype=torch.float64, device=x.device)
    for c in range(C):                              # one channel at a time: the resampled planes are large
        A = resample(coef[:, 4 * c:4 * c + 4], H, W)
        out[:, c] = A[:, 3] + (A[:, :3] * x).sum(1)
    return out


def guided(x: torch.Tensor, g: torch.Tensor, p: torch.Tensor, r: int, eps: float, round_fp32: bool = True):
    """GuidedPredictor.refine: the filter of p [B, C, h, w] against g [B, 3, h, w], applied to x [B, 3, H, W]."""
    return apply(x, coefficients(g, p, r, eps, round_fp32))
