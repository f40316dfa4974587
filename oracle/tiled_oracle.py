"""Tiled inference merge restated in float64 torch (omnidata_b200/csrc/tiled.cu): the tile grid, the gather, the
overlap moments, the alignment objective solved as a dense float64 system, the blend weights and the blend.  Each
definition names the kernel it mirrors (tiled.cu line)."""
from __future__ import annotations

from fractions import Fraction
from typing import List, Tuple

import torch

LAMBDA = 1e-3                                   # tiled.cu:33 kAlignLambda


def axis_origins(length: int, t: int, overlap: int) -> List[int]:
    """tiled.cu:37-43 tile_count / tile_origin: ceil((L - v) / (t - v)) tiles at round(k (L - t) / (n - 1)), halves
    up; one tile at 0 when L <= t."""
    if length <= t:
        return [0]
    n = -(-(length - overlap) // (t - overlap))
    return [int(Fraction(k * (length - t), n - 1) + Fraction(1, 2)) for k in range(n)]


def grid(H: int, W: int, tile: Tuple[int, int], overlap: int):
    return axis_origins(H, tile[0], overlap), axis_origins(W, tile[1], overlap)


def gather(x: torch.Tensor, tile: Tuple[int, int], overlap: int) -> torch.Tensor:
    """tiled.cu:46-68 tile_gather_kernel: [B*T, 3, th, tw], rows / columns past the image replicate its last one."""
    B, C, H, W = x.shape
    th, tw = tile
    oy, ox = grid(H, W, tile, overlap)
    out = []
    for b in range(B):
        for y0 in oy:
            rows = torch.arange(y0, y0 + th).clamp(max=H - 1)
            for x0 in ox:
                cols = torch.arange(x0, x0 + tw).clamp(max=W - 1)
                out.append(x[b][:, rows][:, :, cols])
    return torch.stack(out)


def pairs(ny: int, nx: int) -> List[Tuple[int, int]]:
    """tiled.cu:78-97: horizontal neighbour pairs row-major, then vertical ones; (first, second) tile indices."""
    h = [(ty * nx + tx, ty * nx + tx + 1) for ty in range(ny) for tx in range(nx - 1)]
    v = [(ty * nx + tx, (ty + 1) * nx + tx) for ty in range(ny - 1) for tx in range(nx)]
    return h + v


def overlap_values(pred: torch.Tensor, b: int, i: int, j: int, H: int, W: int, tile, overlap: int):
    """a, b over the overlap of tiles i, j of image b inside the image (tiled.cu:78-103 tile_moments_kernel)."""
    th, tw = tile
    oy, ox = grid(H, W, tile, overlap)
    nx, T = len(ox), len(oy) * len(ox)
    yi, xi, yj, xj = oy[i // nx], ox[i % nx], oy[j // nx], ox[j % nx]
    y0, y1 = max(yi, yj), min(yi + th, yj + th, H)
    x0, x1 = max(xi, xj), min(xi + tw, xj + tw, W)
    a = pred[b * T + i].reshape(th, tw)[y0 - yi:y1 - yi, x0 - xi:x1 - xi]
    c = pred[b * T + j].reshape(th, tw)[y0 - yj:y1 - yj, x0 - xj:x1 - xj]
    return a.double().flatten(), c.double().flatten()


def moments(pred: torch.Tensor, B: int, H: int, W: int, tile, overlap: int) -> torch.Tensor:
    """tiled.cu:70-131 tile_moments_kernel: [B, pairs, 6] = (n, Sa, Sb, Saa, Sbb, Sab)."""
    oy, ox = grid(H, W, tile, overlap)
    out = torch.zeros(B, len(pairs(len(oy), len(ox))), 6, dtype=torch.float64)
    for b in range(B):
        for p, (i, j) in enumerate(pairs(len(oy), len(ox))):
            a, c = overlap_values(pred, b, i, j, H, W, tile, overlap)
            out[b, p] = torch.stack([torch.tensor(float(a.numel()), dtype=torch.float64), a.sum(), c.sum(),
                                     (a * a).sum(), (c * c).sum(), (a * c).sum()])
    return out


def normal_equations(m: torch.Tensor, ny: int, nx: int, lam: float = LAMBDA):
    """tiled.cu:145-185: the gradient of E(s, t) = sum_pairs sum_overlap (s_i a + t_i - s_j b - t_j)^2
    + lam Nbar sum_i ((s_i - 1)^2 + t_i^2) set to zero, unknowns (s_0, t_0, s_1, t_1, ...), for one image's moments
    m [pairs, 6].  Dense float64 (A, rhs)."""
    T = ny * nx
    P = len(pairs(ny, nx))
    nbar = max(float(m[:, 0].sum()) / P, 1.0) if P else 1.0
    A = torch.zeros(2 * T, 2 * T, dtype=torch.float64)
    for p, (i, j) in enumerate(pairs(ny, nx)):
        n, sa, sb, saa, sbb, sab = m[p].tolist()
        # residual r = [a, 1, -b, -1] . [s_i, t_i, s_j, t_j]: sum over the overlap of r r^T
        blk = torch.tensor([[saa, sa, -sab, -sa], [sa, n, -sb, -n], [-sab, -sb, sbb, sb], [-sa, -n, sb, n]],
                           dtype=torch.float64)
        idx = torch.tensor([2 * i, 2 * i + 1, 2 * j, 2 * j + 1])
        A[idx[:, None], idx[None, :]] += blk
    A += lam * nbar * torch.eye(2 * T, dtype=torch.float64)
    rhs = torch.zeros(2 * T, dtype=torch.float64)
    rhs[0::2] = lam * nbar
    return A, rhs


def solve(m: torch.Tensor, ny: int, nx: int, lam: float = LAMBDA) -> torch.Tensor:
    """tiled.cu:133-220 tile_align_solve_kernel, as a dense float64 solve: [B, T, 2] = (s_i, t_i)."""
    out = []
    for b in range(m.shape[0]):
        A, rhs = normal_equations(m[b], ny, nx, lam)
        out.append(torch.linalg.solve(A, rhs).view(ny * nx, 2))
    return torch.stack(out)


def ramp(length: int, t: int, overlap: int) -> torch.Tensor:
    """tiled.cu:232-238 tile_ramp: [n, t] per-tile weights along one axis, rho(d) = min(1, (d + 1) / (v + 1)), d = the
    distance to the nearest tile edge that is not on the image border."""
    o = axis_origins(length, t, overlap)
    n = len(o)
    pos = torch.arange(t, dtype=torch.float64)
    out = []
    for k in range(n):
        d = torch.full((t,), float("inf"), dtype=torch.float64)
        if k > 0:
            d = torch.minimum(d, pos)
        if k < n - 1:
            d = torch.minimum(d, t - 1 - pos)
        out.append(torch.clamp((d + 1) / (overlap + 1), max=1.0))
    return torch.stack(out)


def blend(pred: torch.Tensor, st, B: int, H: int, W: int, tile, overlap: int) -> torch.Tensor:
    """tiled.cu:240-272 tile_blend_kernel: [B, C, H, W] = sum_i w_i (s_i d_i + t_i) / sum_i w_i, tiles row-major.  The
    weights are the kernel's: rho and rho_y * rho_x rounded to fp32."""
    th, tw = tile
    oy, ox = grid(H, W, tile, overlap)
    ry, rx = ramp(H, th, overlap).float(), ramp(W, tw, overlap).float()
    T = len(oy) * len(ox)
    C = pred.shape[1]
    out = torch.zeros(B, C, H, W, dtype=torch.float64)
    wsum = torch.zeros(H, W, dtype=torch.float64)
    for b in range(B):
        acc = torch.zeros(C, H, W, dtype=torch.float64)
        wsum.zero_()
        for ky, y0 in enumerate(oy):
            hy = min(th, H - y0)
            for kx, x0 in enumerate(ox):
                wx = min(tw, W - x0)
                i = ky * len(ox) + kx
                w = (ry[ky, :hy, None] * rx[kx, None, :wx]).double()
                d = pred[b * T + i, :, :hy, :wx].double()
                if st is not None:
                    d = st[b, i, 0] * d + st[b, i, 1]
                acc[:, y0:y0 + hy, x0:x0 + wx] += w * d
                wsum[y0:y0 + hy, x0:x0 + wx] += w
        out[b] = acc / wsum
    return out


def merge(pred: torch.Tensor, B: int, H: int, W: int, tile, overlap: int, lam: float = LAMBDA) -> torch.Tensor:
    """TiledPredictor.merge in float64: align (one channel) and blend; [B,H,W] for one channel, else [B,C,H,W]."""
    oy, ox = grid(H, W, tile, overlap)
    st = None
    if pred.shape[1] == 1:
        st = solve(moments(pred, B, H, W, tile, overlap), len(oy), len(ox), lam)
    out = blend(pred, st, B, H, W, tile, overlap)
    return out.squeeze(1) if pred.shape[1] == 1 else out
