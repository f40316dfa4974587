"""The anchored tiled merge restated in float64 torch (omnidata_b200/csrc/tiled.cu, TiledPredictor(anchor=...)): the
antialiased bilinear resize that makes the anchor (csrc/imageproc.cu), the anchor moments, the anchored alignment
objective solved as a dense float64 system, and the anchored merge.  The grid, the overlap moments, the ridge normal
equations and the blend are those of oracle/tiled_oracle.py.  Each definition names the kernel it mirrors."""
from __future__ import annotations

from typing import Tuple

import torch
import torch.nn.functional as F

from . import tiled_oracle as O

KAPPA = 1e-6                                    # tiled.cu:33 kAnchorKappa


def resize(x: torch.Tensor, size: Tuple[int, int]) -> torch.Tensor:
    """imageproc.cu:140-172 resample_h / resample_v_f32_kernel: torch's antialiased bilinear resize of [..., h, w] in
    float64."""
    lead = x.shape[:-2]
    y = F.interpolate(x.double().reshape(-1, 1, *x.shape[-2:]), size=tuple(size), mode="bilinear",
                      align_corners=False, antialias=True)
    return y.reshape(*lead, *size)


def anchor_moments(pred: torch.Tensor, g: torch.Tensor, B: int, H: int, W: int, tile, overlap: int) -> torch.Tensor:
    """tiled.cu:281-336 tile_anchor_moments_kernel: [B, T, 5] = (n, Sa, Saa, Sg, Sag) over each tile's pixels inside
    the image, a the tile's prediction, g the anchor [B, H, W]."""
    th, tw = tile
    oy, ox = O.grid(H, W, tile, overlap)
    T = len(oy) * len(ox)
    hy, wx = min(th, H), min(tw, W)
    out = torch.zeros(B, T, 5, dtype=torch.float64)
    for b in range(B):
        for i in range(T):
            y0, x0 = oy[i // len(ox)], ox[i % len(ox)]
            a = pred[b * T + i].reshape(th, tw)[:hy, :wx].double().flatten()
            c = g[b, y0:y0 + hy, x0:x0 + wx].double().flatten()
            out[b, i] = torch.stack([torch.tensor(float(a.numel()), dtype=torch.float64), a.sum(), (a * a).sum(),
                                     c.sum(), (a * c).sum()])
    return out


def normal_equations(m: torch.Tensor, am: torch.Tensor, ny: int, nx: int, lam: float = O.LAMBDA,
                     kappa: float = KAPPA):
    """tiled.cu:133-227 tile_align_solve_kernel with anchor moments: the gradient of
    E(s, t) = sum_pairs sum_overlap (s_i a + t_i - s_j b - t_j)^2 + lam Nbar sum_i (1/n_i) sum_tile (s_i a + t_i - g)^2
    + kappa lam Nbar sum_i ((s_i - 1)^2 + t_i^2) set to zero, for one image's overlap moments m [pairs, 6] and anchor
    moments am [T, 5].  The pair terms and the ridge are tiled_oracle.normal_equations at kappa lam.  Dense (A, rhs)."""
    A, rhs = O.normal_equations(m, ny, nx, kappa * lam)
    P = len(O.pairs(ny, nx))
    nbar = max(float(m[:, 0].sum()) / P, 1.0) if P else 1.0
    for i in range(ny * nx):
        n, sa, saa, sg, sag = am[i].tolist()
        mu = lam * nbar / n
        A[2 * i:2 * i + 2, 2 * i:2 * i + 2] += mu * torch.tensor([[saa, sa], [sa, n]], dtype=torch.float64)
        rhs[2 * i] += mu * sag
        rhs[2 * i + 1] += mu * sg
    return A, rhs


def solve(m: torch.Tensor, am: torch.Tensor, ny: int, nx: int, lam: float = O.LAMBDA,
          kappa: float = KAPPA) -> torch.Tensor:
    """The anchored tile_align_solve_kernel as a dense float64 solve: [B, T, 2] = (s_i, t_i) from overlap moments
    m [B, pairs, 6] and anchor moments am [B, T, 5]."""
    out = []
    for b in range(m.shape[0]):
        A, rhs = normal_equations(m[b], am[b], ny, nx, lam, kappa)
        out.append(torch.linalg.solve(A, rhs).view(ny * nx, 2))
    return torch.stack(out)


def pair_energy(m: torch.Tensor, st: torch.Tensor, ny: int, nx: int) -> float:
    """The seam part of E, sum_pairs sum_overlap (s_i a + t_i - s_j b - t_j)^2, of one image's moments m [pairs, 6] at
    st [T, 2]."""
    A, _ = O.normal_equations(m, ny, nx, lam=0.0)
    x = st.reshape(-1).double()
    return float(x @ A @ x)


def merge(pred: torch.Tensor, g: torch.Tensor, B: int, H: int, W: int, tile, overlap: int,
          lam: float = O.LAMBDA) -> torch.Tensor:
    """TiledPredictor.merge with an anchor, in float64: one-channel tile predictions pred [B*T, 1, th, tw] aligned to
    the anchor g [B, H, W] and blended; [B, H, W]."""
    oy, ox = O.grid(H, W, tile, overlap)
    st = solve(O.moments(pred, B, H, W, tile, overlap), anchor_moments(pred, g, B, H, W, tile, overlap), len(oy),
               len(ox), lam)
    return O.blend(pred, st, B, H, W, tile, overlap).squeeze(1)
