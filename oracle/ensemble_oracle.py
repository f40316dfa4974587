"""Test-time ensembles restated in float64 torch (omnidata_b200/csrc/ensemble.cu, EnsemblePredictor): the Gram sums,
the alignment energy solved as a dense float64 system, and both merges with the kernels' rounding points.  Members are
[K, B, C, H, W] as the predictor returned them, member k mirrored where bit k of `flips` is set.  Each definition
names the kernel it mirrors."""
from __future__ import annotations

import math

import numpy as np
import torch

KAPPA = 1e-6                                    # ensemble.cu kEnsKappa
RAD_TO_DEG = 180.0 / 3.141592653589793


def unmirror(members: torch.Tensor, flips: int) -> torch.Tensor:
    """The members in member 0's orientation (what the kernels read in gather form)."""
    return torch.stack([m.flip(-1) if (flips >> k) & 1 else m for k, m in enumerate(members)])


def gram(members: torch.Tensor, flips: int) -> torch.Tensor:
    """ensemble_gram_kernel + ensemble_gram_reduce_kernel: [B, (K+1)(K+2)/2], the packed upper triangle (row-major,
    i <= j) of the Gram matrix of v = (a_0, .., a_{K-1}, 1) over V, the pixels where all K members are finite."""
    a = unmirror(members, flips)[:, :, 0].double()                      # [K, B, H, W]
    K, B = a.shape[:2]
    valid = torch.isfinite(a).all(0)
    v = torch.cat([torch.where(valid, a, 0.0), valid.double()[None]]).reshape(K + 1, B, -1)
    G = torch.einsum("ibp,jbp->bij", v, v)
    iu = torch.triu_indices(K + 1, K + 1)
    return G[:, iu[0], iu[1]]


def unpack(g: torch.Tensor, K: int) -> torch.Tensor:
    """One image's packed gram -> the symmetric (K+1) x (K+1) matrix."""
    G = torch.zeros(K + 1, K + 1, dtype=torch.float64)
    iu = torch.triu_indices(K + 1, K + 1)
    G[iu[0], iu[1]] = g.double()
    return G + G.triu(1).T


def normal_equations(g: torch.Tensor, K: int, kappa: float = KAPPA):
    """ensemble_align_solve_kernel: the gradient of
    E = sum_{i<j} sum_V (s_i a_i + t_i - s_j a_j - t_j)^2 + kappa n sum_{k>=1} ((s_k - 1)^2 + t_k^2),  s_0 = 1, t_0 = 0,
    set to zero, in the unknowns (s_1, t_1, .., s_{K-1}, t_{K-1}), written directly from the pair sum: dense (A, rhs)."""
    G = unpack(g, K)
    n = G[K, K]
    S = G[:K, K]
    M = 2 * (K - 1)
    A = torch.zeros(M, M, dtype=torch.float64)
    rhs = torch.zeros(M, dtype=torch.float64)

    def u(k):                                   # the quadratic form of d_k = s_k a_k + t_k in (s_k, t_k): rows of a_k, 1
        return [(k, 2 * (k - 1)), (K, 2 * (k - 1) + 1)]
    # sum over pairs i < j of |d_i - d_j|^2: expand into the Gram entries; member 0 has (s, t) = (1, 0) fixed
    for i in range(K):
        for j in range(i + 1, K):
            for (p, sgn_p) in ((i, 1.0), (j, -1.0)):
                for (q, sgn_q) in ((i, 1.0), (j, -1.0)):
                    sg = sgn_p * sgn_q
                    if p >= 1 and q >= 1:
                        for rp, cp in u(p):
                            for rq, cq in u(q):
                                A[cp, cq] += sg * G[rp, rq]
                    elif p >= 1 and q == 0:             # cross term with the fixed d_0 = a_0 -> right-hand side
                        for rp, cp in u(p):
                            rhs[cp] -= sg * G[rp, 0]
    for k in range(1, K):
        A[2 * (k - 1), 2 * (k - 1)] += kappa * n
        A[2 * (k - 1) + 1, 2 * (k - 1) + 1] += kappa * n
        rhs[2 * (k - 1)] += kappa * n
    return A, rhs


def solve(g: torch.Tensor, K: int, kappa: float = KAPPA) -> torch.Tensor:
    """The alignment as a dense float64 solve: [B, K, 2] = (s_k, t_k), member 0 (1, 0)."""
    out = torch.zeros(g.shape[0], K, 2, dtype=torch.float64)
    out[:, 0, 0] = 1.0
    for b in range(g.shape[0]):
        if K > 1:
            A, rhs = normal_equations(g[b], K, kappa)
            out[b, 1:] = torch.linalg.solve(A, rhs).view(K - 1, 2)
    return out


def energy(a: torch.Tensor, st: torch.Tensor, kappa: float = KAPPA) -> float:
    """E of one image's un-mirrored members a [K, H, W] at st [K, 2] (over the pixels where all are finite)."""
    valid = torch.isfinite(a).all(0)
    d = st[:, 0, None] * a[:, valid].double() + st[:, 1, None]
    K, n = a.shape[0], float(valid.sum())
    e = sum(float(((d[i] - d[j]) ** 2).sum()) for i in range(K) for j in range(i + 1, K))
    return e + kappa * n * float(((st[1:, 0] - 1) ** 2 + st[1:, 1] ** 2).sum())


def _sqrt(x: torch.Tensor) -> torch.Tensor:
    """The correctly rounded float64 square root (the kernels' __dsqrt_rn).  torch's CPU sqrt is not: it can land one
    ulp low, e.g. sqrt(0.7132372334599495 ** 2)."""
    return torch.from_numpy(np.sqrt(x.double().cpu().numpy()))


def _median(v: torch.Tensor) -> torch.Tensor:
    """The median over dim 0 of float32 values: the middle one for odd K, (lo + hi) * 0.5 in float32 for even K."""
    s = v.sort(0).values
    K = s.shape[0]
    if K % 2:
        return s[(K - 1) // 2]
    return (s[K // 2 - 1] + s[K // 2]) * 0.5


def merge_depth(members: torch.Tensor, flips: int, st: torch.Tensor):
    """ensemble_merge_depth_kernel: (out [B, H, W], spread [B, H, W]) float32.  d_k = float32(s_k a_k + t_k) (float64
    multiply, then add), out = median, spread = median |d_k - out| (float32); where a member is not finite: member 0 and
    NaN."""
    a = unmirror(members, flips)[:, :, 0].float()                       # [K, B, H, W]
    st = st.double().cpu()
    s = st[:, :, 0].T[:, :, None, None]
    t = st[:, :, 1].T[:, :, None, None]
    d = (s * a.double().cpu() + t).float()
    valid = torch.isfinite(a.cpu()).all(0)
    m = _median(d)
    dev = _median((d - m).abs())
    out = torch.where(valid, m, a[0].cpu())
    spread = torch.where(valid, dev, torch.full_like(dev, math.nan))
    return out, spread


def merge_normal(members: torch.Tensor, flips: int):
    """ensemble_merge_normal_kernel: (out [B, 3, H, W], spread [B, H, W]) float32.  n_k = 2 clamp(c, 0, 1) - 1 (fmax /
    fmin: NaN clamps to 0), x negated for a mirrored member, m = (sum_k n_k) / K summed in member order, out =
    (m / |m| + 1) / 2 rounded once to float32, or member 0 clamped where |m| <= 1e-6; spread = mean_k
    atan2(|n_k x o|, n_k . o) in degrees, o = 2 out - 1."""
    a = unmirror(members, flips).float().cpu()                          # [K, B, 3, H, W]
    K = a.shape[0]
    c = torch.fmin(torch.fmax(a, torch.zeros(())), torch.ones(()))
    n = 2.0 * c.double() - 1.0
    sign = torch.tensor([-1.0 if (flips >> k) & 1 else 1.0 for k in range(K)], dtype=torch.float64)
    n[:, :, 0] = n[:, :, 0] * sign[:, None, None, None]
    m = n[0].clone()
    for k in range(1, K):
        m = m + n[k]
    m = m / K
    norm = _sqrt(m[:, 0] * m[:, 0] + m[:, 1] * m[:, 1] + m[:, 2] * m[:, 2])
    enc = ((m / norm[:, None] + 1.0) * 0.5).float()
    out = torch.where((norm <= 1e-6)[:, None], c[0], enc)
    o = 2.0 * out.double() - 1.0
    th = torch.zeros_like(norm)
    for k in range(K):
        p = n[k]
        cx = p[:, 1] * o[:, 2] - p[:, 2] * o[:, 1]
        cy = p[:, 2] * o[:, 0] - p[:, 0] * o[:, 2]
        cz = p[:, 0] * o[:, 1] - p[:, 1] * o[:, 0]
        cr = _sqrt(cx * cx + cy * cy + cz * cz)
        dot = p[:, 0] * o[:, 0] + p[:, 1] * o[:, 1] + p[:, 2] * o[:, 2]
        th = th + torch.atan2(cr, dot) * RAD_TO_DEG
    return out, (th / K).float()
