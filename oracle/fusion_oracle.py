"""Float64 restatement of the depth-normal fusion and of depth_normals (csrc/fusion.cu; definition in DESIGN.md §3
"Depth-normal fusion").  The valid set, the edge rule and the edge coefficients follow the kernels' operation order
(numpy rounds every operation to nearest and never fuses).  The solve is independent of the kernels: the bordered
system in (z, t) is assembled from the energy itself, not from the eliminated form, and solved exactly by a sparse LU
(scipy.sparse.linalg.factorized) with t eliminated last.  `matvec` applies the eliminated operator M, so that a GPU solution can be checked by its
residual where a direct solve is too slow."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

KAPPA = 1e-6
STATUS_OK, STATUS_EMPTY, STATUS_FLAT = 0, 1, 2


def _f64(x):
    return np.asarray(x, dtype=np.float64)


def valid_set(a, mask=None):
    a = _f64(a)
    v = np.isfinite(a)
    if mask is not None:
        v &= np.asarray(mask) != 0
    return v


def depth_range(a, v):
    """(min, max) of a over V; (inf, -inf) when V is empty."""
    a = _f64(a)
    return (float(a[v].min()), float(a[v].max())) if v.any() else (np.inf, -np.inf)


def rays(h, w, intrinsics):
    fx, fy, cx, cy = (float(k) for k in intrinsics)
    return (np.arange(w, dtype=np.float64) - cx) / fx, (np.arange(h, dtype=np.float64) - cy) / fy


def _dot(u, v):
    return (u[0] * v[0] + u[1] * v[1]) + u[2] * v[2]


def unit_normals(c, axes):
    """(usable [H,W], unit normals [3,H,W]) of the encoded normals c [3,H,W]."""
    c = _f64(c)
    finite = np.isfinite(c).all(0)
    with np.errstate(invalid="ignore", divide="ignore"):
        n = np.stack([float(axes[k]) * (2.0 * np.fmin(np.fmax(c[k], 0.0), 1.0) - 1.0) for k in range(3)])
        length = np.sqrt(_dot(n, n))
        usable = finite & (length >= 0.5)
        return usable, n / length


def edges(a, c, intrinsics, axes=(1, -1, -1), jump=0.02, mask=None):
    """The right edges (alpha, beta [H,W-1]) and down edges (alpha, beta [H-1,W]), 0 where dropped, and V."""
    a = _f64(a)
    h, w = a.shape
    v = valid_set(a, mask)
    lo, hi = depth_range(a, v)
    thr = jump * (hi - lo)
    usable, n = unit_normals(c, axes)
    rx, ry = rays(h, w, intrinsics)
    rxg, ryg = np.broadcast_to(rx[None, :], (h, w)), np.broadcast_to(ry[:, None], (h, w))
    out = []
    for sl_p, sl_q in (((slice(None), slice(0, w - 1)), (slice(None), slice(1, w))),
                       ((slice(0, h - 1), slice(None)), (slice(1, h), slice(None)))):
        with np.errstate(invalid="ignore", divide="ignore"):
            np_, nq = n[(slice(None),) + sl_p], n[(slice(None),) + sl_q]
            keep = v[sl_p] & v[sl_q] & (np.abs(a[sl_q] - a[sl_p]) <= thr) & usable[sl_p] & usable[sl_q]
            keep &= _dot(np_, nq) > 0.0
            m = np_ + nq
            m = m / np.sqrt(_dot(m, m))
            alpha = _dot(m, (rxg[sl_p], ryg[sl_p], np.ones_like(rxg[sl_p])))
            beta = _dot(m, (rxg[sl_q], ryg[sl_q], np.ones_like(rxg[sl_q])))
        out.append((np.where(keep, alpha, 0.0), np.where(keep, beta, 0.0)))
    return out[0], out[1], v


def kept_edges(right, down):
    """Kept edges as the kernels count them: those whose two coefficients are not both 0."""
    return int(sum(((al != 0) | (be != 0)).sum() for al, be in (right, down)))


def _edge_list(right, down, h, w):
    """(p, q, alpha, beta) flat arrays of the edges with a nonzero coefficient."""
    idx = np.arange(h * w).reshape(h, w)
    ps, qs, als, bes = [], [], [], []
    for (al, be), (p, q) in ((right, (idx[:, :-1], idx[:, 1:])), (down, (idx[:-1, :], idx[1:, :]))):
        k = (al != 0) | (be != 0)
        ps.append(p[k]); qs.append(q[k]); als.append(al[k]); bes.append(be[k])
    return np.concatenate(ps), np.concatenate(qs), np.concatenate(als), np.concatenate(bes)


def fuse(a, c, intrinsics, weight=0.1, shift=True, jump=0.02, axes=(1, -1, -1), mask=None):
    """dict(z [H,W] float64 (NaN off V), t, n = |V|, kept, status), from the bordered energy solved exactly."""
    a = _f64(a)
    h, w = a.shape
    right, down, v = edges(a, c, intrinsics, axes, jump, mask)
    n = int(v.sum())
    kept = kept_edges(right, down)
    lo, hi = depth_range(a, v)
    z = np.full((h, w), np.nan)
    if n == 0 or not hi > lo:
        return dict(z=z, t=np.nan, n=n, kept=kept, status=STATUS_EMPTY if n == 0 else STATUS_FLAT)
    col = -np.ones(h * w, np.int64)
    col[v.ravel()] = np.arange(n)
    p, q, al, be = _edge_list(right, down, h, w)
    cp, cq = col[p], col[q]
    lam = float(weight)
    # the bordered system [[lam I + N, -lam 1], [-lam 1^T, lam n (1 + kappa)]] [z; t] = [lam a; -lam S a] of the
    # energy's stationarity, solved by block elimination with t last (what a direct LU does with t ordered last)
    Hzz = sp.coo_matrix((np.concatenate([np.full(n, lam), al * al, be * be, -al * be, -al * be]),
                         (np.concatenate([np.arange(n), cp, cq, cp, cq]),
                          np.concatenate([np.arange(n), cp, cq, cq, cp]))), shape=(n, n)).tocsc()
    solve = spla.factorized(Hzz)
    av = a[v]
    y = solve(lam * av)
    t = 0.0
    if shift:
        u = solve(np.full(n, lam))                # Hzz^-1 (lam 1)
        t = (-lam * av.sum() + lam * y.sum()) / (lam * n * (1.0 + KAPPA) - lam * u.sum())
        y = y + t * u
    sol = np.append(y, t)
    z[v] = sol[:n]
    return dict(z=z, t=float(t), n=n, kept=kept, status=STATUS_OK)


def system(a, c, intrinsics, weight=0.1, shift=True, jump=0.02, axes=(1, -1, -1), mask=None):
    """(matvec, b, V): matvec(z [H,W]) = M z on V (0 off V), b = weight (a - s(a)) on V."""
    a = _f64(a)
    h, w = a.shape
    right, down, v = edges(a, c, intrinsics, axes, jump, mask)
    p, q, al, be = _edge_list(right, down, h, w)
    n = int(v.sum())
    lam = float(weight)

    def s(x):
        return x[v].sum() / (n * (1.0 + KAPPA)) if shift else 0.0

    def matvec(z):
        z = np.where(v, _f64(z), 0.0)
        zf = z.ravel()
        e = be * zf[q] - al * zf[p]
        nz = np.zeros(h * w)
        np.add.at(nz, p, -al * e)
        np.add.at(nz, q, be * e)
        return np.where(v, lam * (z - s(z)) + nz.reshape(h, w), 0.0)

    b = np.where(v, lam * (np.where(v, a, 0.0) - s(np.where(v, a, 0.0))), 0.0)
    return matvec, b, v


def depth_normals(a, intrinsics, axes=(1, -1, -1), jump=0.02, mask=None):
    """float32 [3,H,W]: the normals of the depth map a [H,W] in the model's encoding (csrc/fusion.cu
    depth_normals_kernel, operation by operation), NaN off V and where a tangent is missing."""
    a = _f64(a)
    h, w = a.shape
    v = valid_set(a, mask)
    lo, hi = depth_range(a, v)
    thr = jump * (hi - lo)
    rx, ry = rays(h, w, intrinsics)
    with np.errstate(invalid="ignore", divide="ignore"):
        X = np.stack([a * rx[None, :], a * ry[:, None], a])
        Xv = np.where(v[None], X, 0.0)

        def shifted(arr, dy, dx, fill):
            out = np.full_like(arr, fill)
            ys, yd = (slice(dy, None), slice(0, h - dy)) if dy >= 0 else (slice(0, h + dy), slice(-dy, None))
            xs, xd = (slice(dx, None), slice(0, w - dx)) if dx >= 0 else (slice(0, w + dx), slice(-dx, None))
            out[..., yd, xd] = arr[..., ys, xs]
            return out

        def tangent(dy, dx):
            vm, vn = shifted(v, -dy, -dx, False), shifted(v, dy, dx, False)
            am, an = shifted(a, -dy, -dx, 0.0), shifted(a, dy, dx, 0.0)
            km = v & vm & (np.abs(a - am) <= thr)
            kn = v & vn & (np.abs(an - a) <= thr)
            Xm, Xn = shifted(Xv, -dy, -dx, 0.0), shifted(Xv, dy, dx, 0.0)
            t = np.where(kn[None], Xn, Xv) - np.where(km[None], Xm, Xv)
            return t, km | kn

        tx, okx = tangent(0, 1)
        ty, oky = tangent(1, 0)
        n = np.stack([ty[1] * tx[2] - ty[2] * tx[1], ty[2] * tx[0] - ty[0] * tx[2], ty[0] * tx[1] - ty[1] * tx[0]])
        n = n / np.sqrt(_dot(n, n))
        sg = np.where(_dot(n, Xv) > 0.0, -1.0, 1.0)
        out = np.stack([(float(axes[k]) * (sg * n[k]) + 1.0) * 0.5 for k in range(3)])
    ok = v & okx & oky
    return np.where(ok[None], out, np.nan).astype(np.float32)


def planes_scene(h, w, intrinsics, seed, strips=3, step=3.0, tilt=1.0):
    """A piecewise-planar depth map [H,W] float64 and its exact normals [3,H,W] in the model's encoding (default axes):
    `strips` vertical strips, each a plane with a seeded tilt through the optical axis at depth 2 + step k, so that
    neighbouring strips are separated by depth steps and no edge joins two planes without one."""
    rng = np.random.default_rng(seed)
    rx, ry = rays(h, w, intrinsics)
    r = np.stack(np.broadcast_arrays(rx[None, :], ry[:, None], np.ones((h, w))))
    z = np.empty((h, w))
    nrm = np.empty((3, h, w))
    bounds = np.linspace(0, w, strips + 1).round().astype(int)
    for k in range(strips):
        nk = np.array([*rng.uniform(-tilt, tilt, 2), -1.0])
        nk /= np.linalg.norm(nk)
        d = nk[2] * (2.0 + step * k)               # n . X = d through (0, 0, 2 + step k)
        sl = slice(bounds[k], bounds[k + 1])
        z[:, sl] = d / np.tensordot(nk, r[:, :, sl], 1)
        nrm[:, :, sl] = nk[:, None, None]
    enc = (np.array([1.0, -1.0, -1.0])[:, None, None] * nrm + 1.0) * 0.5
    return z, enc
