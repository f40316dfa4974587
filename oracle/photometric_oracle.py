"""Float64 restatement of camera tracking with the photometric term (DESIGN.md §3 "Camera tracking", csrc/track.cu
odb_track_frame_rgbd) in numpy, on top of track_oracle's geometric restatement: luminance, the reference's Sobel
gradient as the kernel stores it (rounded to float32), the bilinear association at the unrounded projection, the
intensity residual, its Huber weight and its Jacobian row, in the kernel's operation order; then the joint normal
equations and track_oracle's scaling, pivot, step, stop and status rules.  As there, the sums are not in the kernel's
order, so they agree to rounding."""
from __future__ import annotations

import numpy as np

from oracle import track_oracle as TO
from oracle.track_oracle import DEGENERATE, NO_OVERLAP, NONFINITE, OK, PIVOT_MIN, _dot

LUMA = (0.299, 0.587, 0.114)
STEP_REL = 0.05              # the largest depth step inside a gradient window, relative to the centre's depth


def luminance(rgb):
    """float64 Y = (0.299 R + 0.587 G) + 0.114 B of float32 planes rgb [3, ...]."""
    c = np.asarray(rgb, np.float32).astype(np.float64)
    return (LUMA[0] * c[0] + LUMA[1] * c[1]) + LUMA[2] * c[2]


def intensity_gradient(ref_depth, ref_rgb, normals):
    """float32 [3,H,W] = (Y, g_u, g_v) as the kernel stores them: Y NaN unless the pixel has a surface, a finite colour
    and a usable normal; the 3 x 3 Sobel gradient / 8 NaN unless all 9 window pixels lie in the image, are usable and
    lie within STEP_REL of the centre's depth."""
    d = np.asarray(ref_depth, np.float32)
    h, w = d.shape
    c = np.asarray(ref_rgb, np.float32).reshape(3, h, w)
    nrm = np.asarray(normals, np.float32).reshape(3, h, w)
    with np.errstate(invalid="ignore"):
        usable = np.isfinite(d) & (d > 0) & np.isfinite(c).all(0) & np.isfinite(nrm).all(0)
        Y = np.where(usable, luminance(c), np.nan)
        d64 = d.astype(np.float64)
        ok = np.zeros((h, w), bool)
        ok[1:-1, 1:-1] = True
        ok &= usable
        win = {}
        for j in (-1, 0, 1):
            for k in (-1, 0, 1):
                ys, xs = slice(1 + j, h - 1 + j), slice(1 + k, w - 1 + k)
                m = np.zeros((h, w), bool)
                m[1:-1, 1:-1] = usable[ys, xs] & (np.abs(d64[ys, xs] - d64[1:-1, 1:-1]) <= STEP_REL *
                                                  d64[1:-1, 1:-1])
                ok &= m
                Yw = np.zeros((h, w))
                Yw[1:-1, 1:-1] = np.where(usable[ys, xs], Y[ys, xs], 0.0)
                win[j, k] = Yw
        dx = [win[j, 1] - win[j, -1] for j in (-1, 0, 1)]
        dy = [win[1, k] - win[-1, k] for k in (-1, 0, 1)]
        gu = ((dx[0] + 2.0 * dx[1]) + dx[2]) / 8.0
        gv = ((dy[0] + 2.0 * dy[1]) + dy[2]) / 8.0
    return np.stack([Y, np.where(ok, gu, np.nan), np.where(ok, gv, np.nan)]).astype(np.float32)


def associate(pred, ref_depth, normals, K, Rm, tm, s, t, max_dist, robust):
    """track_oracle.associate, plus what the photometric term reads of each frame pixel: Q, P, r, a and the unrounded
    projection uv = (u, v), in the same operations."""
    A = TO.associate(pred, ref_depth, normals, K, Rm, tm, s, t, max_dist, robust)
    a32 = np.asarray(pred, np.float32)
    h, w = a32.shape
    fx, fy, cx, cy = (float(v) for v in K)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        a = a32.astype(np.float64)
        z = s * a + t
        y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
        r = [(x - cx) / fx, (y - cy) / fy, np.ones((h, w))]
        P = [z * r[0], z * r[1], z]
        Q = [_dot(Rm[k], P) + tm[k] for k in range(3)]
        uv = ((fx * Q[0]) / Q[2] + cx, (fy * Q[1]) / Q[2] + cy)
    return dict(A, Q=Q, P=P, r=r, a=a, uv=uv)


def photometric(A, rgb, intensity, K, Rm, robust_c):
    """The photometric terms of the correspondences of A (associate): dict(corr [H,W], e, w, J [H,W,8], base (bv, bu),
    I (Y, g_u, g_v) at the projection, uv0 the projection)."""
    fx, fy = float(K[0]), float(K[1])
    ig = np.asarray(intensity, np.float32)
    _, h, w = ig.shape
    uf, vf = A["uv"]
    Q, P, r, a = A["Q"], A["P"], A["r"], A["a"]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        bu, bv = np.floor(uf), np.floor(vf)
        ok = A["corr"] & (bu >= 0) & (bu <= w - 2) & (bv >= 0) & (bv <= h - 2)
        ui, vi = np.where(ok, bu, 0).astype(np.int64), np.where(ok, bv, 0).astype(np.int64)
        fu, fv = uf - bu, vf - bv
        lerp = lambda x, y, t: x + t * (y - x)
        I = []
        for c in range(3):
            x00, x10 = ig[c][vi, ui].astype(np.float64), ig[c][vi, ui + 1].astype(np.float64)
            x01, x11 = ig[c][vi + 1, ui].astype(np.float64), ig[c][vi + 1, ui + 1].astype(np.float64)
            ok &= np.isfinite(x00) & np.isfinite(x10) & np.isfinite(x01) & np.isfinite(x11)
            I.append(lerp(lerp(x00, x10, fu), lerp(x01, x11, fu), fv))
        Yf = luminance(rgb)
        ok &= np.isfinite(Yf)
        e = I[0] - Yf
        ae = np.abs(e)
        wt = np.where(ae <= robust_c, 1.0, robust_c / ae)
        gfu, gfv = I[1] * fx, I[2] * fy
        g3 = [gfu / Q[2], gfv / Q[2], -((gfu * Q[0] + gfv * Q[1]) / (Q[2] * Q[2]))]
        m = [(Rm[0, j] * g3[0] + Rm[1, j] * g3[1]) + Rm[2, j] * g3[2] for j in range(3)]
        ar = [a * r[0], a * r[1], a]
        J = np.stack([m[0], m[1], m[2], P[1] * m[2] - P[2] * m[1], P[2] * m[0] - P[0] * m[2],
                      P[0] * m[1] - P[1] * m[0], _dot(m, ar), _dot(m, r)], -1)
    return dict(corr=ok, e=np.where(ok, e, 0.0), w=np.where(ok, wt, 0.0), J=np.where(ok[..., None], J, 0.0),
                base=(vi, ui), I=I, uv0=(uf, vf))


def photometric_residual(pred, rgb, K, Rm, tm, s, t, Ph):
    """e_c at (Rm, tm, s, t) with the association of Ph (photometric) held fixed: the reference intensity linearised at
    the associated projection, Y + g_u (u - u0) + g_v (v - v0), minus the frame's; for finite differences of the
    Jacobian."""
    h, w = np.asarray(pred).shape
    fx, fy, cx, cy = (float(v) for v in K)
    a = np.asarray(pred, np.float32).astype(np.float64)
    y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    r = [(x - cx) / fx, (y - cy) / fy, np.ones((h, w))]
    z = s * a + t
    P = [z * r[0], z * r[1], z]
    Q = [_dot(Rm[k], P) + tm[k] for k in range(3)]
    u, v = (fx * Q[0]) / Q[2] + cx, (fy * Q[1]) / Q[2] + cy
    Y, gu, gv = Ph["I"]
    u0, v0 = Ph["uv0"]
    return (Y + gu * (u - u0) + gv * (v - v0)) - luminance(rgb)


def _stats(corr, e, wt, robust):
    count, wsum, we2 = float(corr.sum()), float(wt.sum()), float((wt * e * e).sum())
    down = float((corr.reshape(-1) & (np.abs(e) > robust)).sum())
    return count, np.sqrt(we2 / wsum) if wsum > 0 else 0.0, down / count if count > 0 else 0.0


def normal_matrix(A, Ph, lam):
    """(H [8,8], g [8]) of one step with both terms: track_oracle.normal_matrix of the geometric association A plus
    lam times sum w_c J_c J_c^T (and sum w_c J_c e_c) over the photometric terms Ph (photometric)."""
    H, g = TO.normal_matrix(A)
    Jc, ec, wc = Ph["J"].reshape(-1, 8), Ph["e"].reshape(-1), Ph["w"].reshape(-1)
    return H + (Jc * (lam * wc)[:, None]).T @ Jc, g + (Jc * (lam * wc)[:, None]).T @ ec


def step(pred, ref_depth, normals, K, ref, T, s, t, affine, robust, max_dist, min_overlap, rgb, intensity, lam,
         robust_c):
    """One Gauss-Newton iteration with both terms: (status, T', s', t', stats, xi) with stats = (correspondences,
    weighted RMS, fraction down-weighted, valid pixels, photometric terms, their weighted RMS, their fraction
    down-weighted) and xi the solved increment (None unless solved)."""
    Rm, tm = TO.relative_pose(ref, T)
    A = associate(pred, ref_depth, normals, K, Rm, tm, s, t, max_dist, robust)
    Ph = photometric(A, rgb, intensity, K, Rm, robust_c)
    e, wt = A["e"].reshape(-1), A["w"].reshape(-1)
    ec, wc = Ph["e"].reshape(-1), Ph["w"].reshape(-1)
    H, g = normal_matrix(A, Ph, lam)
    count, valid = float(A["corr"].sum()), float(A["valid"].sum())
    stats = _stats(A["corr"], e, wt, robust) + (valid,) + _stats(Ph["corr"], ec, wc, robust_c)
    n = 8 if affine else 6
    if not (np.isfinite(H).all() and np.isfinite(g).all()):
        return NONFINITE, T, s, t, stats, None
    if not (valid > 0 and count >= min_overlap * valid and count > 0):
        return NO_OVERLAP, T, s, t, stats, None
    d = np.diag(H)[:n]
    if not np.all(d > 0):
        return DEGENERATE, T, s, t, stats, None
    sc = np.sqrt(d)
    As = H[:n, :n] / (sc[:, None] * sc[None, :])
    try:
        L = np.linalg.cholesky(As)
    except np.linalg.LinAlgError:
        return DEGENERATE, T, s, t, stats, None
    if not np.all(np.diag(L) ** 2 >= PIVOT_MIN):
        return DEGENERATE, T, s, t, stats, None
    y = np.linalg.solve(L.T, np.linalg.solve(L, -(g[:n] / sc)))
    x = np.zeros(8)
    x[:n] = y / sc
    if not np.isfinite(x).all():
        return NONFINITE, T, s, t, stats, None
    Re, u = TO.se3_exp(x[:6])
    R0, t0 = T[:3, :3], T[:3, 3]
    Tn = np.eye(4)
    for i in range(3):
        for j in range(3):
            Tn[i, j] = (R0[i, 0] * Re[0, j] + R0[i, 1] * Re[1, j]) + R0[i, 2] * Re[2, j]
        Tn[i, 3] = _dot(R0[i], u) + t0[i]
    if not np.isfinite(Tn).all():
        return NONFINITE, T, s, t, stats, None
    return OK, Tn, s + x[6], t + x[7], stats, x


def track(pred, ref_depth, K, ref_pose, rgb, ref_rgb, init_pose=None, init_nodes=None, affine=True, iterations=20,
          tol=1e-6, robust=0.02, max_dist=0.1, min_overlap=0.1, photometric=1e-2, photometric_robust=0.1,
          normals=None):
    """(pose [4,4], nodes (s, t), record [11]) as FrameTracker(photometric=...).track returns them (photometric > 0)."""
    ref = np.asarray(ref_pose, np.float64).reshape(4, 4)
    T0 = ref.copy() if init_pose is None else np.asarray(init_pose, np.float64).reshape(4, 4)
    normals = TO.model_normals(ref_depth, K) if normals is None else normals
    intensity = intensity_gradient(ref_depth, ref_rgb, normals)
    s0, t0 = (float(init_nodes[0]), float(init_nodes[1])) if affine else (1.0, 0.0)
    T, s, t = T0.copy(), s0, t0
    status, iters, stats = OK, 0, (0.0,) * 7
    if not (np.isfinite(s) and np.isfinite(t)):
        status = NONFINITE
    while status == OK and iters < iterations:
        status, T, s, t, stats, x = step(pred, ref_depth, normals, K, ref, T, s, t, affine, robust, max_dist,
                                         min_overlap, rgb, intensity, photometric, photometric_robust)
        iters += 1
        if status != OK:
            break
        if np.sqrt(_dot(x[3:6], x[3:6])) <= tol and np.sqrt(_dot(x[:3], x[:3])) <= tol and abs(x[6]) <= tol and \
                abs(x[7]) <= tol:
            break
    if status != OK:
        T, s, t = T0, s0, t0
    return T, (s, t), np.array([stats[0], status, stats[1], stats[2], iters, s, t, stats[3], *stats[4:]])
