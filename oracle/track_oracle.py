"""Float64 restatement of camera tracking (DESIGN.md §3 "Camera tracking", csrc/track.cu) in numpy: projective
association, point-to-plane residuals, Huber weights and Jacobian rows in the kernel's operation order (numpy rounds
every float64 operation once and never contracts a multiply and an add, like the kernel's __d*_rn operations), the
normal equations assembled densely, the unit-diagonal scaling and pivot rule, numpy.linalg's Cholesky, the SE(3)
exponential, and the stop and status rules.  The sums are not in the kernel's order, so they agree to rounding, and
the kernel's sin and cos (sincospi of theta / pi) agree with numpy's to an ulp.

Also a helper for smooth camera paths through volume_oracle's sphere-in-a-room scene."""
from __future__ import annotations

import numpy as np

from oracle import fusion_oracle, volume_oracle

OK, NO_OVERLAP, DEGENERATE, NONFINITE = 0, 1, 2, 3
PIVOT_MIN = 1e-6
SERIES_THETA = 1e-2


def _dot(u, v):
    return (u[0] * v[0] + u[1] * v[1]) + u[2] * v[2]


def se3_exp(xi):
    """(R [3,3], u [3]) = exp of the twist xi = (v, omega): the rotation and the translation V v."""
    xi = np.asarray(xi, np.float64)
    om = xi[3:6]
    th2 = _dot(om, om)
    th = np.sqrt(th2)
    if th < SERIES_THETA:
        th4 = th2 * th2
        A = (1.0 - th2 / 6.0) + th4 / 120.0
        B = (0.5 - th2 / 24.0) + th4 / 720.0
        C = (1.0 / 6.0 - th2 / 120.0) + th4 / 5040.0
    else:
        sn, cs = np.sin(th), np.cos(th)
        A = sn / th
        B = (1.0 - cs) / th2
        C = (th - sn) / (th2 * th)
    W = np.array([[0.0, -om[2], om[1]], [om[2], 0.0, -om[0]], [-om[1], om[0], 0.0]])
    R, V = np.empty((3, 3)), np.empty((3, 3))
    for i in range(3):
        for j in range(3):
            w2 = om[i] * om[j] - th2 if i == j else om[i] * om[j]
            d = 1.0 if i == j else 0.0
            R[i, j] = (d + A * W[i, j]) + B * w2
            V[i, j] = (d + B * W[i, j]) + C * w2
    return R, np.array([_dot(V[i], xi[:3]) for i in range(3)])


def relative_pose(ref, T):
    """(Rm, tm) of M = ref^-1 T."""
    Rr, tr = ref[:3, :3], ref[:3, 3]
    R, t = T[:3, :3], T[:3, 3]
    Rm = np.empty((3, 3))
    tm = np.empty(3)
    for i in range(3):
        for j in range(3):
            Rm[i, j] = (Rr[0, i] * R[0, j] + Rr[1, i] * R[1, j]) + Rr[2, i] * R[2, j]
        tm[i] = (Rr[0, i] * (t[0] - tr[0]) + Rr[1, i] * (t[1] - tr[1])) + Rr[2, i] * (t[2] - tr[2])
    return Rm, tm


def model_normals(ref_depth, K):
    """The reference normals fp32 [3,H,W] as the tracker computes them (depth_normals, axes (1, 1, 1))."""
    ref = np.asarray(ref_depth, np.float32)
    return fusion_oracle.depth_normals(ref, K, axes=(1, 1, 1), mask=ref > 0)


def associate(pred, ref_depth, normals, K, Rm, tm, s, t, max_dist, robust):
    """Per pixel: dict(valid [H,W], corr [H,W], e, w, J [H,W,8], q) with corr the correspondences."""
    a32 = np.asarray(pred, np.float32)
    h, w = a32.shape
    fx, fy, cx, cy = (float(v) for v in K)
    ref = np.asarray(ref_depth, np.float32)
    nrm = np.asarray(normals, np.float32).reshape(3, h, w)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        a = a32.astype(np.float64)
        z = s * a + t
        valid = np.isfinite(a32) & (z > 0)
        y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
        r = [(x - cx) / fx, (y - cy) / fy, np.ones((h, w))]
        P = [z * r[0], z * r[1], z]
        Q = [_dot(Rm[k], P) + tm[k] for k in range(3)]
        ok = valid & (Q[2] > 0)
        u = np.floor(((fx * Q[0]) / Q[2] + cx) + 0.5)
        v = np.floor(((fy * Q[1]) / Q[2] + cy) + 0.5)
        ok &= (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1)
        ui, vi = np.where(ok, u, 0).astype(np.int64), np.where(ok, v, 0).astype(np.int64)
        dq = ref[vi, ui]
        c = nrm[:, vi, ui]
        ok &= np.isfinite(dq) & (dq > 0) & np.isfinite(c).all(0)
        n = [2.0 * c[k].astype(np.float64) - 1.0 for k in range(3)]
        d = dq.astype(np.float64)
        V = [d * ((u - cx) / fx), d * ((v - cy) / fy), d]
        df = [Q[k] - V[k] for k in range(3)]
        ok &= np.sqrt(_dot(df, df)) <= max_dist
        e = _dot(n, df)
        ae = np.abs(e)
        wt = np.where(ae <= robust, 1.0, robust / ae)
        m = [(Rm[0, j] * n[0] + Rm[1, j] * n[1]) + Rm[2, j] * n[2] for j in range(3)]
        ar = [a * r[0], a * r[1], a]
        J = np.stack([m[0], m[1], m[2], P[1] * m[2] - P[2] * m[1], P[2] * m[0] - P[0] * m[2],
                      P[0] * m[1] - P[1] * m[0], _dot(m, ar), _dot(m, r)], -1)
    return dict(valid=valid, corr=ok, e=np.where(ok, e, 0.0), w=np.where(ok, wt, 0.0),
                J=np.where(ok[..., None], J, 0.0), q=(vi, ui))


def residual(pred, ref_depth, normals, K, Rm, tm, s, t, assoc):
    """e of the pixels of `assoc` at (Rm, tm, s, t) with the association (q, n, V) held fixed: for finite
    differences of the Jacobian."""
    h, w = np.asarray(pred).shape
    fx, fy, cx, cy = (float(v) for v in K)
    a = np.asarray(pred, np.float32).astype(np.float64)
    y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    r = [(x - cx) / fx, (y - cy) / fy, np.ones((h, w))]
    z = s * a + t
    P = [z * r[0], z * r[1], z]
    Q = [_dot(Rm[k], P) + tm[k] for k in range(3)]
    vi, ui = assoc["q"]
    d = np.asarray(ref_depth, np.float32)[vi, ui].astype(np.float64)
    c = np.asarray(normals, np.float32).reshape(3, h, w)[:, vi, ui]
    n = [2.0 * c[k].astype(np.float64) - 1.0 for k in range(3)]
    V = [d * ((ui - cx) / fx), d * ((vi - cy) / fy), d]
    return _dot(n, [Q[k] - V[k] for k in range(3)])


def normal_matrix(A):
    """(H [8,8], g [8]) = (sum w J J^T, sum w J e) over the correspondences of an association A (associate)."""
    J, e, wt = A["J"].reshape(-1, 8), A["e"].reshape(-1), A["w"].reshape(-1)
    return (J * wt[:, None]).T @ J, (J * wt[:, None]).T @ e


def ordered_sum8(parts):
    """Sum over the first axis of parts [P, ...] in common.cuh ordered_sum8's order: lane l adds parts l, l + 8, ... in
    ascending order from 0.0, then the eight lane sums are added in lane order from 0.0 (how track.cu folds its chunk
    partials)."""
    parts = np.asarray(parts, np.float64)
    lanes = []
    for lane in range(8):
        t = np.zeros(parts.shape[1:])
        for p in range(lane, parts.shape[0], 8):
            t = t + parts[p]
        lanes.append(t)
    s = np.zeros(parts.shape[1:])
    for t in lanes:
        s = s + t
    return s


def step(pred, ref_depth, normals, K, ref, T, s, t, affine, robust, max_dist, min_overlap):
    """One Gauss-Newton iteration: (status, T', s', t', stats, xi) with stats = (correspondences, weighted RMS, fraction
    down-weighted, valid pixels) and xi the solved increment (None unless solved)."""
    Rm, tm = relative_pose(ref, T)
    A = associate(pred, ref_depth, normals, K, Rm, tm, s, t, max_dist, robust)
    e, wt = A["e"].reshape(-1), A["w"].reshape(-1)
    H, g = normal_matrix(A)
    count, valid = float(A["corr"].sum()), float(A["valid"].sum())
    wsum, we2 = float(wt.sum()), float((wt * e * e).sum())
    down = float((A["corr"].reshape(-1) & (np.abs(e) > robust)).sum())
    stats = (count, np.sqrt(we2 / wsum) if wsum > 0 else 0.0, down / count if count > 0 else 0.0, valid)
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
    Re, u = se3_exp(x[:6])
    R0, t0 = T[:3, :3], T[:3, 3]
    Tn = np.eye(4)
    for i in range(3):
        for j in range(3):
            Tn[i, j] = (R0[i, 0] * Re[0, j] + R0[i, 1] * Re[1, j]) + R0[i, 2] * Re[2, j]
        Tn[i, 3] = _dot(R0[i], u) + t0[i]
    if not np.isfinite(Tn).all():
        return NONFINITE, T, s, t, stats, None
    return OK, Tn, s + x[6], t + x[7], stats, x


def track(pred, ref_depth, K, ref_pose, init_pose=None, init_nodes=None, affine=True, iterations=20, tol=1e-6,
          robust=0.02, max_dist=0.1, min_overlap=0.1, normals=None):
    """(pose [4,4], nodes (s, t), record [8]) as FrameTracker.track returns them."""
    ref = np.asarray(ref_pose, np.float64).reshape(4, 4)
    T0 = ref.copy() if init_pose is None else np.asarray(init_pose, np.float64).reshape(4, 4)
    normals = model_normals(ref_depth, K) if normals is None else normals
    s0, t0 = (float(init_nodes[0]), float(init_nodes[1])) if affine else (1.0, 0.0)
    T, s, t = T0.copy(), s0, t0
    status, iters, stats = OK, 0, (0.0, 0.0, 0.0, 0.0)
    if not (np.isfinite(s) and np.isfinite(t)):
        status = NONFINITE
    while status == OK and iters < iterations:
        status, T, s, t, stats, x = step(pred, ref_depth, normals, K, ref, T, s, t, affine, robust, max_dist,
                                         min_overlap)
        iters += 1
        if status != OK:
            break
        if np.sqrt(_dot(x[3:6], x[3:6])) <= tol and np.sqrt(_dot(x[:3], x[:3])) <= tol and abs(x[6]) <= tol and \
                abs(x[7]) <= tol:
            break
    if status != OK:
        T, s, t = T0, s0, t0
    return T, (s, t), np.array([stats[0], status, stats[1], stats[2], iters, s, t, stats[3]])


def pose_error(A, B):
    """(position error in metres, rotation error in radians) between two camera-to-world poses."""
    A, B = np.asarray(A, np.float64).reshape(4, 4), np.asarray(B, np.float64).reshape(4, 4)
    c = (np.trace(A[:3, :3].T @ B[:3, :3]) - 1.0) / 2.0
    return float(np.linalg.norm(A[:3, 3] - B[:3, 3])), float(np.arccos(np.clip(c, -1.0, 1.0)))


def perturb(T, dist, angle, rng):
    """T with its position moved by `dist` metres and its orientation turned by `angle` radians, random directions."""
    d = rng.standard_normal(3)
    a = rng.standard_normal(3)
    a *= angle / np.linalg.norm(a)
    th = np.linalg.norm(a)
    k = a / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    out = np.asarray(T, np.float64).copy()
    out[:3, :3] = out[:3, :3] @ R
    out[:3, 3] += dist * d / np.linalg.norm(d)
    return out


def camera_path(n, center, radius=1.2, step_deg=1.5, height=0.25, seed=0):
    """n camera-to-world poses along a smooth arc around center at the given radius (the camera looks at a point
    wandering a few cm around center, with a slow vertical wave): consecutive poses are radius * step_deg apart
    (3.1 cm at the defaults) and turn by about step_deg degrees."""
    rng = np.random.default_rng(seed)
    phase = rng.uniform(0, 2 * np.pi, 3)
    c = np.asarray(center, np.float64)
    out = []
    for q in range(n):
        phi = phase[0] + np.radians(step_deg) * q
        eye = c + np.array([radius * np.cos(phi), radius * np.sin(phi), height * np.sin(0.05 * q + phase[1])])
        target = c + 0.05 * np.array([np.sin(0.11 * q + phase[2]), np.cos(0.07 * q), np.sin(0.05 * q)])
        out.append(volume_oracle.look_at(eye, target))
    return np.stack(out)
