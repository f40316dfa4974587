"""Float64 restatement of the SE(3) pose-graph solve (DESIGN.md §3 "Loop closure and pose graphs", csrc/posegraph.cu)
in numpy: the SE(3) logarithm in the kernel's operation order (numpy rounds every float64 operation once and never
contracts a multiply and an add, like the kernel's __d*_rn operations; numpy's arctan2 and sin / cos agree with the
kernel's to an ulp), the first-order Jacobians, the normal equations assembled densely, the unit-diagonal scaling,
numpy.linalg's Cholesky, the pivot, stop and status rules, and the update T <- T exp(delta) with track_oracle's
exponential.  The sums are not in the kernel's order, so results agree to rounding times the conditioning.

Also helpers that build pose graphs with a known solution for the tests and the profile."""
from __future__ import annotations

import numpy as np

from oracle.track_oracle import SERIES_THETA, _dot, relative_pose, se3_exp

OK, DEGENERATE, NONFINITE = 0, 1, 2
PIVOT_MIN = 1e-12


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def se3_log(T):
    """(r = (v, omega), theta) of a rigid T [4,4] in the kernel's operation order."""
    R, u = T[:3, :3], T[:3, 3]
    w = np.array([0.5 * (R[2, 1] - R[1, 2]), 0.5 * (R[0, 2] - R[2, 0]), 0.5 * (R[1, 0] - R[0, 1])])
    s = np.sqrt(_dot(w, w))
    cth = 0.5 * (((R[0, 0] + R[1, 1]) + R[2, 2]) - 1.0)
    th = float(np.arctan2(s, cth))
    th2 = th * th
    if th < SERIES_THETA:
        th4 = th2 * th2
        f = (1.0 + th2 / 6.0) + (7.0 * th4) / 360.0
        c = (1.0 / 12.0 + th2 / 720.0) + th4 / 30240.0
    else:
        A = np.sin(th) / th
        B = (1.0 - np.cos(th)) / th2
        f = th / s
        c = (1.0 - A / (2.0 * B)) / th2
    om = np.array([f * w[0], f * w[1], f * w[2]])
    o2 = _dot(om, om)
    W = np.array([[0.0, -om[2], om[1]], [om[2], 0.0, -om[0]], [-om[1], om[0], 0.0]])
    r = np.empty(6)
    for i in range(3):
        Vi = [((1.0 if i == j else 0.0) - 0.5 * W[i, j]) + c * (om[i] * om[j] - o2 if i == j else om[i] * om[j])
              for j in range(3)]
        r[i] = _dot(Vi, u)
        r[3 + i] = om[i]
    return r, th


def se3_exp_matrix(xi):
    R, u = se3_exp(xi)
    return _pose(R, u)


def right_update(T, xi):
    """T exp(xi) in the kernel's operation order."""
    Re, u = se3_exp(xi)
    R0, t0 = T[:3, :3], T[:3, 3]
    Tn = np.eye(4)
    for i in range(3):
        for j in range(3):
            Tn[i, j] = (R0[i, 0] * Re[0, j] + R0[i, 1] * Re[1, j]) + R0[i, 2] * Re[2, j]
        Tn[i, 3] = _dot(R0[i], u) + t0[i]
    return Tn


def residual(Ti, Tj, Z):
    """(r, theta, D = Ti^-1 Tj) of one edge: r = Log(Z^-1 Ti^-1 Tj) with the kernel's relative poses."""
    D = _pose(*relative_pose(Ti, Tj))
    M = _pose(*relative_pose(Z, D))
    r, th = se3_log(M)
    return r, th, D


def adjoint(T):
    """Ad(T) = [[R, [t]x R], [0, R]] for (v, omega) twists."""
    R, t = T[:3, :3], T[:3, 3]
    tx = np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])
    A = np.zeros((6, 6))
    A[:3, :3], A[:3, 3:], A[3:, 3:] = R, tx @ R, R
    return A


def jacobians(Ti, Tj, Z):
    """(r, J_i, J_j) with J_i = -Ad(Tj^-1 Ti) and J_j = I (Gauss-Newton's first-order Jacobians)."""
    r, _, D = residual(Ti, Tj, Z)
    return r, -adjoint(np.linalg.inv(D)), np.eye(6)


def cost(poses, edges, Z, W):
    return float(sum(r @ Wk @ r for r, Wk in ((residual(poses[i], poses[j], Z[k])[0], W[k])
                                             for k, (i, j) in enumerate(edges))))


def linearize(poses, edges, Z, W):
    """(H [6(N-1)]^2, g, status) of the free unknowns; status NONFINITE for a NaN or a rotation above pi / 2."""
    n = len(poses)
    m = 6 * (n - 1)
    H, g = np.zeros((m, m)), np.zeros(m)
    status = OK
    for k, (i, j) in enumerate(edges):
        r, th, D = residual(poses[i], poses[j], Z[k])
        Ji = -adjoint(np.linalg.inv(D))
        blocks = {i: Ji, j: np.eye(6)}
        if not (np.isfinite(r).all() and th <= np.pi / 2):
            status = NONFINITE
        for a, Ja in blocks.items():
            if a == 0:
                continue
            g[6 * (a - 1):6 * a] += Ja.T @ W[k] @ r
            for b, Jb in blocks.items():
                if b != 0:
                    H[6 * (a - 1):6 * a, 6 * (b - 1):6 * b] += Ja.T @ W[k] @ Jb
    if not (np.isfinite(H).all() and np.isfinite(g).all()):
        status = NONFINITE
    return H, g, status


def step(poses, edges, Z, W):
    """One Gauss-Newton iteration: (status, new poses, largest |delta|)."""
    H, g, status = linearize(poses, edges, Z, W)
    if status != OK:
        return status, poses, None
    d = np.diag(H)
    if not np.all(d > 0):
        return DEGENERATE, poses, None
    sc = np.sqrt(d)
    try:
        L = np.linalg.cholesky(H / (sc[:, None] * sc[None, :]))
    except np.linalg.LinAlgError:
        return DEGENERATE, poses, None
    if not np.all(np.diag(L) ** 2 >= PIVOT_MIN):
        return DEGENERATE, poses, None
    x = np.linalg.solve(L.T, np.linalg.solve(L, -g / sc)) / sc
    out = [poses[0].copy()]
    dmax = 0.0
    for k in range(1, len(poses)):
        xi = x[6 * (k - 1):6 * k]
        dmax = max(dmax, np.sqrt(_dot(xi[:3], xi[:3])), np.sqrt(_dot(xi[3:], xi[3:])))
        out.append(right_update(poses[k], xi))
    out = np.stack(out)
    if not (np.isfinite(x).all() and np.isfinite(out).all()):
        return NONFINITE, poses, None
    return OK, out, dmax


def optimize(poses, edges, Z, W, iterations=10, tol=1e-8):
    """(poses [N,4,4], record [7]) as PoseGraph.optimize returns them."""
    P0 = np.asarray(poses, np.float64).reshape(-1, 4, 4)
    edges = np.asarray(edges).reshape(-1, 2)
    Z, W = np.asarray(Z, np.float64).reshape(-1, 4, 4), np.asarray(W, np.float64).reshape(-1, 6, 6)
    P, status, iters, dlast = P0.copy(), OK, 0, 0.0
    while iters < iterations:
        iters += 1
        status, P, dmax = step(P, edges, Z, W)
        if status != OK:
            break
        dlast = dmax
        if dmax <= tol:
            break
    if status != OK:
        P = P0.copy()
    c0 = cost(P0, edges, Z, W)
    return P, np.array([status, iters, c0, cost(P, edges, Z, W) if status == OK else c0, dlast, len(P0),
                        len(edges)], np.float64)


def random_rotation(angle, rng):
    a = rng.standard_normal(3)
    return se3_exp_matrix(np.r_[0.0, 0.0, 0.0, a * angle / np.linalg.norm(a)])


def chain_graph(n, rng, loops=0, step=0.05, turn=0.05, noise=(0.0, 0.0), info_scale=(1e4, 1e3)):
    """A random walk of n poses (each `step` m and `turn` rad from the last), odometry edges (k, k + 1) and `loops`
    random loop edges (i, j), j >= i + 2, with measurements the true relative poses times exp of Gaussian noise of
    (position, rotation) standard deviations `noise`, and diagonal information (info_scale[0] on v, [1] on omega,
    each entry scaled by a random factor in [0.5, 2]).  Returns (truth [n,4,4], edges [E,2], Z [E,4,4], W [E,6,6])."""
    T = _walk(n, rng, step, turn)
    edges = [(k, k + 1) for k in range(n - 1)]
    while len(edges) < n - 1 + loops and n > 2:
        i = int(rng.integers(0, n - 2))
        j = int(rng.integers(i + 2, n))
        edges.append((i, j) if rng.random() < 0.5 else (j, i))
    Z, W = [], []
    for i, j in edges:
        xi = np.r_[noise[0] * rng.standard_normal(3), noise[1] * rng.standard_normal(3)]
        Z.append(np.linalg.inv(T[i]) @ T[j] @ se3_exp_matrix(xi))
        W.append(np.diag(np.r_[[info_scale[0]] * 3, [info_scale[1]] * 3] * rng.uniform(0.5, 2.0, 6)))
    Z = np.stack(Z)
    Z[:, :3, :3] = [_orthonormal(R) for R in Z[:, :3, :3]]
    return T, np.array(edges, np.int64), Z, np.stack(W)


def _walk(n, rng, step, turn):
    T = [np.eye(4)]
    for _ in range(n - 1):
        d = rng.standard_normal(3)
        inc = random_rotation(turn, rng)
        inc[:3, 3] = step * d / np.linalg.norm(d)
        T.append(T[-1] @ inc)
    return np.stack(T)


def full_information(rng, scale=1e3, spread=1e2):
    """A random SPD 6 x 6 W = Q diag(lam) Q^T, exactly symmetric, with eigenvalues from scale to scale * spread
    (log-uniform between the two ends, both of which occur) and random eigenvectors Q: v-omega coupling in every
    entry."""
    lam = scale * spread ** np.r_[0.0, 1.0, rng.uniform(0.0, 1.0, 4)]
    Q, _ = np.linalg.qr(rng.standard_normal((6, 6)))
    W = (Q * lam) @ Q.T
    return (W + W.T) / 2


def loop_graph(n, rng, n_edges=None, hubs=(), star=False, reverse=False, step=0.05, turn=0.05, noise=(0.01, 0.01),
               scale=1e3, spread=1e2):
    """A keyframe graph as loop closure builds it: a random walk of n poses (chain_graph's) with
    - odometry edges (k, k + 1), or with `star` one edge between every node and node 0 (and nothing else), so that the
      normal matrix is block-diagonal;
    - for every node h in `hubs`, an edge between h and every other node;
    - random loop edges (i, j), i < j, between any two distinct nodes until there are n_edges edges (parallel edges
      included; at n = 2 every edge joins nodes 0 and 1);
    - with `reverse`, every odd edge listed as (j, i) instead of (i, j) (its measurement taken the other way).
    Measurements are the true relative poses times exp of Gaussian noise of (position, rotation) standard deviations
    `noise`; every W is full_information(rng, scale, spread).  Returns (truth [n,4,4], edges [E,2], Z [E,4,4],
    W [E,6,6]); E <= 8 n is the caller's to respect."""
    T = _walk(n, rng, step, turn)
    if star:
        edges = [(0, k) if rng.random() < 0.5 else (k, 0) for k in range(1, n)]
    else:
        edges = [(k, k + 1) for k in range(n - 1)]
    edges += [(h, k) for h in hubs for k in range(n) if k != h]
    while n_edges is not None and len(edges) < n_edges:
        i, j = sorted(int(v) for v in rng.choice(n, 2, replace=False))
        edges.append((i, j))
    if reverse:
        edges = [(j, i) if e % 2 else (i, j) for e, (i, j) in enumerate(edges)]
    Z, W = [], []
    for i, j in edges:
        xi = np.r_[noise[0] * rng.standard_normal(3), noise[1] * rng.standard_normal(3)]
        Z.append(np.linalg.inv(T[i]) @ T[j] @ se3_exp_matrix(xi))
        W.append(full_information(rng, scale, spread))
    Z = np.stack(Z)
    Z[:, :3, :3] = [_orthonormal(R) for R in Z[:, :3, :3]]
    return T, np.array(edges, np.int64), Z, np.stack(W)


def _orthonormal(R):
    U, _, Vt = np.linalg.svd(R)
    return U @ Vt
