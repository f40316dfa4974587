"""Float64 restatement of the mesh metrics (csrc/mesh_metrics.cu; DESIGN.md §3 "Mesh metrics"): the surface sampler
operation by operation (the counter-based generator is exact in numpy uint64), nearest neighbours by brute force or
through scipy's cKDTree candidates with the distance recomputed in the kernel's order, frustum culling, the metric
definitions, and an exact ground-truth mesh of the analytic sphere-in-a-room scene the volume tests render."""
from __future__ import annotations

import math

import numpy as np

def splitmix64(x) -> np.ndarray:
    z = np.asarray(x, dtype=np.uint64) + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def stream_key(seed: int, stream: int) -> np.uint64:
    return splitmix64(splitmix64(np.array([seed], np.uint64)) ^ np.uint64(stream))[0]


def draw(key, t, j) -> np.ndarray:
    """u(t, j) = (splitmix64(splitmix64(key ^ t) ^ j) >> 11) 2^-53."""
    x = splitmix64(splitmix64(np.uint64(key) ^ np.asarray(t, np.uint64)) ^ np.asarray(j, np.uint64))
    return (x >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def face_areas(vertices, faces) -> np.ndarray:
    v = np.asarray(vertices, np.float32).astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    e1, e2 = b - a, c - a
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    return 0.5 * np.sqrt((cx * cx + cy * cy) + cz * cz)


def sample_counts(vertices, faces, density, seed=0, stream=0) -> np.ndarray:
    """n_t = floor(A_t density + u(t, 0)) per face, int64 [F]."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    key = stream_key(seed, stream)
    t = np.arange(len(faces), dtype=np.uint64)
    with np.errstate(invalid="ignore", over="ignore"):
        x = np.floor(face_areas(vertices, faces) * float(density) + draw(key, t, 0))
    return np.where(x < 2.0 ** 31, x, 2.0 ** 31).astype(np.int64)


def sample_surface(vertices, faces, density, seed=0, stream=0):
    """(counts int64 [F], points fp32 [N,3]) of the sampler, in (face, k) order.  ValueError as the device raises."""
    v = np.asarray(vertices, np.float32)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    if faces.size and (faces.min() < 0 or faces.max() >= len(v)):
        raise ValueError("a face index lies outside the vertices")
    if faces.size and not np.isfinite(v[np.unique(faces)]).all():
        raise ValueError("a face uses a non-finite vertex")
    n = sample_counts(v, faces, density, seed, stream)
    key = stream_key(seed, stream)
    t = np.repeat(np.arange(len(faces), dtype=np.int64), n)
    k = np.arange(int(n.sum()), dtype=np.int64) - np.repeat(np.cumsum(n) - n, n)
    r1 = draw(key, t.astype(np.uint64), (2 * k + 1).astype(np.uint64))
    r2 = draw(key, t.astype(np.uint64), (2 * k + 2).astype(np.uint64))
    s = np.sqrt(r1)
    w0, w1, w2 = 1.0 - s, s * (1.0 - r2), s * r2
    vd = v.astype(np.float64)
    a, b, c = vd[faces[t, 0]], vd[faces[t, 1]], vd[faces[t, 2]]
    p = (w0[:, None] * a + w1[:, None] * b) + w2[:, None] * c
    return n, p.astype(np.float32)


def _d2(q, r):
    """(dx^2 + dy^2) + dz^2 in float64, q [M,3] against r [K,3] or [M,K,3]."""
    d = q.astype(np.float64)[:, None, :] - r.astype(np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def nearest_brute(query, reference, chunk=1024):
    """(distance float64 [M], index int32 [M]) by exhaustive search: the minimal d^2, ties to the smallest index."""
    q, r = np.asarray(query, np.float32), np.asarray(reference, np.float32)
    if len(r) == 0:
        return np.full(len(q), np.inf), np.full(len(q), -1, np.int32)
    dist, idx = np.empty(len(q)), np.empty(len(q), np.int32)
    for s in range(0, len(q), chunk):
        d2 = _d2(q[s:s + chunk], r[None])
        j = np.argmin(d2, axis=1)                              # the first minimum: the smallest index
        idx[s:s + chunk] = j
        dist[s:s + chunk] = np.sqrt(d2[np.arange(len(j)), j])
    return dist, idx


def nearest_kdtree(query, reference, k=16):
    """nearest_brute's result through cKDTree candidates: the k nearest by the tree, the distance recomputed in the
    kernel's order; queries whose k-th candidate lies within a relative 1e-9 of the nearest (near-ties the tree may
    order differently) are searched among all points within that radius."""
    from scipy.spatial import cKDTree
    q, r = np.asarray(query, np.float32), np.asarray(reference, np.float32)
    if len(r) == 0:
        return np.full(len(q), np.inf), np.full(len(q), -1, np.int32)
    k = min(k, len(r))
    tree = cKDTree(r.astype(np.float64))
    kd, ki = tree.query(q.astype(np.float64), k=k, workers=-1)
    kd, ki = kd.reshape(len(q), k), ki.reshape(len(q), k)
    d2 = _d2(q, r[ki])
    best = d2.min(1)
    cand = np.where(d2 == best[:, None], ki, np.iinfo(np.int64).max)
    idx = cand.min(1)
    radius = np.sqrt(best) * (1 + 1e-9) + 1e-12
    open_ = (kd[:, -1] <= radius) if k < len(r) else np.zeros(len(q), bool)
    for i in np.flatnonzero(open_):
        js = np.asarray(tree.query_ball_point(q[i].astype(np.float64), radius[i] * (1 + 1e-9) + 1e-12), np.int64)
        dd = _d2(q[i:i + 1], r[js][None])[0]
        m = dd.min()
        best[i], idx[i] = m, js[dd == m].min()
    return np.sqrt(best), idx.astype(np.int32)


def frustum_mask(points, K, size, poses, max_depth=10.0) -> np.ndarray:
    """uint8 [N]: 1 where a camera sees the point (odb_tsdf_integrate's projection and nearest-pixel rule)."""
    X = np.asarray(points, np.float32).astype(np.float64)
    fx, fy, cx, cy = K
    h, w = size
    seen = np.zeros(len(X), bool)
    for T in np.asarray(poses, np.float64).reshape(-1, 4, 4):
        m = T.reshape(16)
        dx, dy, dz = X[:, 0] - m[3], X[:, 1] - m[7], X[:, 2] - m[11]
        zc = (m[2] * dx + m[6] * dy) + m[10] * dz
        xc = (m[0] * dx + m[4] * dy) + m[8] * dz
        yc = (m[1] * dx + m[5] * dy) + m[9] * dz
        ok = (zc > 0) & (zc <= max_depth)
        with np.errstate(divide="ignore", invalid="ignore"):
            u = np.floor(((fx * xc) / zc + cx) + 0.5)
            v = np.floor(((fy * yc) / zc + cy) + 0.5)
        seen |= ok & (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1)
    return seen.astype(np.uint8)


def scene_record(dp, dg, thresholds):
    """The per-scene record (n_pred, n_gt, accuracy, completion, chamfer, (precision, recall, F) per threshold), NaN
    where undefined, from the distances of each side's samples to the other side."""
    dp, dg = np.asarray(dp, np.float64), np.asarray(dg, np.float64)
    rec = [float(len(dp)), float(len(dg))] + [math.nan] * 15
    if len(dg) == 0:
        return rec
    for k, t in enumerate(thresholds):
        P = float((dp < t).sum()) / len(dp) if len(dp) else 0.0
        R = float((dg < t).sum()) / len(dg)
        rec[5 + 3 * k: 8 + 3 * k] = [P, R, (2 * P * R) / (P + R) if P + R > 0 else 0.0]
    if len(dp):
        acc, comp = math.fsum(dp) / len(dp), math.fsum(dg) / len(dg)
        rec[2:5] = [acc, comp, (acc + comp) * 0.5]
    return rec


# ---------------------------------------------------------------- the analytic scene's ground truth
def icosphere(subdiv: int):
    """(unit vertices float64 [V,3], faces int64 [F,3] wound outward) of the icosahedron subdivided subdiv times."""
    p = (1 + math.sqrt(5)) / 2
    v = np.array([[-1, p, 0], [1, p, 0], [-1, -p, 0], [1, -p, 0], [0, -1, p], [0, 1, p], [0, -1, -p], [0, 1, -p],
                  [p, 0, -1], [p, 0, 1], [-p, 0, -1], [-p, 0, 1]], np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5],
                  [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], np.int64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    for _ in range(subdiv):
        e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
        uniq, inv = np.unique(e, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        mid = v[uniq[:, 0]] + v[uniq[:, 1]]
        mid /= np.linalg.norm(mid, axis=1, keepdims=True)
        m = len(v) + inv.reshape(3, -1).T                     # the midpoints of edges (01, 12, 20) of each face
        v = np.concatenate([v, mid])
        a, b, c = f[:, 0], f[:, 1], f[:, 2]
        m01, m12, m20 = m[:, 0], m[:, 1], m[:, 2]
        f = np.concatenate([np.stack([a, m01, m20], 1), np.stack([b, m12, m01], 1), np.stack([c, m20, m12], 1),
                            np.stack([m01, m12, m20], 1)])
    return v, f


def box_surface(lo, hi, n: int):
    """(vertices float64 [V,3], faces int64 [F,3]) of the closed surface of the box [lo, hi], n x n quads per side
    (two triangles each), wound inward (normals into the box)."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    keys, tris = [], []
    u, w = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    u, w = u.reshape(-1), w.reshape(-1)
    for a in range(3):
        b, c = (a + 1) % 3, (a + 2) % 3
        for side in (0, n):
            corner = []
            for du, dw in ((0, 0), (1, 0), (1, 1), (0, 1)):
                g = np.zeros((len(u), 3), np.int64)
                g[:, a], g[:, b], g[:, c] = side, u + du, w + dw
                corner.append(g)
            q0, q1, q2, q3 = corner
            # (b, c, a) is right-handed: the quad (q0, q1, q2, q3) has normal +a, inward on the side at 0
            t = [(q0, q1, q2), (q0, q2, q3)] if side == 0 else [(q0, q2, q1), (q0, q3, q2)]
            for tri in t:
                tris.append(np.stack(tri, 1))
    g = np.concatenate(tris).reshape(-1, 3)
    uniq, inv = np.unique(g, axis=0, return_inverse=True)
    verts = lo + (hi - lo) * (uniq / n)
    verts[uniq == n] = np.broadcast_to(hi, uniq.shape)[uniq == n]             # the far faces exactly at hi
    return verts, inv.reshape(-1, 3)


def sphere_room_mesh(center, radius, room_lo, room_hi, subdiv: int = 6):
    """Exact ground-truth mesh (vertices float64 [V,3], faces int64 [F,3]) of the analytic scene: the room's six faces
    (2^subdiv x 2^subdiv quads each, wound into the room) and an icosphere (subdivided subdiv times, vertices on the
    sphere, wound outward).  At subdivision 6 the sphere's chord error is about 17 um at radius 0.5 m."""
    rv, rf = box_surface(room_lo, room_hi, 2 ** subdiv)
    sv, sf = icosphere(subdiv)
    sv = np.asarray(center, np.float64) + radius * sv
    return np.concatenate([rv, sv]), np.concatenate([rf, sf + len(rv)])
