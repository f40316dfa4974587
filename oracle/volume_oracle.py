"""Float64 restatement of the TSDF volume (DESIGN.md §3 "TSDF volumes", csrc/volume.cu) in numpy, for small grids:
integration, raycasting and marching-tetrahedra extraction, in the kernels' operation order (numpy performs every
float64 operation with one rounding and never contracts a multiply and an add, like the kernels' __d*_rn operations;
the running means are float32 operations as the definition states).  Also an analytic scene: a sphere inside a box
room, rendered to exact depth maps by ray-primitive intersection in float64.

Arrays follow the device layout: F, W float32 [nz, ny, nx], colour float32 [3, nz, ny, nx]; a pose is a 4 x 4
camera-to-world matrix."""
from __future__ import annotations

import numpy as np

# Kuhn split: corner codes (bit 0 x, bit 1 y, bit 2 z) of tetrahedron q = the q-th permutation of the axes; odd
# permutations give negatively oriented tetrahedra
TET_CORNER = np.array([[0, 1, 3, 7], [0, 1, 5, 7], [0, 2, 3, 7], [0, 2, 6, 7], [0, 4, 5, 7], [0, 4, 6, 7]])
TET_ODD = np.array([0, 1, 1, 0, 0, 1])
TET_EDGE = np.array([[0, 1], [0, 2], [0, 3], [1, 2], [1, 3], [2, 3]])
# triangles (edge indices) of a positively oriented tetrahedron by the mask of its corners with F < 0; -1: none
TET_TRI = np.array([
    [[-1, -1, -1], [-1, -1, -1]], [[0, 1, 2], [-1, -1, -1]], [[0, 4, 3], [-1, -1, -1]], [[1, 2, 4], [1, 4, 3]],
    [[1, 3, 5], [-1, -1, -1]], [[0, 5, 2], [0, 3, 5]], [[0, 4, 5], [0, 5, 1]], [[2, 4, 5], [-1, -1, -1]],
    [[2, 5, 4], [-1, -1, -1]], [[0, 1, 5], [0, 5, 4]], [[0, 5, 3], [0, 2, 5]], [[1, 5, 3], [-1, -1, -1]],
    [[1, 3, 4], [1, 4, 2]], [[0, 3, 4], [-1, -1, -1]], [[0, 2, 1], [-1, -1, -1]], [[-1, -1, -1], [-1, -1, -1]]])


def corner_vec(code):
    return np.array([code & 1, (code >> 1) & 1, (code >> 2) & 1], dtype=np.float64)


def kuhn_volumes() -> np.ndarray:
    """Signed volumes of the 6 tetrahedra of the unit cell (v0, v1, v2, v3)."""
    out = []
    for q in range(6):
        v = [corner_vec(c) for c in TET_CORNER[q]]
        out.append(np.linalg.det(np.stack([v[1] - v[0], v[2] - v[0], v[3] - v[0]])) / 6.0)
    return np.array(out)


def _indices(dims, index_offset=(0, 0, 0)):
    """float64 (i, j, k) [nz, ny, nx] of the points of a dims grid whose first point is index_offset of a larger
    grid (integers, so exact)."""
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    return [(q + int(o)).astype(np.float64) for q, o in zip((i, j, k), index_offset)]


def _points(dims, origin, voxel, index_offset=(0, 0, 0)):
    """X = origin + voxel (i, j, k) of the points of a dims grid; index_offset: the grid is the sub-box of a larger grid
    starting at that point, whose positions the kernels compute from the larger grid's indices."""
    idx = _indices(dims, index_offset)
    return [origin[a] + voxel * idx[a] for a in range(3)]


def integrate(F, W, C, origin, voxel, trunc, depth, K, poses, rgb=None, index_offset=(0, 0, 0)):
    """(F, W, C) after integrating depth [B,H,W] (rgb [B,3,H,W] with C) from poses [B,4,4]; new arrays.
    index_offset: F, W, C are the sub-box from that point of a larger grid with this origin and voxel."""
    F, W = F.astype(np.float32).copy(), W.astype(np.float32).copy()
    C = None if C is None else C.astype(np.float32).copy()
    nz, ny, nx = F.shape
    X, Y, Z = _points((nx, ny, nz), origin, voxel, index_offset)
    fx, fy, cx, cy = (float(v) for v in K)
    depth = np.asarray(depth, np.float32)
    _, h, w = depth.shape
    for b, T in enumerate(np.asarray(poses, np.float64).reshape(-1, 4, 4)):
        R, t = T[:3, :3], T[:3, 3]
        dx, dy, dz = X - t[0], Y - t[1], Z - t[2]
        zc = (R[0, 2] * dx + R[1, 2] * dy) + R[2, 2] * dz
        xc = (R[0, 0] * dx + R[1, 0] * dy) + R[2, 0] * dz
        yc = (R[0, 1] * dx + R[1, 1] * dy) + R[2, 1] * dz
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            u = np.floor((fx * xc) / zc + cx + 0.5)
            v = np.floor((fy * yc) / zc + cy + 0.5)
            ok = (zc > 0) & (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1)
        ui, vi = np.where(ok, u, 0).astype(np.int64), np.where(ok, v, 0).astype(np.int64)
        d = depth[b][vi, ui]
        with np.errstate(invalid="ignore"):
            ok &= np.isfinite(d) & (d > 0)
            eta = d.astype(np.float64) - zc
            ok &= ~(eta < -trunc)
            f = np.minimum(1.0, eta / trunc).astype(np.float32)
            w1 = W + np.float32(1)
            F = np.where(ok, (F * W + f) / w1, F).astype(np.float32)
            if C is not None:
                for a in range(3):
                    c = np.asarray(rgb, np.float32)[b, a][vi, ui]
                    C[a] = np.where(ok, (C[a] * W + c) / w1, C[a])
            W = np.where(ok, w1, W).astype(np.float32)
    return F, W, C


def raycast(F, W, origin, voxel, K, pose, size, step=None):
    """z-depth float32 [H,W] of the first + to - crossing of valid trilinear samples, 0 where none."""
    nz, ny, nx = F.shape
    n = (nx, ny, nz)
    h, w = size
    step = 0.5 * voxel if step is None else step
    fx, fy, cx, cy = (float(v) for v in K)
    T = np.asarray(pose, np.float64).reshape(4, 4)
    y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    rx, ry = (x - cx) / fx, (y - cy) / fy
    nrm = np.sqrt((rx * rx + ry * ry) + 1.0)
    ux, uy, uz = rx / nrm, ry / nrm, 1.0 / nrm
    d = [(T[a, 0] * ux + T[a, 1] * uy) + T[a, 2] * uz for a in range(3)]
    o = [np.full((h, w), T[a, 3]) for a in range(3)]
    t0, t1 = np.zeros((h, w)), np.full((h, w), np.inf)
    miss = np.zeros((h, w), bool)
    for a in range(3):
        lo = float(origin[a])
        hi = lo + voxel * float(n[a] - 1)
        zero = d[a] == 0.0
        miss |= zero & ((o[a] < lo) | (o[a] > hi))
        with np.errstate(divide="ignore", invalid="ignore"):
            ta, tb = (lo - o[a]) / d[a], (hi - o[a]) / d[a]
        t0 = np.where(zero, t0, np.maximum(t0, np.minimum(ta, tb)))
        t1 = np.where(zero, t1, np.minimum(t1, np.maximum(ta, tb)))
    Ff, Wf = F.reshape(-1).astype(np.float64), W.reshape(-1)
    sy, sz = nx, nx * ny

    def sample(t):
        c, fr = [], []
        for a in range(3):
            g = ((o[a] + t * d[a]) - float(origin[a])) / voxel
            fl = np.minimum(np.maximum(np.floor(g), 0.0), float(n[a] - 2))
            c.append(fl.astype(np.int64))
            fr.append(np.minimum(np.maximum(g - fl, 0.0), 1.0))
        base = c[0] + c[1] * sy + c[2] * sz
        ok = np.ones(base.shape, bool)
        cv = []
        for q in range(4):
            e = base + (q & 1) * sy + (q >> 1) * sz
            ok &= (Wf[e] > 0) & (Wf[e + 1] > 0)
            a0, a1 = Ff[e], Ff[e + 1]
            cv.append(a0 + fr[0] * (a1 - a0))
        lerp = lambda a, b, s: a + s * (b - a)
        return ok, lerp(lerp(cv[0], cv[1], fr[1]), lerp(cv[2], cv[3], fr[1]), fr[2])

    out = np.zeros((h, w), np.float32)
    live = ~miss & (t0 <= t1)
    prev_ok, prev, tp = np.zeros((h, w), bool), np.zeros((h, w)), t0.copy()
    s = 0
    while live.any():
        t = t0 + float(s) * step
        live &= t <= t1
        tt = np.where(live, t, t0)
        ok, val = sample(np.where(np.isfinite(tt), tt, 0.0))
        hit = live & ok & prev_ok & (prev > 0) & (val <= 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            th = tp + step * (prev / (prev - val))
        out = np.where(hit, (th * uz).astype(np.float32), out)
        live &= ~hit
        prev_ok, prev, tp = ok, val, tt
        s += 1
    return out


def _shift(a, code, fill):
    """a[k + dz, j + dy, i + dx] for the corner code, `fill` outside the grid."""
    dx, dy, dz = code & 1, (code >> 1) & 1, (code >> 2) & 1
    out = np.full_like(a, fill)
    nz, ny, nx = a.shape
    out[:nz - dz, :ny - dy, :nx - dx] = a[dz:, dy:, dx:]
    return out


def extract_mesh(F, W, C, origin, voxel, index_offset=(0, 0, 0)):
    """(vertices float32 [V,3], faces int32 [F,3], colors float32 [V,3] or None) in the kernels' order.
    index_offset: F, W, C are the sub-box from that point of a larger grid with this origin and voxel, whose points
    outside the sub-box have W = 0; the vertices are the larger grid's, and the face ids count from the sub-box's
    first vertex."""
    nz, ny, nx = F.shape
    N = F.size
    obs = [_shift(W, c, 0.0).reshape(-1) > 0 for c in range(8)]
    fv = [_shift(F, c, 0.0).reshape(-1) for c in range(8)]
    neg = [f < 0 for f in fv]
    bits = np.stack([obs[0] & obs[c] & (neg[0] != neg[c]) for c in range(1, 8)], axis=1)      # [N, 7]
    mask = (bits * (1 << np.arange(7))).sum(1)
    counts = bits.sum(1)
    vbase = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    idx = [q.reshape(-1) for q in _indices((nx, ny, nz), index_offset)]
    verts, cols = [], []
    fp = fv[0].astype(np.float64)
    for c in range(1, 8):
        with np.errstate(divide="ignore", invalid="ignore"):
            s = fp / (fp - fv[c].astype(np.float64))
        d = corner_vec(c)
        verts.append(np.stack([float(origin[a]) + voxel * (idx[a] + (s if d[a] else 0.0)) for a in range(3)], 1))
        if C is not None:
            cp = [C[a].reshape(-1).astype(np.float64) for a in range(3)]
            cq = [_shift(C[a], c, 0.0).reshape(-1).astype(np.float64) for a in range(3)]
            with np.errstate(invalid="ignore"):
                cols.append(np.stack([cp[a] + s * (cq[a] - cp[a]) for a in range(3)], 1))
    V = np.stack(verts, 1)[bits].astype(np.float32)                  # [N, 7, 3] selected in (point, direction) order
    Cv = np.stack(cols, 1)[bits].astype(np.float32) if C is not None else None
    cell = ((i < nx - 1) & (j < ny - 1) & (k < nz - 1)).reshape(-1)
    p = np.arange(N)
    off = lambda code: (code & 1) + ((code >> 1) & 1) * nx + ((code >> 2) & 1) * nx * ny
    tris = np.full((N, 6, 2, 3), -1, np.int64)
    valid = np.zeros((N, 6, 2), bool)
    for q in range(6):
        corners = TET_CORNER[q]
        all_obs = cell.copy()
        m = np.zeros(N, np.int64)
        for v, c in enumerate(corners):
            all_obs &= obs[c]
            m |= neg[c].astype(np.int64) << v
        for t in range(2):
            ok = all_obs & (TET_TRI[m, t, 0] >= 0)
            valid[:, q, t] = ok
            ids = []
            for e in range(3):
                edge = TET_TRI[m, t, e]
                a, b = TET_EDGE[np.maximum(edge, 0), 0], TET_EDGE[np.maximum(edge, 0), 1]
                ca, cb = corners[a], corners[b]
                owner = np.where(ok, p + off(ca), 0)
                dirn = (ca ^ cb) - 1
                ids.append(vbase[owner] + _popcount(mask[owner] & ((1 << dirn) - 1)))
            if TET_ODD[q]:
                ids = [ids[0], ids[2], ids[1]]
            tris[:, q, t] = np.stack(ids, 1)
    faces = tris[valid].astype(np.int32)
    return V, faces, Cv


def _popcount(x):
    x = np.asarray(x, np.int64)
    return sum((x >> b) & 1 for b in range(7))


# ---------------------------------------------------------------- analytic scene
def sphere_room_depth(K, pose, size, center, radius, room_lo, room_hi):
    """Exact z-depth float64 [H,W] of a sphere inside a box room (the camera inside the room, outside the sphere): the
    nearer of the ray's sphere entry and its exit through the room's walls."""
    h, w = size
    fx, fy, cx, cy = K
    T = np.asarray(pose, np.float64)
    y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    r = np.stack([(x - cx) / fx, (y - cy) / fy, np.ones_like(x)], -1)          # z component 1: s is the z-depth
    d = r @ T[:3, :3].T
    o = T[:3, 3]
    oc = o - np.asarray(center, np.float64)
    a = (d * d).sum(-1)
    b = 2.0 * (d @ oc)
    c = oc @ oc - radius * radius
    disc = b * b - 4 * a * c
    with np.errstate(invalid="ignore", divide="ignore"):
        s_sph = np.where(disc >= 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), np.inf)
        s_sph = np.where(s_sph > 0, s_sph, np.inf)
        walls = [np.where(d[..., q] > 0, (room_hi[q] - o[q]) / d[..., q],
                          np.where(d[..., q] < 0, (room_lo[q] - o[q]) / d[..., q], np.inf)) for q in range(3)]
    return np.minimum(s_sph, np.minimum.reduce(walls))


def look_at(eye, target, up=(0.0, 0.0, 1.0)):
    """Camera-to-world [4,4] (OpenCV frame) at eye looking at target."""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    z = target - eye
    z /= np.linalg.norm(z)
    up = np.asarray(up, np.float64)
    if abs(z @ up) > 0.99:
        up = np.array([0.0, 1.0, 0.0])
    x = np.cross(z, up)                       # y = z x x points down when up is up
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, y, z, eye
    return T


def orbit_poses(n, radius, center=(0.0, 0.0, 0.0)):
    """n look-at poses on a Fibonacci sphere of the given radius around center."""
    out = []
    g = np.pi * (3.0 - np.sqrt(5.0))
    for q in range(n):
        zq = 1.0 - 2.0 * (q + 0.5) / n
        rq = np.sqrt(1.0 - zq * zq)
        e = np.asarray(center) + radius * np.array([rq * np.cos(g * q), rq * np.sin(g * q), zq])
        out.append(look_at(e, center))
    return np.stack(out)


def sphere_sdf_volume(dims, origin, voxel, center, radius, trunc):
    """(F, W) float32 of a sphere's signed distance, truncated to [-1, 1] in units of trunc, W = 1 everywhere."""
    X, Y, Z = _points(dims, origin, voxel)
    dist = np.sqrt((X - center[0]) ** 2 + (Y - center[1]) ** 2 + (Z - center[2]) ** 2) - radius
    return np.clip(dist / trunc, -1.0, 1.0).astype(np.float32), np.ones(X.shape, np.float32)


def mesh_edges(faces):
    """Undirected index edges [E, 2] with multiplicity: (unique edges, count per edge)."""
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    e = np.sort(e, axis=1)
    return np.unique(e, axis=0, return_counts=True)


def signed_volume(vertices, faces):
    v = vertices.astype(np.float64)[faces]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


def face_normals(vertices, faces):
    v = vertices.astype(np.float64)[faces]
    return np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
