"""Float64 restatement of the coloured TSDF raycast (DESIGN.md §3 "TSDF volumes", csrc/volume.cu
odb_tsdf_raycast_color) in numpy, in the kernel's operation order, and a smooth solid texture for volume_oracle's
analytic sphere-in-a-room scene, so that its frames come with exact colour.

Arrays follow volume_oracle's device layout: F, W float32 [nz, ny, nx], colour float32 [3, nz, ny, nx]."""
from __future__ import annotations

import numpy as np

from oracle import volume_oracle

# the solid texture of sphere_room_rgb: unit wave vectors (none along an axis), wavelengths in metres, amplitudes
TEXTURE_DIRS = np.array([[0.48, 0.64, 0.6], [-0.72, 0.3, 0.625], [0.2, -0.85, 0.487]])
TEXTURE_DIRS /= np.linalg.norm(TEXTURE_DIRS, axis=1, keepdims=True)
TEXTURE_WAVELENGTHS = (0.15, 0.2, 0.25)
TEXTURE_AMPLITUDES = (0.2, 0.15, 0.1)


def raycast_color(F, W, C, origin, voxel, K, pose, size, step=None):
    """(depth float32 [H,W], rgb float32 [3,H,W]): depth as volume_oracle.raycast (the first + to - crossing of valid
    trilinear samples, 0 where none) and the colour at the hit, trilinear in C at the two samples bracketing the crossing
    (the same corners and x, y, z order as F), blended by the crossing's fraction; NaN where nothing is hit."""
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
    lerp = lambda a, b, s: a + s * (b - a)

    def locate(t):
        c, fr = [], []
        for a in range(3):
            g = ((o[a] + t * d[a]) - float(origin[a])) / voxel
            fl = np.minimum(np.maximum(np.floor(g), 0.0), float(n[a] - 2))
            c.append(fl.astype(np.int64))
            fr.append(np.minimum(np.maximum(g - fl, 0.0), 1.0))
        return c[0] + c[1] * sy + c[2] * sz, fr

    def trilinear(V, base, fr):
        cv = [lerp(V[base + (q & 1) * sy + (q >> 1) * sz], V[base + (q & 1) * sy + (q >> 1) * sz + 1], fr[0])
              for q in range(4)]
        return lerp(lerp(cv[0], cv[1], fr[1]), lerp(cv[2], cv[3], fr[1]), fr[2])

    def sample(t):
        base, fr = locate(t)
        ok = np.ones(base.shape, bool)
        for q in range(4):
            e = base + (q & 1) * sy + (q >> 1) * sz
            ok &= (Wf[e] > 0) & (Wf[e + 1] > 0)
        return ok, trilinear(Ff, base, fr)

    out = np.zeros((h, w), np.float32)
    hit_any = np.zeros((h, w), bool)
    t_lo, t_hi, frac = np.zeros((h, w)), np.zeros((h, w)), np.zeros((h, w))
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
            fk = prev / (prev - val)
            th = tp + step * fk
        out = np.where(hit, (th * uz).astype(np.float32), out)
        hit_any |= hit
        t_lo, t_hi, frac = np.where(hit, tp, t_lo), np.where(hit, tt, t_hi), np.where(hit, fk, frac)
        live &= ~hit
        prev_ok, prev, tp = ok, val, tt
        s += 1
    rgb = np.full((3, h, w), np.nan, np.float32)
    b0, f0 = locate(t_lo)
    b1, f1 = locate(t_hi)
    for a in range(3):
        Ca = np.asarray(C[a], np.float32).reshape(-1).astype(np.float64)
        c = lerp(trilinear(Ca, b0, f0), trilinear(Ca, b1, f1), frac)
        rgb[a] = np.where(hit_any, c.astype(np.float32), np.nan)
    return out, rgb


def texture_rgb(X):
    """float64 [3, ...] colour in [0.05, 0.95] of world points X [..., 3]: per channel 0.5 plus three sinusoids on the
    TEXTURE_DIRS wave vectors, each channel with its own phases, so the luminance varies everywhere."""
    X = np.asarray(X, np.float64)
    out = []
    for c in range(3):
        v = np.full(X.shape[:-1], 0.5)
        for k in range(3):
            ph = 2.0 * np.pi * (X @ TEXTURE_DIRS[k]) / TEXTURE_WAVELENGTHS[k] + 1.3 * c * (k + 1)
            v = v + TEXTURE_AMPLITUDES[k] * np.sin(ph)
        out.append(v)
    return np.stack(out)


def sphere_room_rgb(K, pose, size, center, radius, room_lo, room_hi):
    """Exact colour float64 [3,H,W] at each ray's hit of the sphere-in-a-room scene (volume_oracle.sphere_room_depth):
    the solid texture texture_rgb of the hit point's world position, so the sphere and every wall carry it."""
    h, w = size
    fx, fy, cx, cy = K
    T = np.asarray(pose, np.float64)
    z = volume_oracle.sphere_room_depth(K, pose, size, center, radius, room_lo, room_hi)
    y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    r = np.stack([(x - cx) / fx, (y - cy) / fy, np.ones_like(x)], -1)
    X = T[:3, 3] + (z[..., None] * r) @ T[:3, :3].T
    return texture_rgb(X)
