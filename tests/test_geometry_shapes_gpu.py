"""The TSDF volume and camera-tracking kernels against their float64 oracles at the geometries reconstruct.py
launches (csrc/volume.cu, csrc/track.cu; oracle/volume_oracle.py, color_volume_oracle.py, track_oracle.py,
photometric_oracle.py).  test_volume_gpu.py and test_track*_gpu.py compare them at toy geometries; here the block, scan,
launch-split, chunk and branch edges are compared too.

- Extraction: grids of 8 points, one-point and 255-point last blocks, 1024 and 1025 blocks (the scan's one and two
  totals per thread), a non-cubic 2.5M-point grid (ten totals per scan thread, partial last run and block), an axis
  of ODB_TSDF_MAX_DIM, the closed-form counts of a sign checkerboard, and a grid of ODB_TSDF_MAX_POINTS points with a
  sphere at its far corner.  Faces identical, vertices and colours within 1e-6.
- Integration: 17 and 33 frames in one call (across the 16-frame launch split), 640x480, 641x479, 1296x968, 1xN and Nx1
  images, axis-aligned poses on a binary voxel grid whose points project onto pixel-rounding ties, truncation below one
  voxel and at ten.  W identical, F and colour within 1e-6, one call bit-identical to frame-by-frame calls.
- Raycast with colour: identity and axis-aligned poses (exactly zero direction components), cameras outside the box
  that miss it, rays along a box face, and the step at both ends of its range.  Hit masks identical, depth within 1e-5
  relative, colour within 1e-6 and NaN exactly off the hit mask.
- Tracking, geometric and photometric, affine on and off: 480x640 and 968x1296, 2048 k pixels and 2048 k + 1 (a one-pixel
  last chunk), 3x3 (a textured wall: one Sobel window), 2xN and Nx2 (no Sobel window fits), and identity reference
  and initial poses.  One iteration: the oracle's counts exactly, pose and nodes within 1e-10 (the two-row and
  two-column strips: within their conditioning's bound); 20 iterations within 1e-7; (Y, g_u, g_v) bit for bit, with
  the expected numbers of finite values."""
import numpy as np
import pytest
import torch

from oracle import color_volume_oracle as CO
from oracle import photometric_oracle as PO
from oracle import track_oracle as TO
from oracle import volume_oracle as VO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)
LAMBDA = 1e-2


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(dev)


def _volume(dims, origin, voxel, color=False, trunc=None):
    from omnidata_b200.volume import TSDFVolume
    return TSDFVolume(origin, voxel, dims, trunc=trunc, color=color, device=dev)


def _host(vol):
    c = None if vol.color is None else vol.color.cpu().numpy()
    return vol.tsdf.cpu().numpy(), vol.weight.cpu().numpy(), c


def _binary_grid(dims):
    """(origin, voxel) of a grid about 1 m long centred near 0: voxel a power of two and the origin a multiple of it,
    so every grid point, and its difference from a grid-aligned camera, is exact in float64."""
    voxel = 2.0 ** -int(np.ceil(np.log2(max(dims) - 1)))
    return tuple(-voxel * ((d - 1) // 2) for d in dims), voxel


# ------------------------------------------------------------------------------------------------ extraction
def _sphere_fields(dims, rng, color, holes=0.05):
    """(origin, voxel, F, W, C): a sphere's truncated SDF through the grid, W in {1, 2, 3} with random W = 0 holes, and a
    random colour field."""
    origin, voxel = _binary_grid(dims)
    ext = voxel * (np.asarray(dims) - 1.0)
    center = np.asarray(origin) + ext * np.array([0.3, 0.35, 0.4])
    radius = max(0.3 * ext.max(), 0.75 * voxel)
    F, _ = VO.sphere_sdf_volume(dims, origin, voxel, center, radius, 3 * voxel)
    W = rng.integers(1, 4, F.shape).astype(np.float32)
    W[rng.random(F.shape) < holes] = 0.0
    C = rng.random((3,) + F.shape).astype(np.float32) if color else None
    return origin, voxel, F, W, C


def _load(vol, F, W, C):
    vol.tsdf.copy_(_t(F))
    vol.weight.copy_(_t(W))
    if C is not None:
        vol.color.copy_(_t(C))


def _compare_mesh(got, want, what, first_vertex=0):
    v, f, c = (None if x is None else x.cpu().numpy() for x in got)
    ov, of, oc = want
    assert v.shape == ov.shape and f.shape == of.shape, (what, v.shape, ov.shape, f.shape, of.shape)
    verr = float(np.max(np.abs(v - ov) / np.maximum(np.abs(ov), 1.0), initial=0.0))
    cerr = 0.0 if oc is None else float(np.max(np.abs(c - oc), initial=0.0))
    print(f"{what}: {len(v)} vertices, {len(f)} faces; vertex diff {verr:.2e} (relative), colour diff {cerr:.2e}")
    assert np.array_equal(f, of + first_vertex)
    assert verr <= 1e-6 and cerr <= 1e-6


EXTRACT_GRIDS = [
    (2, 2, 2),           # the smallest grid: one cell, one block of 8 points
    (19, 9, 3),          # 513 points: a last block of 1 point
    (31, 11, 3),         # 1023 points: a last block of 255 points
    (64, 64, 64),        # 1024 x 256 points: 1024 full blocks, one block total per scan thread
    (109, 37, 65),       # 1024 x 256 + 1 points: 1025 blocks, two totals per scan thread, a one-point last block
    (173, 91, 157),      # 2 471 651 points, non-cubic: 9655 blocks, ten per scan thread, partial last run and block
    (2048, 5, 3),        # an axis at ODB_TSDF_MAX_DIM
]


@pytest.mark.parametrize("dims", EXTRACT_GRIDS, ids=lambda d: "x".join(map(str, d)))
def test_extraction_matches_the_oracle(dims):
    rng = np.random.default_rng(sum(dims))
    origin, voxel, F, W, C = _sphere_fields(dims, rng, color=True)
    vol = _volume(dims, origin, voxel, color=True)
    _load(vol, F, W, C)
    got = vol.extract_mesh()
    want = VO.extract_mesh(F, W, C, origin, voxel)
    assert len(want[1]) > 0
    _compare_mesh(got, want, f"extraction {'x'.join(map(str, dims))} ({F.size} points)")


def _checkerboard_counts(dims):
    """Vertices and faces of F = +-1 by the parity of i + j + k, W = 1: a vertex on the edges from each point to its
    odd-parity corners (+x, +y, +z, +xyz) inside the grid, and every tetrahedron has two corners of each sign, so two
    triangles per tetrahedron, 12 per cell."""
    nx, ny, nz = dims
    verts = (nx - 1) * ny * nz + nx * (ny - 1) * nz + nx * ny * (nz - 1) + (nx - 1) * (ny - 1) * (nz - 1)
    return verts, 12 * (nx - 1) * (ny - 1) * (nz - 1)


@pytest.mark.parametrize("dims", [(7, 5, 6), (109, 37, 65), (2048, 5, 3)], ids=lambda d: "x".join(map(str, d)))
def test_checkerboard_closed_form(dims):
    origin, voxel = _binary_grid(dims)
    k, j, i = np.meshgrid(*(np.arange(d) for d in dims[::-1]), indexing="ij")
    F = np.where((i + j + k) % 2 == 0, 1.0, -1.0).astype(np.float32)
    W = np.ones_like(F)
    vol = _volume(dims, origin, voxel)
    _load(vol, F, W, None)
    got = vol.extract_mesh()
    nv, nf = _checkerboard_counts(dims)
    assert got[0].shape == (nv, 3) and got[1].shape == (nf, 3)
    _compare_mesh(got, VO.extract_mesh(F, W, None, origin, voxel), f"checkerboard {'x'.join(map(str, dims))}")


def test_extraction_at_the_point_limit():
    """2^28 points (2048 x 2048 x 64) with W = 0 except a 24^3 box at the far corner holding a sphere cut by the grid's
    faces: the highest point indices, 2^20 blocks and 1024 block totals per scan thread.  The oracle runs on the box
    with index_offset; every vertex lies in the box, so the GPU's first vertex there is vertex 0."""
    from omnidata_b200 import ops
    from omnidata_b200.volume import MAX_DIM, MAX_POINTS
    dims = (MAX_DIM, MAX_DIM, MAX_POINTS // (MAX_DIM * MAX_DIM))
    assert dims[0] * dims[1] * dims[2] == MAX_POINTS
    need = 8 * MAX_POINTS + ops.tsdf_mesh_workspace_bytes(dims) + (256 << 20)
    torch.cuda.empty_cache()                            # what earlier tests left in torch's cache is free to reuse
    free, _ = torch.cuda.mem_get_info(dev)
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free (the device is "
                    f"shared)")
    box = 24
    off = tuple(d - box for d in dims)
    origin, voxel = (-1.0, -2.0, 0.5), 2.0 ** -10
    sub_origin = tuple(o + voxel * q for o, q in zip(origin, off))
    center = np.asarray(sub_origin) + voxel * np.array([19.5, 19.0, 20.0])
    F, W = VO.sphere_sdf_volume((box,) * 3, sub_origin, voxel, center, 8.4 * voxel, 3 * voxel)
    W[np.random.default_rng(28).random(W.shape) < 0.05] = 0.0
    W[-1, -1, -1] = 1.0
    vol = _volume(dims, origin, voxel)
    try:
        vol.tsdf[off[2]:, off[1]:, off[0]:] = _t(F)
        vol.weight[off[2]:, off[1]:, off[0]:] = _t(W)
        got = vol.extract_mesh()
        want = VO.extract_mesh(F, W, None, origin, voxel, index_offset=off)
        assert len(want[1]) > 200 and F[-1, -1, -1] < 0           # the last point lies inside the sphere
        _compare_mesh(got, want, f"extraction at {MAX_POINTS} points, {box}^3 box at {off}")
    finally:
        del vol
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ integration
def _axis_rotations():
    """The 24 proper rotations with entries in {0, 1, -1}."""
    out = []
    for perm in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):
        for signs in np.ndindex(2, 2, 2):
            R = np.zeros((3, 3))
            for r, c in enumerate(perm):
                R[r, c] = 1.0 - 2.0 * signs[r]
            if np.linalg.det(R) > 0:
                out.append(R)
    return out


def _axis_poses(rng, n, dims, voxel, origin, dist, rotations=None):
    """n camera-to-world poses with axis-aligned rotations, each camera `dist` voxels from a random grid point along its
    optical axis: every coordinate is a whole number of voxels."""
    rots = _axis_rotations() if rotations is None else rotations
    out = []
    for q in range(n):
        R = rots[q % len(rots)]
        p = np.array([rng.integers(d // 4, d - d // 4) if d > 3 else d // 2 for d in dims], np.float64)
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = np.asarray(origin) + voxel * (p - dist * R[:, 2])
        out.append(T)
    return np.stack(out)


def _generic_poses(rng, n, target, dist):
    out = []
    for _ in range(n):
        d = rng.standard_normal(3)
        T = VO.look_at(np.asarray(target) + dist * d / np.linalg.norm(d), np.asarray(target) + 0.05 * rng.standard_normal(3))
        a = rng.uniform(-np.pi, np.pi)
        T[:3, :3] = T[:3, :3] @ np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        out.append(T)
    return np.stack(out)


def _frames(rng, b, h, w, lo, hi, color):
    depth = rng.uniform(lo, hi, (b, h, w)).astype(np.float32)
    bad = rng.random((b, h, w))
    depth[bad < 0.04] = np.nan
    depth[(bad >= 0.04) & (bad < 0.06)] = 0.0
    depth[(bad >= 0.06) & (bad < 0.07)] = -1.0
    return depth, rng.random((b, 3, h, w)).astype(np.float32) if color else None


def _ties(dims, origin, voxel, K, poses, h, w):
    """Grid points that project inside the image onto a pixel-rounding tie (u + 0.5 or v + 0.5 a whole number), with
    the projection's operations."""
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    X = [origin[0] + voxel * i.astype(np.float64), origin[1] + voxel * j.astype(np.float64),
         origin[2] + voxel * k.astype(np.float64)]
    fx, fy, cx, cy = K
    n = 0
    for T in poses:
        dx, dy, dz = (X[a] - T[a, 3] for a in range(3))
        zc = (T[0, 2] * dx + T[1, 2] * dy) + T[2, 2] * dz
        xc = (T[0, 0] * dx + T[1, 0] * dy) + T[2, 0] * dz
        yc = (T[0, 1] * dx + T[1, 1] * dy) + T[2, 1] * dz
        with np.errstate(divide="ignore", invalid="ignore"):
            u, v = (fx * xc) / zc + cx + 0.5, (fy * yc) / zc + cy + 0.5
            inside = (zc > 0) & (np.floor(u) >= 0) & (np.floor(u) <= w - 1) & (np.floor(v) >= 0) & (np.floor(v) <= h - 1)
        n += int((inside & ((u == np.floor(u)) | (v == np.floor(v)))).sum())
    return n


# (grid, (h, w), frames, truncation in voxels, poses, colour)
INTEGRATE_CASES = {
    "19x9x3-480x640-17f": ((19, 9, 3), (480, 640), 17, 3.0, "generic", True),
    "31x11x3-479x641-33f-trunc0.5": ((31, 11, 3), (479, 641), 33, 0.5, "generic", False),
    "109x37x65-480x640-17f-ties-trunc10": ((109, 37, 65), (480, 640), 17, 10.0, "axis", True),
    "109x37x65-479x641-33f-ties-trunc0.5": ((109, 37, 65), (479, 641), 33, 0.5, "axis", False),
    "64x64x64-968x1296-17f": ((64, 64, 64), (968, 1296), 17, 3.0, "generic", False),
    "2048x5x3-1x1023-17f-ties": ((2048, 5, 3), (1, 1023), 17, 3.0, "row", True),
    "2048x5x3-1023x1-17f-ties-trunc10": ((2048, 5, 3), (1023, 1), 17, 10.0, "column", False),
}


@pytest.mark.parametrize("case", list(INTEGRATE_CASES))
def test_integration_matches_the_oracle(case):
    dims, (h, w), b, trunc_vox, kind, color = INTEGRATE_CASES[case]
    rng = np.random.default_rng(len(case) * 31 + b)
    origin, voxel = _binary_grid(dims)
    centre = np.asarray(origin) + voxel * ((np.asarray(dims) - 1) // 2)
    extent = voxel * max(dims)
    if kind == "generic":
        dist = 1.5 * extent
        f = 0.9 * max(h, w)
        K = (f * 1.02, f, (w - 1) / 2, (h - 1) / 2)
        T = _generic_poses(rng, b, centre, dist)
    else:
        # the camera 64 voxels from a grid point, f = 96 px: that point's plane projects at 1.5 px per voxel, onto ties
        # (u + 0.5 whole: odd i' with integer cx, even i' with half-integer cx), and so do other planes
        dist, f = 64, 96.0
        K = (f, f, (w - 1) / 2, (h - 1) / 2)
        # 1xN: the camera's y axis across the thin axes (the row through the camera sees a plane of points); Nx1 its x
        rows = {"row": [np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]]), np.array([[-1.0, 0, 0], [0, 0, -1], [0, -1, 0]])],
                "column": [np.array([[0.0, 1, 0], [0, 0, 1], [1, 0, 0]]), np.array([[0.0, 1, 0], [0, 0, -1], [-1, 0, 0]])]}
        T = _axis_poses(rng, b, dims, voxel, origin, dist, rows.get(kind))
        dist *= voxel
    depth, rgb = _frames(rng, b, h, w, max(dist - extent, 0.05), dist + extent, color)
    trunc = trunc_vox * voxel
    vol = _volume(dims, origin, voxel, color, trunc)
    vol.integrate(_t(depth), K, T, None if rgb is None else _t(rgb))
    z = np.zeros(dims[::-1], np.float32)
    F, W, C = VO.integrate(z, z, np.zeros((3,) + z.shape, np.float32) if color else None, origin, voxel, trunc, depth,
                           K, T, rgb)
    gF, gW, gC = _host(vol)
    ferr = float(np.abs(gF - F).max())
    cerr = 0.0 if C is None else float(np.abs(gC - C).max())
    ties = _ties(dims, origin, voxel, K, T, h, w) if kind != "generic" else 0
    print(f"integration {case}: {int((W > 0).sum())} of {W.size} points observed, W max {int(W.max())}, "
          f"{ties} pixel-rounding ties; F diff {ferr:.2e}, colour diff {cerr:.2e}")
    assert (W > 0).sum() > 0.01 * W.size and W.max() >= 2
    assert kind == "generic" or ties > 0
    assert np.array_equal(gW, W) and ferr <= 1e-6 and cerr <= 1e-6
    one = vol._data.clone()
    vol.reset()
    for q in range(b):                                  # frame by frame: the same bits as one call
        vol.integrate(_t(depth[q:q + 1]), K, T[q:q + 1], None if rgb is None else _t(rgb[q:q + 1]))
    assert torch.equal(vol._data.view(torch.int32), one.view(torch.int32))


# ------------------------------------------------------------------------------------------------ raycast
@pytest.fixture(scope="module")
def room_volume():
    """The sphere-in-a-room scene fused with colour from 20 orbit poses, on a binary 53 x 51 x 49 grid (1/16 m)."""
    voxel = 0.0625
    origin, dims = (-1.625, -1.5625, -1.5), (53, 51, 49)
    vol = _volume(dims, origin, voxel, color=True)
    size, k = (120, 160), (150.0, 150.0, 79.5, 59.5)
    T = VO.orbit_poses(20, 1.2, CENTER)
    depth = np.stack([VO.sphere_room_depth(k, t, size, CENTER, RADIUS, ROOM_LO, ROOM_HI) for t in T])
    rgb = np.stack([CO.sphere_room_rgb(k, t, size, CENTER, RADIUS, ROOM_LO, ROOM_HI) for t in T])
    vol.integrate(_t(depth.astype(np.float32)), k, T, _t(rgb.astype(np.float32)))
    return vol


def _pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


ROT = {"identity": np.eye(3),
       "-x": np.array([[0.0, 0, -1], [0, 1, 0], [1, 0, 0]]),         # optical axis along -x
       "+y": np.array([[1.0, 0, 0], [0, 0, 1], [0, -1, 0]]),         # optical axis along +y
       "+x": np.array([[0.0, 0, 1], [0, 1, 0], [-1, 0, 0]])}

# (pose, (h, w), intrinsics, step in voxels or None, expected: "hit" | "miss")
RAYCAST_CASES = {
    "identity-480x640": (_pose(ROT["identity"], (0.03, -0.02, -1.2)), (480, 640), (500.0, 500.0, 320.0, 240.0), None,
                         "hit"),
    "identity-479x641": (_pose(ROT["identity"], (0.03, -0.02, -1.2)), (479, 641), (520.0, 510.0, 320.0, 239.0), None,
                         "hit"),
    "axis-x-479x641": (_pose(ROT["-x"], (1.25, 0.0625, 0.0)), (479, 641), (400.0, 400.0, 320.0, 239.0), None, "hit"),
    "axis+y-479x641-step1": (_pose(ROT["+y"], (0.0, -1.25, 0.125)), (479, 641), (400.0, 400.0, 320.0, 239.0), 1.0,
                             "hit"),
    # outside the box (x > 1.625): looking away, and looking along +y past it (the widest ray reaches x = 1.625 at
    # y = 3.1, beyond the box)
    "outside-away": (_pose(ROT["+x"], (2.0, 0.1, 0.2)), (479, 641), (500.0, 500.0, 320.0, 239.0), None, "miss"),
    "outside-past": (_pose(ROT["+y"], (3.6, 0.0, 0.0)), (479, 641), (500.0, 500.0, 320.0, 239.0), None, "miss"),
    # the camera on the face x = lo: the centre column's rays (d_x = 0) run inside the face, half the others leave
    "face-x-on": (_pose(ROT["identity"], (-1.625, 0.0, -1.4)), (241, 321), (200.0, 200.0, 160.0, 120.0), None, "hit"),
    # just outside it: the centre column misses by the d = 0 rule, the rest enter through the face at a grazing angle
    "face-x-outside": (_pose(ROT["identity"], (-1.625 - 2.0 ** -20, 0.0, -1.4)), (241, 321),
                       (200.0, 200.0, 160.0, 120.0), None, "hit"),
    "face-z-grazing": (_pose(ROT["+y"], (0.5, -1.5, 1.5)), (241, 321), (200.0, 200.0, 160.0, 120.0), None, "hit"),
}


def _compare_raycast(vol, pose, size, K, step, expect, what):
    F, W, C = _host(vol)
    got_d = vol.raycast(K, pose, size, step)
    d, c = vol.raycast(K, pose, size, step, color=True)
    assert torch.equal(d, got_d)
    want_d, want_c = CO.raycast_color(F, W, C, vol.origin, vol.voxel, K, pose, size, step)
    d, c = d.cpu().numpy(), c.cpu().numpy()
    hit = want_d > 0
    derr = float(np.max(np.abs(d[hit] - want_d[hit]) / want_d[hit], initial=0.0))
    cerr = float(np.max(np.abs(c[:, hit] - want_c[:, hit]), initial=0.0))
    print(f"raycast {what}: {size[0]}x{size[1]}, {int(hit.sum())} hits; depth diff {derr:.2e} (relative), colour diff "
          f"{cerr:.2e}")
    assert np.array_equal(d > 0, hit)
    assert np.array_equal(np.isnan(c), np.broadcast_to(~hit, c.shape)) and np.array_equal(np.isnan(c), np.isnan(want_c))
    assert derr <= 1e-5 and cerr <= 1e-6
    assert hit.any() if expect == "hit" else not hit.any()
    return hit


def _zero_direction_rays(pose, size, K):
    """Rays with an exactly zero world direction component, with the kernel's operations."""
    h, w = size
    fx, fy, cx, cy = K
    y, x = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    rx, ry = (x - cx) / fx, (y - cy) / fy
    nrm = np.sqrt((rx * rx + ry * ry) + 1.0)
    ux, uy, uz = rx / nrm, ry / nrm, 1.0 / nrm
    return np.any([((pose[a, 0] * ux + pose[a, 1] * uy) + pose[a, 2] * uz) == 0.0 for a in range(3)], axis=0)


@pytest.mark.parametrize("case", list(RAYCAST_CASES))
def test_raycast_matches_the_oracle(room_volume, case):
    pose, size, K, step, expect = RAYCAST_CASES[case]
    step = None if step is None else step * room_volume.voxel
    zero = _zero_direction_rays(pose, size, K)
    if case.startswith(("identity", "axis", "face")):
        assert zero.sum() >= min(size)
    _compare_raycast(room_volume, pose, size, K, step, expect, f"{case} ({int(zero.sum())} rays with a zero component)")


def test_raycast_finest_step():
    """step = voxel / 64 on a small grid and image (the oracle marches every ray 64 samples a voxel)."""
    dims = (24, 20, 22)
    rng = np.random.default_rng(64)
    origin, voxel, F, W, C = _sphere_fields(dims, rng, color=True, holes=0.02)
    vol = _volume(dims, origin, voxel, color=True)
    _load(vol, F, W, C)
    centre = np.asarray(origin) + voxel * (np.asarray(dims) - 1) / 2
    for q, pose in enumerate((VO.look_at(centre + np.array([0.2, -0.9, 0.3]), centre),
                              _pose(np.eye(3), centre - np.array([0.0, 0.0, 1.0])))):
        _compare_raycast(vol, pose, (23, 31), (30.0, 30.0, 15.0, 11.0), voxel / 64, "hit", f"step voxel/64, pose {q}")


# ------------------------------------------------------------------------------------------------ tracking
# (h, w), scene: "room" the sphere-in-a-room scene from a camera on test_track_gpu's path, "identity" the reference and
# initial poses the identity, "wall" a fronto-parallel textured wall seen through a narrow field of view
TRACK_CASES = [
    ((480, 640), "room"), ((968, 1296), "room"),
    ((64, 96), "room"),          # 2048 x 3 pixels: three full chunks
    ((113, 145), "room"),        # 2048 x 8 + 1 pixels: a one-pixel last chunk
    # one Sobel window.  The tracker's normals need neighbouring depths within 2 % of the image's depth range, so at
    # 3 x 3 only a plane at one depth gives all nine.  A single plane leaves three unknowns free: the solve ends
    # degenerate in the kernel and the oracle alike, after the association's counts are compared.  One gradient
    # is no 2 x 2 block to interpolate, so there are no photometric terms
    ((3, 3), "wall"),
    # no Sobel window fits.  Both strips solve their first iteration (poorly conditioned, see _condition) and then
    # lose their overlap: the 20-iteration runs compare the no_overlap refusal
    ((2, 1537), "room"), ((1537, 2), "room"),
    ((479, 641), "identity"),
]


def _tracking_scene(hw, affine, rng, scene):
    """(pred, ref depth, frame rgb, reference rgb, K, ref pose, init nodes) in the sphere-in-a-room scene, as
    test_track_rgbd_gpu.test_matches_the_oracle builds them, at the reference pose of the scene (TRACK_CASES)."""
    h, w = hw
    f = 30.0 if scene == "wall" else 0.9 * max(h, w)
    k = (f, f, (w - 1) / 2 + 0.3, (h - 1) / 2 - 0.2)
    center, radius, lo, hi = CENTER, RADIUS, ROOM_LO, ROOM_HI
    if scene == "identity":
        center, hi = (0.05, -0.03, 1.2), (1.5, 1.5, 2.5)
        radius, ref = 0.4, np.eye(4)
    elif scene == "wall":                               # looking along +x at the wall x = 1.5, 0.6 m away
        ref = _pose(ROT["+x"], (0.9, 0.7, 0.4))
    else:
        ref = TO.camera_path(1, CENTER, seed=h + w)[0]
    truth = TO.perturb(ref, 0.02, np.radians(1.5), rng)
    depth = lambda T: VO.sphere_room_depth(k, T, hw, center, radius, lo, hi)
    colour = lambda T: CO.sphere_room_rgb(k, T, hw, center, radius, lo, hi).astype(np.float32)
    d_ref = depth(ref).astype(np.float32)
    c_ref = colour(ref)
    if scene != "wall":                                 # holes (they would empty the one window)
        d_ref[rng.random(hw) < 0.03] = 0.0
        c_ref[:, rng.random(hw) < 0.03] = np.nan
    s1, t1 = (rng.uniform(0.6, 1.8), rng.uniform(-0.2, 0.2)) if affine else (1.0, 0.0)
    pred = (s1 * depth(truth) + t1).astype(np.float32)
    bad = rng.random(hw)
    pred[bad < 0.02] = np.nan
    pred[(bad >= 0.02) & (bad < 0.03)] = 0.0
    pred[(bad >= 0.03) & (bad < 0.04)] = -1.0
    init = (1 / s1 * 1.01, -t1 / s1 + 0.01) if affine else None
    return pred, d_ref, colour(truth), c_ref, k, ref, init


def _condition(pred, d_ref, normals, k, ref, init, affine):
    """The condition number of the first iteration's unit-diagonal geometric normal matrix (the oracle's association).
    The solve's error is about it times the rounding of the sums, which the kernel adds in chunk order and the oracle
    in another: a two-row strip sees little of the pitch (about 5e5), and its first step agrees with the oracle's to
    a few 1e-10, not 1e-10."""
    s, t = init if affine else (1.0, 0.0)
    Rm, tm = TO.relative_pose(ref, ref)
    A = TO.associate(pred, d_ref, normals, k, Rm, tm, s, t, 0.1, 0.02)
    J, wt = A["J"].reshape(-1, 8), A["w"].reshape(-1)
    n = 8 if affine else 6
    H = ((J * wt[:, None]).T @ J)[:n, :n]
    d = np.sqrt(np.diag(H))
    return float(np.linalg.cond(H / np.outer(d, d))) if np.all(d > 0) else 1.0


@pytest.mark.parametrize("photometric", [False, True], ids=["geometric", "photometric"])
@pytest.mark.parametrize("affine", [True, False], ids=["affine", "metric"])
@pytest.mark.parametrize("hw,scene", TRACK_CASES,
                         ids=[f"{h}x{w}" + ("" if c == "room" else f"-{c}") for (h, w), c in TRACK_CASES])
def test_tracking_matches_the_oracle(hw, scene, affine, photometric):
    from omnidata_b200.track import FrameTracker
    h, w = hw
    strip = min(h, w) < 3
    rng = np.random.default_rng(h * 7 + w + affine)
    pred, d_ref, rgb, c_ref, k, ref, init = _tracking_scene(hw, affine, rng, scene)
    nodes0 = torch.tensor(init, dtype=torch.float64, device=dev).reshape(1, 1, 1, 2) if affine else None
    cond = None
    for iters in (1, 20):
        lam = LAMBDA if photometric else 0.0
        tr = FrameTracker(affine=affine, iterations=iters, photometric=lam)
        kw = dict(rgb=_t(rgb), ref_rgb=_t(c_ref)) if photometric else {}
        pose, nodes, rec = tr.track(_t(pred), _t(d_ref), k, ref, init_nodes=nodes0, **kw)
        normals = tr._bufs["normals"][0].cpu().numpy()
        cond = _condition(pred, d_ref, normals, k, ref, init, affine) if cond is None else cond
        if photometric:
            ig = tr._bufs["intensity"].cpu().numpy()
            want_ig = PO.intensity_gradient(d_ref, c_ref, normals)
            assert np.array_equal(ig, want_ig, equal_nan=True)
            n_y, n_g = int(np.isfinite(want_ig[0]).sum()), int(np.isfinite(want_ig[1]).sum())
            assert n_y > 0.9 * h * w                                    # not an empty comparison
            if strip:
                assert n_g == 0
            elif (h, w) == (3, 3):
                assert n_g == 1
            else:
                assert n_g > 0
            T, (s, t), orec = PO.track(pred, d_ref, k, ref, rgb, c_ref, None, init, affine=affine, iterations=iters,
                                       photometric=LAMBDA, normals=normals)
        else:
            T, (s, t), orec = TO.track(pred, d_ref, k, ref, None, init, affine=affine, iterations=iters,
                                       normals=normals)
        rec, pose = rec.cpu().numpy(), pose.cpu().numpy()
        # one iteration: 1e-10, and for the poorly conditioned strips the conditioning's bound (_condition)
        tol = (max(1e-10, 3e-15 * cond) if strip else 1e-10) if iters == 1 else 1e-7
        perr = float(np.abs(pose - T).max())
        nerr = float(np.abs(nodes.reshape(2).cpu().numpy() - np.array([s, t])).max())
        extra = (f", {int(rec[8])} photometric terms (oracle {int(orec[8])}), {n_y} luminances and {n_g} "
                 f"gradients") if photometric else ""
        print(f"tracking {h}x{w} ({-(-h * w // 2048)} chunks, {scene}) affine={affine} iterations={iters}: status "
              f"{int(rec[1])} (oracle {int(orec[1])}), {int(rec[0])} correspondences of {int(rec[7])} (oracle "
              f"{int(orec[0])}){extra}, {int(rec[4])} run; pose diff {perr:.2e}, nodes diff {nerr:.2e} (tolerance "
              f"{tol:.1e}, condition {cond:.1e})")
        assert rec.shape == orec.shape and rec[1] == orec[1] and rec[4] == orec[4]
        if iters == 1:
            assert rec[0] == orec[0] and rec[7] == orec[7]
            if photometric:
                assert rec[8] == orec[8]
        assert perr <= tol and nerr <= tol
        assert abs(rec[2] - orec[2]) <= 1e-9 and abs(rec[3] - orec[3]) <= 1e-12
        if photometric:
            assert abs(rec[9] - orec[9]) <= 1e-9 and abs(rec[10] - orec[10]) <= 1e-12
        if min(h, w) > 3:
            assert rec[1] == 0 and rec[0] > 0.5 * rec[7]             # a real solve, not a refusal
            assert not photometric or rec[8] > 0
        elif iters == 1:
            assert rec[0] > 0.5 * rec[7]                              # the association is compared, not empty
            assert not strip or rec[1] == 0                           # and a strip solves its first step
