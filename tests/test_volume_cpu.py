"""TSDF volumes on the CPU: the float64 oracle's Kuhn split and marching tetrahedra on an analytic sphere (watertight,
Euler characteristic 2, outward-wound, within a voxel of the sphere), the host-side refusals of TSDFVolume, ops and
reconstruct.py, and the ptxas check of csrc/volume.cu (no spills or stack frames)."""
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import volume_oracle as VO

CENTER, RADIUS = (0.013, -0.021, 0.007), 0.61
DIMS, ORIGIN, VOXEL = (24, 24, 24), (-0.92, -0.92, -0.92), 0.08


def _sphere_mesh():
    F, W = VO.sphere_sdf_volume(DIMS, ORIGIN, VOXEL, CENTER, RADIUS, 3 * VOXEL)
    return VO.extract_mesh(F, W, None, ORIGIN, VOXEL)


def test_kuhn_split_covers_the_cell():
    vol = VO.kuhn_volumes()
    assert np.isclose(np.abs(vol).sum(), 1.0, atol=1e-15)
    assert np.all(np.abs(np.abs(vol) - 1 / 6) < 1e-15)
    assert np.array_equal(vol < 0, VO.TET_ODD.astype(bool))


def test_sphere_mesh_is_watertight_with_euler_characteristic_two():
    v, f, c = _sphere_mesh()
    assert c is None and len(f) > 500
    edges, mult = VO.mesh_edges(f)
    assert np.all(mult == 2)
    assert len(v) - len(edges) + len(f) == 2
    assert np.unique(f).size == len(v)               # every vertex is used


def test_sphere_mesh_is_outward_wound_and_within_a_voxel():
    v, f, _ = _sphere_mesh()
    assert VO.signed_volume(v, f) > 0
    n = VO.face_normals(v, f)
    area = np.linalg.norm(n, axis=1)
    centroid = v.astype(np.float64)[f].mean(1) - np.asarray(CENTER)
    big = area > 1e-12
    assert np.all(np.einsum("ij,ij->i", n[big], centroid[big]) > 0)
    dist = np.abs(np.linalg.norm(v.astype(np.float64) - np.asarray(CENTER), axis=1) - RADIUS)
    assert dist.max() < VOXEL
    vol = 4 / 3 * np.pi * RADIUS ** 3
    assert abs(VO.signed_volume(v, f) - vol) / vol < 0.05


def test_integrate_oracle_on_a_plane():
    """A fronto-parallel wall at z = 1 seen from the origin: F is the truncated projective distance."""
    dims, origin, voxel, trunc = (8, 8, 8), (-0.35, -0.35, 0.6), 0.1, 0.25
    K = (40.0, 40.0, 15.5, 11.5)
    depth = np.ones((1, 24, 32), np.float32)
    F, W, _ = VO.integrate(np.zeros(dims[::-1], np.float32), np.zeros(dims[::-1], np.float32), None, origin, voxel,
                           trunc, depth, K, np.eye(4)[None])
    z = origin[2] + voxel * np.arange(8)
    seen = W[:, 4, 4] > 0
    assert np.array_equal(seen, z <= 1.0 + trunc + 1e-12)
    assert np.allclose(F[seen, 4, 4], np.minimum(1.0, (1.0 - z[seen]) / trunc), atol=1e-7)


def test_volume_refusals():
    from omnidata_b200.volume import TSDFVolume
    for dims in ((1, 4, 4), (4, 4, 2049), (2048, 2048, 65), (4, 4)):
        with pytest.raises(ValueError):
            TSDFVolume((0, 0, 0), 0.1, dims, device="cuda:0")
    for voxel in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            TSDFVolume((0, 0, 0), voxel, (4, 4, 4), device="cuda:0")
    for trunc in (0.0, -0.1, float("nan")):
        with pytest.raises(ValueError):
            TSDFVolume((0, 0, 0), 0.1, (4, 4, 4), trunc=trunc, device="cuda:0")
    with pytest.raises(ValueError):
        TSDFVolume((0, float("nan"), 0), 0.1, (4, 4, 4), device="cuda:0")
    with pytest.raises(ValueError):
        TSDFVolume((0, 0, 0), 0.1, (4, 4, 4), device="cpu")


def test_pose_and_intrinsics_checks():
    from omnidata_b200 import _capi, ops
    T = VO.look_at((1.0, 2.0, 0.5), (0.0, 0.0, 0.0))
    assert ops.check_poses("t", T).shape == (1, 16)
    assert ops.check_poses("t", torch.from_numpy(np.stack([T, T]))).shape == (2, 16)
    bad = []
    s = T.copy(); s[:3, :3] *= 1.001; bad.append(s)                    # scaled: not rigid
    s = T.copy(); s[0, 3] = np.nan; bad.append(s)
    s = T.copy(); s[3, 2] = 0.1; bad.append(s)
    s = T.copy(); s[:3, 0] = s[:3, 1]; bad.append(s)                    # sheared
    for s in bad:
        with pytest.raises(_capi.OdbError):
            ops.check_poses("t", s)
    for shape in ((3, 4), (2, 4, 3), (0, 4, 4)):
        with pytest.raises(_capi.OdbError):
            ops.check_poses("t", np.zeros(shape))
    for K in ((0, 1, 0, 0), (1, -1, 0, 0), (1, 1, float("nan"), 0), (1, 1, 1)):
        with pytest.raises(_capi.OdbError):
            ops.check_intrinsics("t", K)
    with pytest.raises(_capi.OdbError):
        ops.check_volume_grid("t", (4, 4, 4), (0, 0, 0), 0.0)


def test_reconstruct_argument_errors():
    import reconstruct
    base = ["--img_path", "i", "--pose_path", "p", "--intrinsics", "500,500,319.5,239.5", "--voxel", "0.02",
            "--bounds=-1,-1,-1,1,1,1", "--out", "m.ply", "--synthetic_weights", "--sparse_path", "s"]
    a = reconstruct.parse_args(base)
    assert a.dims == (101, 101, 101) and a.origin == (-1.0, -1.0, -1.0)
    bad = [
        [x for x in base if x != "--synthetic_weights"],                       # no weights
        base + ["--checkpoint", "c.pt"],                                       # both
        [x if x != "500,500,319.5,239.5" else "500,0,1,1" for x in base],      # intrinsics
        [x if x != "0.02" else "0" for x in base],                             # voxel
        [x if x != "--bounds=-1,-1,-1,1,1,1" else "--bounds=1,-1,-1,-1,1,1" for x in base],      # empty bounds
        [x if x != "--bounds=-1,-1,-1,1,1,1" else "--bounds=-1,-1,-1,1,1" for x in base],        # five numbers
        [x if x != "0.02" else "0.0001" for x in base],                        # too many points
        base[:-2],                                                             # no sparse depths for frame 0
        base + ["--depth_scale", "0"],
        base + ["--trunc", "-1"],
    ]
    for argv in bad:
        with pytest.raises(SystemExit):
            reconstruct.parse_args(argv)


def test_volume_kernels_do_not_spill(tmp_path):
    """csrc/volume.cu compiled as the build compiles it (without fast-math): no stack frame, no spills."""
    from omnidata_b200 import build
    assert "volume.cu" in build.SOURCES and "volume.cu" not in build.FAST_MATH_SOURCES
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "volume.cu"), "-o",
           str(tmp_path / "volume.o")]
    try:
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600).stdout
    except FileNotFoundError:
        pytest.skip("nvcc not available")
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert len(frames) >= 6, out
    assert all(f == ("0", "0", "0") for f in frames), out


def test_oracle_index_offset():
    """A sub-box of a larger grid with index_offset: offset 0 is the plain call bit for bit; a box holding every W > 0
    point of the grid gives the grid's vertices and colours bit for bit and its faces less the box's first vertex;
    integrating the box gives the grid's integration of it bit for bit."""
    rng = np.random.default_rng(5)
    dims, origin, voxel = (13, 11, 12), (-0.45, -0.41, -0.43), 0.07
    F, W = VO.sphere_sdf_volume(dims, origin, voxel, (0.02, -0.03, 0.01), 0.25, 2 * voxel)
    C = rng.random((3,) + F.shape).astype(np.float32)
    W[rng.random(F.shape) < 0.05] = 0.0
    plain = VO.extract_mesh(F, W, C, origin, voxel)
    zero = VO.extract_mesh(F, W, C, origin, voxel, index_offset=(0, 0, 0))
    assert len(plain[1]) > 100
    for a, b in zip(plain, zero):
        assert a.dtype == b.dtype and np.array_equal(a, b)
    big = (dims[0] + 5, dims[1] + 3, dims[2] + 4)
    off = (5, 2, 3)
    box = (slice(off[2], off[2] + dims[2]), slice(off[1], off[1] + dims[1]), slice(off[0], off[0] + dims[0]))
    Fb, Wb, Cb = np.ones(big[::-1], np.float32), np.zeros(big[::-1], np.float32), np.zeros((3,) + big[::-1], np.float32)
    Fb[box], Wb[box], Cb[(slice(None),) + box] = F, W, C
    borigin = tuple(o - voxel * q for o, q in zip(origin, off))
    whole = VO.extract_mesh(Fb, Wb, Cb, borigin, voxel)
    sub = VO.extract_mesh(F, W, C, borigin, voxel, index_offset=off)
    assert np.array_equal(whole[0], sub[0]) and np.array_equal(whole[2], sub[2])
    assert np.array_equal(whole[1], sub[1])                       # no W > 0 point before the box: first vertex 0
    assert np.array_equal(VO._points(dims, borigin, voxel, off)[0], VO._points(big, borigin, voxel)[0][box])
    K = (40.0, 42.0, 15.5, 11.0)
    T = np.stack([VO.look_at((0.1, -1.2, 0.3), (0.0, 0.0, 0.0)), VO.look_at((1.0, 0.4, -0.6), (0.05, 0.0, 0.0))])
    depth = rng.uniform(0.8, 1.6, (2, 24, 32)).astype(np.float32)
    rgb = rng.random((2, 3, 24, 32)).astype(np.float32)
    z = np.zeros(big[::-1], np.float32)
    gF, gW, gC = VO.integrate(z, z, np.zeros((3,) + z.shape, np.float32), borigin, voxel, 0.2, depth, K, T, rgb)
    zb = np.zeros(dims[::-1], np.float32)
    bF, bW, bC = VO.integrate(zb, zb, np.zeros((3,) + zb.shape, np.float32), borigin, voxel, 0.2, depth, K, T, rgb,
                              index_offset=off)
    assert (bW > 0).any() and np.array_equal(bW, gW[box]) and np.array_equal(bF, gF[box])
    assert np.array_equal(bC, gC[(slice(None),) + box])
    pF, pW, pC = VO.integrate(zb, zb, None, origin, voxel, 0.2, depth, K, T)
    qF, qW, qC = VO.integrate(zb, zb, None, origin, voxel, 0.2, depth, K, T, index_offset=(0, 0, 0))
    assert pC is None and qC is None and np.array_equal(pF, qF) and np.array_equal(pW, qW)
