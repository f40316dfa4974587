"""Sparse TSDF volumes on the GPU (SparseTSDFVolume, reconstruct.py without --bounds; csrc/sparse_volume.cu).

- Against the float64 oracle (oracle/sparse_volume_oracle.py) on random generic poses, several image sizes, bad depths,
  colour on and off, over two calls: block set, birth stamps and ids exact, W identical, F and colour within 1e-6.
- Frames in one call, one by one or 3 + 5, and two runs: the same bits for the data, the ids and the mesh.
- Against the dense kernels at a dyadic voxel: blocks born at frame 0 equal a dense TSDFVolume bit for bit; the raycast
  (depth and colour) equals the dense raycast of to_dense(); the mesh equals the dense extraction of to_dense().
- Skipping is exact: on a scene with large empty regions the raycast equals the oracle's full march bit for bit.
- Graph capture of the raycast; the empty volume.
- Beyond the dense limit: the sphere-in-a-room scene at 1/256 m voxels.
- LoopClosure.refuse into a sparse volume; the unposed photometric paths; reconstruct.py without --bounds."""
import json

import numpy as np
import pytest
import torch

from oracle import sparse_volume_oracle as SO
from oracle import track_oracle as TO
from oracle import volume_oracle as VO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _sparse(voxel, color=False, origin=(0.0, 0.0, 0.0), trunc=None):
    from omnidata_b200.volume import SparseTSDFVolume
    return SparseTSDFVolume(voxel, trunc=trunc, color=color, origin=origin, device=dev)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _state(vol):
    return vol.block_keys.clone(), vol.block_birth.clone(), vol._data[:vol.blocks].clone()


def _same_state(a, b):
    return all(torch.equal(_bits(x) if x.dtype == torch.float32 else x, _bits(y) if y.dtype == torch.float32 else y)
               for x, y in zip(a, b))


@pytest.mark.parametrize("color", [False, True])
@pytest.mark.parametrize("hw", [(24, 32), (37, 53), (64, 48)])
def test_integrate_matches_the_oracle(hw, color):
    from test_volume_gpu import _random_frames, _random_intrinsics, _random_poses
    rng = np.random.default_rng(hash(hw) % 1000 + color)
    h, w = hw
    origin = (-0.5, -0.45, -0.55)
    vol = _sparse(0.05, color, origin)
    ov = SO.SparseVolume(0.05, color=color, origin=origin)
    for call in range(2):
        depth, rgb = _random_frames(rng, 3, h, w)
        K = _random_intrinsics(rng, h, w)
        T = _random_poses(rng, 3, (0.0, 0.0, 0.0), 1.2)
        vol.integrate(torch.from_numpy(depth).to(dev), K, T, torch.from_numpy(rgb).to(dev) if color else None)
        ov.integrate(depth, K, T, rgb if color else None)
    assert vol.blocks == len(ov.keys) and len(set(ov.birth.tolist())) >= 4
    assert np.array_equal(vol.block_keys.cpu().numpy(), ov.keys)
    assert np.array_equal(vol.block_birth.cpu().numpy(), ov.birth)
    data = vol._data[:vol.blocks].cpu().numpy()
    assert np.array_equal(data[:, 1], ov.data[:, 1]) and ov.data[:, 1].max() >= 2 and (ov.data[:, 1] == 0).any()
    assert np.abs(data[:, 0] - ov.data[:, 0]).max() <= 1e-6
    if color:
        assert np.abs(data[:, 2:] - ov.data[:, 2:]).max() <= 1e-6


def _mesh_bits(vol):
    v, f, c = vol.extract_mesh()
    return [_bits(v), f] + ([] if c is None else [_bits(c)])


def test_split_invariance_and_determinism():
    from test_volume_gpu import _random_frames, _random_intrinsics, _random_poses
    rng = np.random.default_rng(7)
    depth, rgb = _random_frames(rng, 8, 40, 56)
    K = _random_intrinsics(rng, 40, 56)
    T = _random_poses(rng, 8, (0.0, 0.0, 0.0), 1.2)
    d, c = torch.from_numpy(depth).to(dev), torch.from_numpy(rgb).to(dev)
    runs = []
    for split in ([8], [1] * 8, [3, 5], [8]):
        vol = _sparse(0.05, True, (-0.5, -0.45, -0.55))
        s = 0
        for n in split:
            vol.integrate(d[s:s + n], K, T[s:s + n], c[s:s + n])
            s += n
        runs.append((_state(vol), _mesh_bits(vol)))
    assert len(set(runs[0][0][1].tolist())) >= 4
    for state, mesh in runs[1:]:
        assert _same_state(state, runs[0][0])
        assert all(torch.equal(x, y) for x, y in zip(mesh, runs[0][1]))


def _scene(voxel, n_poses=12, size=(90, 120), f=110.0, color=False, radius=1.2):
    h, w = size
    K = (f, f, (w - 1) / 2, (h - 1) / 2)
    T = VO.orbit_poses(n_poses, radius, CENTER)
    depth = np.stack([VO.sphere_room_depth(K, t, size, CENTER, RADIUS, ROOM_LO, ROOM_HI) for t in T]).astype(np.float32)
    rgb = None
    if color:
        y, x = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
        rgb = np.stack([np.stack([x, y, 0.5 + 0 * x])] * n_poses).astype(np.float32)
    return K, T, depth, rgb


def _dense_copy(vol):
    """A TSDFVolume holding vol.to_dense()."""
    from omnidata_b200.volume import TSDFVolume
    origin, dims, F, W, C = vol.to_dense()
    dense = TSDFVolume(origin, vol.voxel, dims, trunc=vol.trunc, color=C is not None, device=dev)
    dense.tsdf.copy_(F)
    dense.weight.copy_(W)
    if C is not None:
        dense.color.copy_(C)
    return dense


def _canonical_faces(v, f, ref_v):
    """faces of mesh (v, f) in the vertex ids of ref_v (matched by coordinates), each rotated to start at its least id."""
    from scipy.spatial import cKDTree
    dist, idx = cKDTree(ref_v.astype(np.float64)).query(v.astype(np.float64))
    assert dist.max() <= 1e-6 and len(np.unique(idx)) == len(v) == len(ref_v)
    g = idx[f]
    r = np.argmin(g, 1)
    g = np.stack([g[np.arange(len(g)), (r + q) % 3] for q in range(3)], 1)
    return g[np.lexsort(g.T[::-1])]


@pytest.mark.parametrize("color", [False, True])
def test_against_the_dense_kernels(color):
    from omnidata_b200.volume import TSDFVolume
    voxel = 1.0 / 32
    K, T, depth, rgb = _scene(voxel, color=color)
    vol = _sparse(voxel, color)
    d = torch.from_numpy(depth).to(dev)
    c = None if rgb is None else torch.from_numpy(rgb).to(dev)
    vol.integrate(d, K, T, c)
    origin, dims, F, W, C = vol.to_dense()
    dense = TSDFVolume(origin, voxel, dims, trunc=vol.trunc, color=color, device=dev)
    dense.integrate(d, K, T, c)
    born0 = torch.zeros_like(W, dtype=torch.bool)
    bmin = vol.block_coords.min(0).values
    for (bx, by, bz) in (vol.block_coords[vol.block_birth == 0] - bmin).tolist():
        born0[8 * bz:8 * bz + 8, 8 * by:8 * by + 8, 8 * bx:8 * bx + 8] = True
    assert born0.float().mean() > 0.02 and (vol.block_birth > 0).any()
    assert torch.equal(_bits(F[born0]), _bits(dense.tsdf[born0])) and torch.equal(_bits(W[born0]),
                                                                               _bits(dense.weight[born0]))
    if color:
        assert torch.equal(_bits(C[:, born0]), _bits(dense.color[:, born0]))
    copy = _dense_copy(vol)
    for q, (step, size) in enumerate(((None, (45, 60)), (0.7 * voxel, (31, 47)))):
        pose = VO.look_at((0.9, -0.7, 0.4 - 0.5 * q), CENTER)
        got, want = vol.raycast(K, pose, size, step, color=color), copy.raycast(K, pose, size, step, color=color)
        got, want = (got, want) if color else ((got,), (want,))
        assert (want[0] > 0).float().mean() > 0.2
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(got, want))
    v, f, cv = vol.extract_mesh()
    dv, df, dc = copy.extract_mesh()
    assert len(f) > 1000 and len(f) == len(df)
    v, dv = v.cpu().numpy(), dv.cpu().numpy()
    assert np.array_equal(_canonical_faces(v, f.cpu().numpy(), dv), _canonical_faces(dv, df.cpu().numpy(), dv))


def test_skipping_is_exact():
    """Two small patches 2.5 m apart: the bounding box is mostly unallocated.  Rays that start inside allocated space,
    rays that cross the empty middle and rays that miss everything equal the oracle's full march bit for bit."""
    voxel = 0.02
    size = (48, 64)
    K = (120.0, 120.0, 31.5, 23.5)
    vol = _sparse(voxel, True, (0.013, -0.007, 0.002))
    poses = [VO.look_at((0.0, 0.0, 0.0), (0.0, 0.0, 1.0)), VO.look_at((2.5, 1.0, 0.6), (2.5, 1.0, 1.6)),
             VO.look_at((1.2, 0.5, 0.8), (1.2, 0.5, 2.0))]
    depth = np.full((3,) + size, 0.8, np.float32)
    depth[2] = 0.03                                   # < trunc: allocates the camera's own block
    rgb = np.random.default_rng(1).random((3, 3) + size).astype(np.float32)
    vol.integrate(torch.from_numpy(depth).to(dev), K, np.stack(poses), torch.from_numpy(rgb).to(dev))
    lo, dims, F, W, C = vol.to_dense()
    W_host = W.cpu().numpy()
    assert (W_host > 0).mean() < 0.02
    from oracle import color_volume_oracle as CO
    views = [VO.look_at((-0.5, 0.0, -1.0), (3.0, 1.0, 1.0)),    # across both patches and the empty middle
             VO.look_at((0.0, 0.0, 0.7), (0.0, 0.0, 2.0)),      # starting inside an allocated block
             VO.look_at((0.0, 0.0, -1.0), (0.0, 0.0, -2.0)),    # facing away: misses everything
             VO.look_at((2.0, 0.8, -0.5), (2.5, 1.0, 1.4))]     # from outside the box, across empty blocks
    hits = 0
    for step in (0.5 * voxel, 0.7 * voxel):
        for pose in views:
            got, grgb = vol.raycast(K, pose, size, step, color=True)
            want, wrgb = CO.raycast_color(F.cpu().numpy(), W_host, C.cpu().numpy(), lo, voxel, K, pose, size, step)
            assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32))
            grgb = grgb.cpu().numpy()
            assert np.array_equal(np.isnan(grgb), np.isnan(wrgb)) and np.isnan(wrgb).any() == (want == 0).any()
            ok = ~np.isnan(wrgb)
            assert np.array_equal(grgb[ok].view(np.int32), wrgb[ok].view(np.int32))
            hits += int((want > 0).sum())
    assert hits > 5000


def test_graph_capture_and_the_empty_volume():
    vol = _sparse(0.05, True)
    K = (100.0, 100.0, 39.5, 29.5)
    pose = VO.look_at((0.0, 0.0, -1.0), CENTER)
    z, c = vol.raycast(K, pose, (60, 80), color=True)
    assert not z.any() and torch.isnan(c).all()
    v, f, cv = vol.extract_mesh()
    assert v.shape == (0, 3) and f.shape == (0, 3) and cv.shape == (0, 3)
    assert vol.to_dense()[1] == (0, 0, 0)
    K2, T, depth, rgb = _scene(0.05, color=True)
    vol.integrate(torch.from_numpy(depth).to(dev), K2, T, torch.from_numpy(rgb).to(dev))
    eager = vol.raycast(K2, pose, (45, 60), color=True)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = vol.raycast(K2, pose, (45, 60), color=True)
    g.replay()
    torch.cuda.synchronize()
    assert (eager[0] > 0).any()
    assert torch.equal(_bits(out[0]), _bits(eager[0])) and torch.equal(_bits(out[1]), _bits(eager[1]))
    vol.reset()
    assert vol.blocks == 0 and not vol.raycast(K2, pose, (45, 60)).any()


def test_refusals():
    from omnidata_b200 import _capi
    vol = _sparse(0.05, True)
    d = torch.ones(1, 24, 32, device=dev)
    rgb = torch.zeros(1, 3, 24, 32, device=dev)
    K = (30.0, 30.0, 15.5, 11.5)
    far = np.eye(4)
    far[0, 3] = 0.4 * _capi.SPARSE_TSDF_BLOCK_RANGE
    n0 = _capi.launch_count()
    for call in (lambda: vol.integrate(d, K, far, rgb), lambda: vol.raycast(K, far, (24, 32)),
                 lambda: vol.integrate(d, K, np.eye(4)), lambda: vol.raycast(K, np.eye(4), (24, 32), step=1.0)):
        with pytest.raises(ValueError):
            call()
    assert _capi.launch_count() == n0 and vol.blocks == 0 and vol.frames == 0


def test_beyond_the_dense_limit():
    """1/256 m voxels over the 3 m room: 769^3 points, which the dense volume refuses.  20 frames at 640 x 480 and
    f = 500 px: a pixel covers at most 0.7 / 500 = 1.4 mm of the sphere, below the 3.9 mm voxel."""
    from omnidata_b200.volume import TSDFVolume
    from test_volume_gpu import _check_sphere, _sphere_part
    voxel = 1.0 / 256
    with pytest.raises(ValueError):
        TSDFVolume((-1.5, -1.5, -1.5), voxel, (769, 769, 769), device=dev)
    K, T, depth, _ = _scene(voxel, n_poses=20, size=(480, 640), f=500.0)
    vol = _sparse(voxel)
    for q in range(0, 20, 5):
        vol.integrate(torch.from_numpy(depth[q:q + 5]).to(dev), K, T[q:q + 5])
    dense_bytes = 8 * 769 ** 3
    print(f"1/256 m voxels: {vol.blocks} blocks, {vol.blocks * 512 * 8 / 2**20:.0f} MB against {dense_bytes / 2**20:.0f}"
          f" MB dense")
    v, f, _ = vol.extract_mesh()
    v, fs, r = _sphere_part(v, f, voxel)
    _check_sphere(v, fs, r, voxel, "1/256 m sparse")


# ---------------------------------------------------------------- loop closure and the unposed paths
SIZE, FOCAL = (120, 160), 150.0
KL = (FOCAL, FOCAL, (SIZE[1] - 1) / 2, (SIZE[0] - 1) / 2)
FINE = 0.0125
LAMBDA = 1e-2


def _run(path, seed, closure, lam):
    """test_loop_gpu._run with a SparseTSDFVolume in place of the dense volume."""
    import reconstruct
    from omnidata_b200.loop import LoopClosure
    from omnidata_b200.sparse import SparseDepthAligner
    from omnidata_b200.track import FrameTracker
    from test_loop_gpu import _depth, _rgb, _t
    rng = np.random.default_rng(seed)
    T0 = path[0]
    vol = _sparse(FINE, lam > 0)
    aligner = SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST)
    trackers = {a: FrameTracker(affine=a, photometric=lam) for a in (False, True)}
    loop = LoopClosure(KL, SIZE, photometric=lam) if closure else None
    last, poses = np.eye(4), []
    for q, T in enumerate(path):
        d = _depth(T)
        s1, t1 = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
        pred = _t((s1 * d + t1).astype(np.float32)).unsqueeze(0)
        rgb = _rgb(T) if lam > 0 else None
        if q == 0:
            sp = np.zeros(SIZE, np.float32)
            idx = rng.choice(d.size, 300, replace=False)
            sp.reshape(-1)[idx] = d.reshape(-1)[idx]
            rec, _ = reconstruct.align_and_integrate(vol, aligner, pred, KL, np.eye(4), _t(sp).unsqueeze(0), rgb,
                                                     loop=loop)
            assert int(rec[1]) == 0
            poses.append(np.eye(4))
            continue
        failure, pose, _ = reconstruct.track_and_integrate(vol, aligner, trackers, pred, KL, last, None, rgb, loop)
        assert failure is None, (q, failure)
        last = pose
        poses.append(pose)
    final = loop.poses if closure else np.stack(poses)
    errs = np.array([TO.pose_error(P, np.linalg.inv(T0) @ T) for P, T in zip(final, path)])
    return vol, loop, errs


def test_unposed_photometric_path():
    """test_track_rgbd_gpu.test_unposed_reconstruction_with_colour's bound with the sparse volume."""
    _, _, errs = _run(TO.camera_path(48, CENTER, seed=3), 17, False, LAMBDA)
    print(f"unposed, sparse colour volume, lambda {LAMBDA}: position error max {errs[:, 0].max() * 1e3:.2f} mm (last "
          f"{errs[-1, 0] * 1e3:.2f}), rotation max {np.degrees(errs[:, 1].max()):.3f} deg")
    assert errs[:, 0].max() < 2 * FINE and errs[:, 1].max() < np.radians(1.0)


def test_closed_orbit_and_refusion():
    """test_loop_gpu.test_closed_orbit's assertions with the sparse volume, and LoopClosure.refuse giving the bits of a
    fresh sparse volume that integrates the stored frames at the final poses."""
    path = TO.camera_path(240, CENTER, step_deg=1.5, seed=3)
    _, _, e0 = _run(path, 17, False, LAMBDA)
    vol, loop, e1 = _run(path, 17, True, LAMBDA)
    print(f"closed orbit, sparse volume: {len(loop.keyframes)} keyframes, loops {loop.loops}, {loop.refusions} "
          f"re-fusions, {vol.blocks} blocks")
    for what, e in (("without", e0), ("with", e1)):
        print(f"  {what} loop closure: position error last {e[-1, 0] * 1e3:.2f} mm, max {e[:, 0].max() * 1e3:.2f} mm, "
              f"mean {e[:, 0].mean() * 1e3:.2f} mm; rotation max {np.degrees(e[:, 1].max()):.3f} deg")
    assert loop.loops and max(j for _, j in loop.loops) >= 200 and loop.refusions >= 1
    assert e1[-1, 0] < e0[-1, 0] and e1[:, 0].max() < e0[:, 0].max() and e1[:, 0].mean() < e0[:, 0].mean()
    fresh = _sparse(FINE, True)
    f = loop.frames
    fresh.integrate(loop._metres[:f], KL, loop.poses, loop._rgb[:f])
    assert _same_state(_state(vol), _state(fresh))


def test_reconstruct_cli_without_bounds(tmp_path, capsys):
    """reconstruct.py --synthetic_weights with a sparse volume: runs and writes a mesh; no claim on its quality."""
    import reconstruct
    from PIL import Image
    from test_volume_gpu import _read_ply
    rng = np.random.default_rng(5)
    h = w = 384
    K = (300.0, 300.0, (w - 1) / 2, (h - 1) / 2)
    for sub in ("img", "pose", "sparse"):
        (tmp_path / sub).mkdir()
    for q, pose in enumerate(VO.orbit_poses(3, 1.2, CENTER)):
        Image.fromarray(rng.integers(0, 255, (h, w, 3), dtype=np.uint8)).save(tmp_path / "img" / f"f{q}.png")
        np.savetxt(tmp_path / "pose" / f"f{q}.txt", pose)
        if q in (0, 2):
            d = VO.sphere_room_depth(K, pose, (h, w), CENTER, RADIUS, ROOM_LO, ROOM_HI)
            sp = np.zeros((h, w), np.uint16)
            idx = rng.choice(h * w, 500, replace=False)
            sp.reshape(-1)[idx] = np.rint(d.reshape(-1)[idx] * 1000).astype(np.uint16)
            Image.fromarray(sp).save(tmp_path / "sparse" / f"f{q}.png")
    out = tmp_path / "mesh.ply"
    res = reconstruct.main(["--img_path", str(tmp_path / "img"), "--pose_path", str(tmp_path / "pose"),
                            "--intrinsics", ",".join(str(v) for v in K), "--voxel", "0.05", "--out", str(out),
                            "--synthetic_weights", "--mode", "direct", "--sparse_path", str(tmp_path / "sparse"),
                            "--color"])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert line == res and res["frames"] == 3 and "dims" not in res
    assert res["frames_used"] >= 1 and res["blocks"] > 0 and len(res["bounds"]) == 2
    xyz, idx, rgb = _read_ply(out)
    assert len(xyz) == res["vertices"] and len(idx) == res["faces"] and rgb is not None
