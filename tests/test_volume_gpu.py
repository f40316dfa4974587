"""TSDF volumes on the GPU (TSDFVolume, write_ply, reconstruct.py; csrc/volume.cu).

- Integration against the float64 oracle (oracle/volume_oracle.py) on random generic poses and intrinsics, several
  image sizes, NaN / <= 0 / out-of-frustum depths, with and without colour: W identical, F and colour within 1e-6.
- Frames integrated in one call, one by one, or 3 + 5 give the same bits; a captured CUDA graph replays to eager's bits.
- Raycast against the oracle (hit masks identical, depth within 1e-5 relative) and extraction against the oracle on a
  48^3 grid (faces identical, vertices within 1e-6 relative, repeat extractions bit-identical).
- End to end on the analytic sphere-in-a-room scene: a watertight, outward-wound sphere within a voxel of the truth,
  also when every frame has its own scale and shift and only frame 0 has sparse depths (frame-to-model alignment).
- The empty volume, refusals before any launch, write_ply round trips and reconstruct.py --synthetic_weights."""
import json

import numpy as np
import pytest
import torch

from oracle import volume_oracle as VO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _random_poses(rng, b, target, dist):
    out = []
    for _ in range(b):
        d = rng.standard_normal(3)
        eye = np.asarray(target) + dist * d / np.linalg.norm(d)
        T = VO.look_at(eye, np.asarray(target) + 0.1 * rng.standard_normal(3))
        a = rng.uniform(-np.pi, np.pi)                       # roll about the optical axis
        Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        T[:3, :3] = T[:3, :3] @ Rz
        out.append(T)
    return np.stack(out)


def _random_frames(rng, b, h, w):
    depth = rng.uniform(0.6, 1.6, (b, h, w)).astype(np.float32)
    bad = rng.random((b, h, w))
    depth[bad < 0.05] = np.nan
    depth[(bad >= 0.05) & (bad < 0.08)] = 0.0
    depth[(bad >= 0.08) & (bad < 0.1)] = -1.0
    rgb = rng.random((b, 3, h, w)).astype(np.float32)
    return depth, rgb


def _random_intrinsics(rng, h, w):
    f = rng.uniform(0.6, 1.2) * max(h, w)
    return (f * rng.uniform(0.9, 1.1), f, (w - 1) / 2 + rng.uniform(-3, 3), (h - 1) / 2 + rng.uniform(-3, 3))


def _vol(color=False, dims=(20, 18, 22), origin=(-0.5, -0.45, -0.55), voxel=0.05, trunc=None):
    from omnidata_b200.volume import TSDFVolume
    return TSDFVolume(origin, voxel, dims, trunc=trunc, color=color, device=dev)


def _host(vol):
    c = None if vol.color is None else vol.color.cpu().numpy()
    return vol.tsdf.cpu().numpy(), vol.weight.cpu().numpy(), c


@pytest.mark.parametrize("color", [False, True])
@pytest.mark.parametrize("hw", [(24, 32), (37, 53), (64, 48)])
def test_integrate_matches_the_oracle(hw, color):
    rng = np.random.default_rng(hash(hw) % 1000 + color)
    h, w = hw
    vol = _vol(color)
    F, W, C = _host(vol)
    for call in range(2):
        depth, rgb = _random_frames(rng, 3, h, w)
        K = _random_intrinsics(rng, h, w)
        T = _random_poses(rng, 3, (0.0, 0.0, 0.0), 1.2)
        vol.integrate(torch.from_numpy(depth).to(dev), K, T, torch.from_numpy(rgb).to(dev) if color else None)
        F, W, C = VO.integrate(F, W, C, vol.origin, vol.voxel, vol.trunc, depth, K, T, rgb if color else None)
    g = _host(vol)
    assert np.array_equal(g[1], W) and W.max() >= 2 and (W == 0).any()
    assert np.abs(g[0] - F).max() <= 1e-6
    if color:
        assert np.abs(g[2] - C).max() <= 1e-6


def test_frame_split_gives_the_same_bits():
    rng = np.random.default_rng(7)
    depth, rgb = _random_frames(rng, 8, 40, 56)
    K = _random_intrinsics(rng, 40, 56)
    T = _random_poses(rng, 8, (0.0, 0.0, 0.0), 1.2)
    d, c = torch.from_numpy(depth).to(dev), torch.from_numpy(rgb).to(dev)
    results = []
    for split in ([8], [1] * 8, [3, 5]):
        vol = _vol(True)
        s = 0
        for n in split:
            vol.integrate(d[s:s + n], K, T[s:s + n], c[s:s + n])
            s += n
        results.append(vol._data.clone())
    assert torch.equal(results[0].view(torch.int32), results[1].view(torch.int32))
    assert torch.equal(results[0].view(torch.int32), results[2].view(torch.int32))


def _scene_volume(dims=(48, 48, 48), voxel=None, n_poses=12, size=(90, 120), f=110.0, color=False):
    """A volume over the room's interior with the analytic scene integrated from n orbit poses."""
    voxel = voxel or 3.2 / (dims[0] - 1)
    h, w = size
    K = (f, f, (w - 1) / 2, (h - 1) / 2)
    T = VO.orbit_poses(n_poses, 1.2, CENTER)
    depth = np.stack([VO.sphere_room_depth(K, t, size, CENTER, RADIUS, ROOM_LO, ROOM_HI) for t in T])
    vol = _vol(color, dims=dims, origin=(-1.6, -1.6, -1.6), voxel=voxel)
    rgb = None
    if color:
        y, x = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
        rgb = torch.from_numpy(np.stack([np.stack([x, y, 0.5 + 0 * x])] * n_poses).astype(np.float32)).to(dev)
    vol.integrate(torch.from_numpy(depth.astype(np.float32)).to(dev), K, T, rgb)
    return vol, K, T, depth


def test_raycast_matches_the_oracle():
    vol, K, T, _ = _scene_volume()
    F, W, _ = _host(vol)
    for q, (step, size) in enumerate(((None, (45, 60)), (0.7 * vol.voxel, (31, 47)))):
        pose = VO.look_at((0.9, -0.7, 0.4 - 0.5 * q), CENTER)
        got = vol.raycast(K, pose, size, step).cpu().numpy()
        want = VO.raycast(F, W, vol.origin, vol.voxel, K, pose, size, step)
        assert np.array_equal(got > 0, want > 0) and (want > 0).mean() > 0.2
        hit = want > 0
        assert np.max(np.abs(got[hit] - want[hit]) / want[hit]) <= 1e-5


@pytest.mark.parametrize("color", [False, True])
def test_extraction_matches_the_oracle(color):
    vol, *_ = _scene_volume(color=color)
    F, W, C = _host(vol)
    v, f, c = vol.extract_mesh()
    ov, of, oc = VO.extract_mesh(F, W, C, vol.origin, vol.voxel)
    assert len(of) > 1000
    assert np.array_equal(f.cpu().numpy(), of)
    assert np.all(np.abs(v.cpu().numpy() - ov) <= 1e-6 * np.maximum(np.abs(ov), 1.0))
    if color:
        assert np.all(np.abs(c.cpu().numpy() - oc) <= 1e-6)
    v2, f2, c2 = vol.extract_mesh()
    assert torch.equal(v.view(torch.int32), v2.view(torch.int32)) and torch.equal(f, f2)
    if color:
        assert torch.equal(c.view(torch.int32), c2.view(torch.int32))


def _sphere_part(v, f, voxel):
    v, f = v.cpu().numpy(), f.cpu().numpy()
    r = np.linalg.norm(v.astype(np.float64) - np.asarray(CENTER), axis=1)
    keep = np.all(r[f] < RADIUS + 0.3, axis=1)
    return v, f[keep], r


def _check_sphere(v, f, r, voxel, what):
    edges, mult = VO.mesh_edges(f)
    n = VO.face_normals(v, f)
    area = np.linalg.norm(n, axis=1) / 2
    out = v.astype(np.float64)[f].mean(1) - np.asarray(CENTER)
    inward = np.einsum("ij,ij->i", n, out) <= 0
    # below 1e-3 voxel^2 a sliver's normal is set by the fp32 rounding of its vertices, not by its winding
    big = area > 1e-3 * voxel ** 2
    err = np.abs(r[np.unique(f)] - RADIUS)
    print(f"{what}: {len(f)} faces, sphere distance mean {err.mean() * 1e3:.2f} mm, max {err.max() * 1e3:.2f} mm "
          f"(voxel {voxel * 1e3:.0f} mm); {int(inward.sum())} inward faces, largest {area[inward].max(initial=0):.2e} "
          f"m^2")
    assert len(f) > 1000 and np.all(mult == 2)                     # watertight
    assert VO.signed_volume(v, f) > 0
    assert not np.any(inward & big)                                # outward
    assert err.max() < voxel


# 20 poses on a 1.2 m orbit, 160 x 120 at f = 150 px: a pixel covers at most 1.1 / 150 = 7.3 mm on the sphere, below a
# quarter of the 50 mm voxel
SCENE = dict(dims=(65, 65, 65), voxel=0.05, n_poses=20, size=(120, 160), f=150.0)


def test_sphere_end_to_end():
    vol, *_ = _scene_volume(**SCENE)
    v, f, _ = vol.extract_mesh()
    v, fs, r = _sphere_part(v, f, vol.voxel)
    _check_sphere(v, fs, r, vol.voxel, "end to end")


def test_frame_to_model_alignment():
    import reconstruct
    from omnidata_b200.sparse import SparseDepthAligner
    rng = np.random.default_rng(11)
    h, w = SCENE["size"]
    f = SCENE["f"]
    K = (f, f, (w - 1) / 2, (h - 1) / 2)
    T = VO.orbit_poses(SCENE["n_poses"], 1.2, CENTER)
    order = np.argsort([np.arctan2(t[1, 3], t[0, 3]) + 10 * t[2, 3] for t in T])   # a path: neighbours overlap
    T = T[order]
    vol = _vol(dims=SCENE["dims"], origin=(-1.6, -1.6, -1.6), voxel=SCENE["voxel"])
    aligner = SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST)
    errs = []
    for q, pose in enumerate(T):
        d = VO.sphere_room_depth(K, pose, (h, w), CENTER, RADIUS, ROOM_LO, ROOM_HI)
        s, t = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
        pred = torch.from_numpy((s * d + t).astype(np.float32)).unsqueeze(0).to(dev)
        sparse = None
        if q == 0:
            sp = np.zeros((h, w), np.float32)
            idx = rng.choice(h * w, 300, replace=False)
            sp.reshape(-1)[idx] = d.reshape(-1)[idx]
            sparse = torch.from_numpy(sp).unsqueeze(0).to(dev)
        rec, (sf, tf) = reconstruct.align_and_integrate(vol, aligner, pred, K, pose, sparse)
        assert int(rec[1]) == 0
        errs.append(abs(sf * s - 1.0))                              # the fit maps s d + t back to d: sf = 1 / s
    print(f"recovered scales: |s_fit s - 1| max {max(errs):.2e}, mean {np.mean(errs):.2e}")
    v, f, _ = vol.extract_mesh()
    v, fs, r = _sphere_part(v, f, vol.voxel)
    _check_sphere(v, fs, r, vol.voxel, "aligned")
    assert max(errs) < 0.02


def test_empty_volume_and_graph_replay():
    vol = _vol(True)
    v, f, c = vol.extract_mesh()
    assert v.shape == (0, 3) and f.shape == (0, 3) and c.shape == (0, 3)
    rng = np.random.default_rng(3)
    depth, rgb = _random_frames(rng, 4, 40, 56)
    K = _random_intrinsics(rng, 40, 56)
    T = _random_poses(rng, 4, (0.0, 0.0, 0.0), 1.2)
    d, c = torch.from_numpy(depth).to(dev), torch.from_numpy(rgb).to(dev)
    vol.integrate(d, K, T, c)                                     # the first call at this shape
    vol.reset()
    vol.integrate(d, K, T, c)
    vol.integrate(d, K, T, c)
    eager = vol._data.clone()
    vol.reset()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        vol.integrate(d, K, T, c)
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(vol._data.view(torch.int32), eager.view(torch.int32))


def test_refusals_before_any_launch():
    from omnidata_b200 import _capi
    vol = _vol(True)
    plain = _vol()
    d = torch.ones(2, 24, 32, device=dev)
    rgb = torch.zeros(2, 3, 24, 32, device=dev)
    K = (30.0, 30.0, 15.5, 11.5)
    T = np.stack([np.eye(4)] * 2)
    bad_rot = T.copy()
    bad_rot[0, :3, :3] *= 1.01
    n0 = _capi.launch_count()
    calls = [
        lambda: vol.integrate(d, K, T),                            # no rgb with colour
        lambda: plain.integrate(d, K, T, rgb),                     # rgb without colour
        lambda: vol.integrate(d, K, T[:1], rgb),                   # pose count
        lambda: vol.integrate(d, K, bad_rot, rgb),
        lambda: vol.integrate(d, (0.0, 30.0, 1.0, 1.0), T, rgb),
        lambda: vol.integrate(d.double(), K, T, rgb),
        lambda: vol.integrate(d, K, torch.from_numpy(T).to(dev), rgb),
        lambda: vol.integrate(d, K, T, rgb[:, :2]),
        lambda: vol.raycast(K, T, (24, 32)),                       # two poses
        lambda: vol.raycast(K, T[0], (0, 32)),
        lambda: vol.raycast(K, T[0], (24, 32), step=vol.voxel * 2),
        lambda: vol.raycast(K, T[0], (24, 32), step=0.0),
    ]
    for call in calls:
        with pytest.raises((ValueError, _capi.OdbError)):
            call()
    assert _capi.launch_count() == n0


def _read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode().splitlines()
    nv = int(next(l for l in header if l.startswith("element vertex")).split()[-1])
    nf = int(next(l for l in header if l.startswith("element face")).split()[-1])
    color = any("red" in l for l in header)
    vt = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")] + ([("r", "u1"), ("g", "u1"), ("b", "u1")] if color else [])
    v = np.frombuffer(data, dtype=vt, count=nv, offset=end)
    f = np.frombuffer(data, dtype=[("n", "u1"), ("i", "<i4", (3,))], count=nf, offset=end + v.nbytes)
    assert np.all(f["n"] == 3) and end + v.nbytes + f.nbytes == len(data)
    xyz = np.stack([v["x"], v["y"], v["z"]], 1)
    rgb = np.stack([v["r"], v["g"], v["b"]], 1) if color else None
    return xyz, f["i"], rgb


def test_write_ply_round_trip(tmp_path):
    from omnidata_b200.volume import write_ply
    vol, *_ = _scene_volume(dims=(24, 24, 24), color=True)
    v, f, c = vol.extract_mesh()
    write_ply(tmp_path / "m.ply", v, f, c)
    xyz, idx, rgb = _read_ply(tmp_path / "m.ply")
    assert np.array_equal(xyz, v.cpu().numpy()) and np.array_equal(idx, f.cpu().numpy())
    assert np.array_equal(rgb, np.rint(np.clip(c.cpu().numpy(), 0, 1) * 255).astype(np.uint8))


def test_reconstruct_cli_synthetic_weights(tmp_path, capsys):
    """Runs end to end with random weights; no claim on the mesh's quality."""
    import reconstruct
    from PIL import Image
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
                            "--intrinsics", ",".join(str(v) for v in K), "--voxel", "0.05",
                            "--bounds=-1.6,-1.6,-1.6,1.6,1.6,1.6", "--out", str(out), "--synthetic_weights",
                            "--mode", "direct", "--sparse_path", str(tmp_path / "sparse")])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert line == res and res["frames"] == 3
    assert res["frames_used"] + len(res["frames_skipped"]) == 3
    xyz, idx, rgb = _read_ply(out)
    assert rgb is None and xyz.shape == (res["vertices"], 3) and idx.shape == (res["faces"], 3)
    if len(idx):
        assert idx.min() >= 0 and idx.max() < len(xyz)
