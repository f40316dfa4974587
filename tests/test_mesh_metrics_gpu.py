"""Mesh metrics on the GPU (omnidata_b200.mesh, MeshMetrics, reconstruct.py --gt_mesh, evaluate_mesh.py;
csrc/mesh_metrics.cu) against the float64 oracle (oracle/mesh_oracle.py).

- Surface sampling equals the oracle bit for bit on seeded random meshes with degenerate and sliver faces and on a mesh
  extracted from the analytic volume; bad indices and NaN vertices are refused before any sample is emitted.
- nearest equals brute force exactly (distance bits, indices) on ties, lattices, cell boundaries, far queries, one
  reference point, one cell, clustered sets and an empty reference, and the cKDTree oracle on 4e6 x 4e6 points of the
  analytic room; the cell size changes no bit.
- Culling equals the oracle's mask; MeshMetrics matches the oracle (counts exact, values within 1e-12) and repeats
  bit for bit.
- End to end on the analytic scene: dense and sparse volumes fused from exact depth at 12.5 mm voxels against the exact
  ground-truth mesh, and uncorrected per-frame scale / shift errors scoring worse than frame-to-model alignment.
- reconstruct.py --gt_mesh --gt_cull and evaluate_mesh.py run end to end."""
import json

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as MO
from oracle import volume_oracle as VO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _t(a, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).to(dev)


def _bits(x):
    return np.asarray(x).view(np.uint64 if np.asarray(x).dtype == np.float64 else np.uint32)


def _random_mesh(rng, nv=300, nf=800):
    v = rng.uniform(-1.0, 1.0, (nv, 3)).astype(np.float32)
    f = rng.integers(0, nv, (nf, 3)).astype(np.int32)
    f[:40, 1] = f[:40, 0]                                         # degenerate: a repeated vertex
    v[f[40:80, 2]] = (v[f[40:80, 0]] + v[f[40:80, 1]]) * 0.5      # collinear slivers (up to fp32 rounding)
    v[f[80:120, 2]] = v[f[80:120, 0]] + 1e-4 * rng.standard_normal((40, 3)).astype(np.float32)   # thin slivers
    return v, f


@pytest.mark.parametrize("seed,stream,density", [(0, 0, 300.0), (7, 1, 50.0), (2 ** 40 + 3, 5, 2000.0)])
def test_sampling_matches_the_oracle_on_random_meshes(seed, stream, density):
    from omnidata_b200 import mesh
    v, f = _random_mesh(np.random.default_rng(seed % 1000))
    got = mesh.sample_surface(_t(v), _t(f), density, seed, stream).cpu().numpy()
    n, want = MO.sample_surface(v, f, density, seed, stream)
    assert got.shape == want.shape and len(want) == n.sum() > 1000
    assert np.array_equal(_bits(got), _bits(want))


def test_sampling_matches_the_oracle_on_an_extracted_mesh():
    from omnidata_b200 import mesh
    from omnidata_b200.volume import TSDFVolume
    F, W = VO.sphere_sdf_volume((40, 40, 40), (-0.6, -0.6, -0.6), 0.03, (0.01, 0.02, -0.03), 0.45, 0.09)
    vol = TSDFVolume((-0.6, -0.6, -0.6), 0.03, (40, 40, 40), device=dev)
    vol.tsdf.copy_(_t(F))
    vol.weight.copy_(_t(W))
    v, f, _ = vol.extract_mesh()
    got = mesh.sample_surface(v, f, 2e4, 3, 1).cpu().numpy()
    n, want = MO.sample_surface(v.cpu().numpy(), f.cpu().numpy(), 2e4, 3, 1)
    assert len(want) > 10000 and np.array_equal(_bits(got), _bits(want))
    assert mesh.sample_surface(v[:0], f[:0]).shape == (0, 3)


def test_sampling_refuses_bad_input_before_emitting():
    from omnidata_b200 import _capi, mesh
    v, f = _random_mesh(np.random.default_rng(1))
    bad_index = f.copy()
    bad_index[17, 2] = len(v)
    nan = v.copy()
    nan[f[33, 1]] = np.nan
    for vv, ff, what in ((v, bad_index, "outside"), (nan, f, "non-finite")):
        n0 = _capi.launch_count()
        with pytest.raises(ValueError, match=what):
            mesh.sample_surface(_t(vv), _t(ff), 100.0)
        assert _capi.launch_count() - n0 <= 4                     # count + scan: no emit
    with pytest.raises(ValueError, match="exceed"):
        mesh.sample_surface(_t(v), _t(f), 1e9)


def _check_nearest(q, r, cells=(None,)):
    from omnidata_b200 import mesh
    want_d, want_i = MO.nearest_brute(q, r)
    for cell in cells:
        d, i = mesh.nearest(_t(q, np.float32), _t(r, np.float32), cell)
        assert np.array_equal(_bits(d.cpu().numpy()), _bits(want_d)), cell
        assert np.array_equal(i.cpu().numpy(), want_i), cell


def test_nearest_equals_brute_force_on_hard_cases():
    rng = np.random.default_rng(4)
    lattice = np.stack(np.meshgrid(*[np.arange(6) * 0.25] * 3, indexing="ij"), -1).reshape(-1, 3)
    dup = np.concatenate([lattice, lattice[::-1], lattice[5:40]])          # every point twice or three times
    q_lattice = np.concatenate([lattice + 0.125, lattice, rng.uniform(-0.2, 1.5, (500, 3))])
    # ties and points on cell boundaries: with cell 0.25 every lattice point lies on a boundary
    _check_nearest(q_lattice.astype(np.float32), dup.astype(np.float32), cells=(None, 0.25, 0.125, 0.1, 2.0))
    # far queries, outside the box on every side
    r = rng.uniform(-1, 1, (3000, 3)).astype(np.float32)
    far = rng.standard_normal((600, 3)) * np.array([[1.0], [30.0], [1e4]]).repeat(200, 0)
    _check_nearest(far.astype(np.float32), r, cells=(None, 0.05, 10.0))
    # one reference point; all points in one cell; strongly clustered
    _check_nearest(rng.uniform(-2, 2, (400, 3)).astype(np.float32), np.array([[0.1, -0.2, 0.3]], np.float32))
    _check_nearest(rng.uniform(-2, 2, (400, 3)).astype(np.float32), r, cells=(5.0,))
    centres = rng.uniform(-5, 5, (4, 3))
    cl = (centres[rng.integers(0, 4, 4000)] + 1e-3 * rng.standard_normal((4000, 3))).astype(np.float32)
    _check_nearest(np.concatenate([cl[:500] + 1e-4, rng.uniform(-6, 6, (500, 3))]).astype(np.float32), cl,
                   cells=(None, 0.05, 0.3))


def test_nearest_empty_and_refusals():
    from omnidata_b200 import mesh
    q = torch.rand(10, 3, device=dev)
    d, i = mesh.nearest(q, q[:0])
    assert torch.isinf(d).all() and (i == -1).all()
    d, i = mesh.nearest(q[:0], q)
    assert d.shape == (0,) and i.shape == (0,)
    bad = q.clone()
    bad[3, 1] = float("nan")
    with pytest.raises(ValueError, match="reference"):
        mesh.nearest(q, bad)
    with pytest.raises(ValueError, match="query"):
        mesh.nearest(bad, q)


def _room_samples(density, stream):
    from omnidata_b200 import mesh
    gv, gf = MO.sphere_room_mesh(CENTER, RADIUS, ROOM_LO, ROOM_HI, 6)
    return mesh.sample_surface(_t(gv, np.float32), _t(gf, np.int32), density, 0, stream)


def test_nearest_equals_the_kdtree_oracle_on_4e6_points_and_cell_size_changes_nothing():
    from omnidata_b200 import mesh
    P, G = _room_samples(7e4, 0), _room_samples(7e4, 1)
    assert P.shape[0] > 3.9e6 and G.shape[0] > 3.9e6
    d, i = mesh.nearest(P, G)
    want_d, want_i = MO.nearest_kdtree(P.cpu().numpy(), G.cpu().numpy())
    assert np.array_equal(_bits(d.cpu().numpy()), _bits(want_d)) and np.array_equal(i.cpu().numpy(), want_i)
    for cell, m in ((0.01, 50000), (0.05, 50000), (0.2, 50000), (4.0, 512)):   # 4 m: one cell holds the room
        d2, i2 = mesh.nearest(P[:m].contiguous(), G, cell)
        assert torch.equal(d2.view(torch.int64), d[:m].view(torch.int64)) and torch.equal(i2, i[:m])


def test_culling_equals_the_oracle():
    from omnidata_b200 import mesh
    P = _room_samples(2e3, 0)
    K, size = (150.0, 150.0, 79.5, 59.5), (120, 160)
    T = VO.orbit_poses(7, 1.2, CENTER)
    got = mesh.frustum_mask(P, K, size, torch.from_numpy(T).to(dev), max_depth=2.5).cpu().numpy()
    want = MO.frustum_mask(P.cpu().numpy(), K, size, T, 2.5)
    assert np.array_equal(got, want) and 0.05 < want.mean() < 0.95
    kept = mesh.compact(P, torch.from_numpy(want).to(dev)).cpu().numpy()
    assert np.array_equal(kept, P.cpu().numpy()[want.astype(bool)])
    # any nonzero mask value keeps a point once (image masks often hold 255)
    m = want * np.random.default_rng(3).choice(np.array([1, 7, 128, 255], np.uint8), len(want))
    kept = mesh.compact(P, torch.from_numpy(m).to(dev)).cpu().numpy()
    assert np.array_equal(kept, P.cpu().numpy()[m != 0])


def _scenes(rng):
    out = []
    for q in range(5):
        gv, gf = _random_mesh(rng, 200, 300)
        pv = gv + rng.normal(0, 0.02 * (q + 1), gv.shape).astype(np.float32)
        out.append((pv, gf[: 200 + 20 * q], gv, gf))
    return out


def test_mesh_metrics_match_the_oracle_and_repeat_bit_for_bit():
    from omnidata_b200 import mesh
    from omnidata_b200.metrics import MeshMetrics
    rng = np.random.default_rng(9)
    scenes = _scenes(rng)
    gv, gf = scenes[0][2:]
    scenes.append((gv[:0], gf[:0], gv, gf))                      # empty prediction
    scenes.append((gv, gf, gv[:0], gf[:0]))                      # no ground truth
    th = (0.02, 0.05, 0.1)
    states, records = [], []
    for run in range(2):
        m = MeshMetrics(thresholds=th, density=300.0, seed=4)
        recs = [m.update(*(_t(a) for a in s)).cpu().numpy()[0] for s in scenes]
        states.append({k: t.cpu().numpy().copy() for k, t in m._state.items()})
        records.append(np.stack(recs))
    assert all(np.array_equal(states[0][k].view(np.uint8), states[1][k].view(np.uint8)) for k in states[0])
    assert np.array_equal(_bits(records[0]), _bits(records[1]))
    # a scene's record does not depend on the scenes before it
    alone = MeshMetrics(thresholds=th, density=300.0, seed=4).update(*(_t(a) for a in scenes[3])).cpu().numpy()[0]
    assert np.array_equal(_bits(alone), _bits(records[0][3]))
    want_sums, want_counts = np.zeros(15), [0] * 7
    for s, got in zip(scenes, records[0]):
        _, P = MO.sample_surface(s[0], s[1], 300.0, 4, 0)
        _, G = MO.sample_surface(s[2], s[3], 300.0, 4, 1)
        dp, _ = MO.nearest_brute(P, G)
        dg, _ = MO.nearest_brute(G, P)
        want = np.asarray(MO.scene_record(dp, dg, th))
        assert np.array_equal(np.isnan(got), np.isnan(want))
        ok = ~np.isnan(want)
        assert np.all(np.abs(got[ok] - want[ok]) <= 1e-12 * np.maximum(np.abs(want[ok]), 1e-300))
        want_counts[0] += 1
        want_counts[1] += len(G) == 0
        want_counts[2] += len(G) > 0 and len(P) == 0
        want_counts[3] += len(P)
        want_counts[4] += len(G)
        if len(G):
            want_sums[3:12] += np.nan_to_num(want[5:14])
            if len(P):
                want_sums[:3] += want[2:5]
    assert states[0]["counts"].tolist() == want_counts
    assert np.allclose(states[0]["sums"], want_sums, rtol=1e-12, atol=0)
    out = m.compute()
    assert out["scenes"] == 7 and out["no_gt"] == 1 and out["empty_pred"] == 1
    assert abs(out["fscore@0.05"] - want_sums[8] / 6) <= 1e-12
    _, dists = MeshMetrics(density=300.0).update(*(_t(a) for a in scenes[1]), return_distances=True)
    assert dists["pred_distance"].shape[0] == dists["pred_points"].shape[0] > 0
    d, _ = mesh.nearest(dists["pred_points"], dists["gt_points"])
    assert torch.equal(d, dists["pred_distance"])


VOXEL = 0.0125
SCENE = dict(n_poses=20, size=(120, 160), f=150.0)


def _scene_frames():
    h, w = SCENE["size"]
    f = SCENE["f"]
    K = (f, f, (w - 1) / 2, (h - 1) / 2)
    T = VO.orbit_poses(SCENE["n_poses"], 1.2, CENTER)
    depth = np.stack([VO.sphere_room_depth(K, t, (h, w), CENTER, RADIUS, ROOM_LO, ROOM_HI) for t in T])
    return K, T, depth


def _score(v, f, K, T, thresholds=(VOXEL, 2 * VOXEL, 0.05), return_distances=False):
    from omnidata_b200.metrics import MeshMetrics
    gv, gf = MO.sphere_room_mesh(CENTER, RADIUS, ROOM_LO, ROOM_HI, 6)
    m = MeshMetrics(thresholds=thresholds)
    r = m.update(v, f, _t(gv, np.float32), _t(gf, np.int32), views=(K, SCENE["size"], T),
                 return_distances=return_distances)
    return (m.compute(), r[1]) if return_distances else m.compute()


def _visible(points, K, T, depth, tol=0.1):
    """The points some frame sees unoccluded: in its frustum and at most tol behind the frame's exact depth there."""
    X = points.astype(np.float64)
    h, w = depth.shape[1:]
    seen = np.zeros(len(X), bool)
    for pose, d in zip(T, depth):
        Xc = (X - pose[:3, 3]) @ pose[:3, :3]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = np.floor(K[0] * Xc[:, 0] / Xc[:, 2] + K[2] + 0.5)
            v = np.floor(K[1] * Xc[:, 1] / Xc[:, 2] + K[3] + 0.5)
        ok = (Xc[:, 2] > 0) & (u >= 0) & (u <= w - 1) & (v >= 0) & (v <= h - 1)
        idx = np.flatnonzero(ok)
        ok[idx] = Xc[idx, 2] <= d[v[idx].astype(int), u[idx].astype(int)] + tol
        seen |= ok
    return seen


@pytest.mark.parametrize("sparse", [False, True])
def test_analytic_scene_end_to_end(sparse):
    """Culling by the frames' frustums keeps the whole room: every wall point lies in some frustum, while the sphere
    hides about half of the walls from every orbit camera.  Occlusion is not modelled, so completion and recall
    against the frustum-culled truth count the hidden walls as missed (7.2 cm, 0.56 at 2 voxels, both volumes).
    Against the truth the frames see unoccluded (the test's own visibility check on the exact depth) completion lies
    within a voxel and F at 2 voxels above 0.9."""
    from omnidata_b200.volume import SparseTSDFVolume, TSDFVolume
    K, T, depth = _scene_frames()
    vol = SparseTSDFVolume(VOXEL, device=dev) if sparse else \
        TSDFVolume((-1.6, -1.6, -1.6), VOXEL, (257, 257, 257), device=dev)
    vol.integrate(_t(depth, np.float32), K, T)
    v, f, _ = vol.extract_mesh()
    out, dist = _score(v, f, K, T, return_distances=True)
    seen = _visible(dist["gt_points"].cpu().numpy(), K, T, depth)
    dg = dist["gt_distance"].cpu().numpy()[seen]
    completion, recall = dg.mean(), (dg < 2 * VOXEL).mean()
    precision = out[f"precision@{2 * VOXEL:g}"]
    fscore = 2 * precision * recall / (precision + recall)
    print(f"{'sparse' if sparse else 'dense'} at {VOXEL * 1e3} mm: {json.dumps(out)}; against the unoccluded truth "
          f"({seen.mean():.3f} of it): completion {completion * 1e3:.2f} mm, recall {recall:.4f}, F {fscore:.4f}")
    assert out["gt_culled"] == 0 and out["completion"] > 4 * VOXEL            # the hidden walls count as missed
    assert out["accuracy"] < VOXEL and precision > 0.99
    assert completion < VOXEL and fscore > 0.9


def test_uncorrected_scale_and_shift_score_worse_than_alignment():
    import reconstruct
    from omnidata_b200.sparse import SparseDepthAligner
    from omnidata_b200.volume import TSDFVolume
    rng = np.random.default_rng(11)
    K, T, depth = _scene_frames()
    order = np.argsort([np.arctan2(t[1, 3], t[0, 3]) + 10 * t[2, 3] for t in T])   # a path: neighbours overlap
    T, depth = T[order], depth[order]
    h, w = SCENE["size"]
    raw = TSDFVolume((-1.6, -1.6, -1.6), VOXEL, (257, 257, 257), device=dev)
    aligned = TSDFVolume((-1.6, -1.6, -1.6), VOXEL, (257, 257, 257), device=dev)
    aligner = SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST)
    for q, (pose, d) in enumerate(zip(T, depth)):
        s, t = (1.0, 0.0) if q == 0 else (rng.uniform(0.9, 1.1), rng.uniform(-0.05, 0.05))
        pred = _t((s * d + t)[None], np.float32)
        raw.integrate(pred, K, pose[None])
        sparse = None
        if q == 0:
            sp = np.zeros((h, w), np.float32)
            idx = rng.choice(h * w, 300, replace=False)
            sp.reshape(-1)[idx] = d.reshape(-1)[idx]
            sparse = _t(sp[None])
        rec, _ = reconstruct.align_and_integrate(aligned, aligner, pred, K, pose, sparse)
        assert int(rec[1]) == 0
    a = _score(*aligned.extract_mesh()[:2], K, T)
    r = _score(*raw.extract_mesh()[:2], K, T)
    key = f"fscore@{2 * VOXEL:g}"
    print(f"aligned: {json.dumps(a)}\nuncorrected: {json.dumps(r)}")
    assert r["chamfer"] > 1.5 * a["chamfer"] and r[key] < a[key] - 0.05


def test_reconstruct_gt_mesh_and_evaluate_mesh_cli(tmp_path, capsys):
    """reconstruct.py --gt_mesh --gt_cull with random weights reports the key (no claim on its values);
    evaluate_mesh.py compares two PLYs."""
    import evaluate_mesh
    import reconstruct
    from PIL import Image
    from omnidata_b200.volume import write_ply
    rng = np.random.default_rng(5)
    h = w = 384
    K = (300.0, 300.0, (w - 1) / 2, (h - 1) / 2)
    for sub in ("img", "pose", "sparse"):
        (tmp_path / sub).mkdir()
    for q, pose in enumerate(VO.orbit_poses(3, 1.2, CENTER)):
        Image.fromarray(rng.integers(0, 255, (h, w, 3), dtype=np.uint8)).save(tmp_path / "img" / f"f{q}.png")
        np.savetxt(tmp_path / "pose" / f"f{q}.txt", pose)
        d = VO.sphere_room_depth(K, pose, (h, w), CENTER, RADIUS, ROOM_LO, ROOM_HI)
        sp = np.zeros((h, w), np.uint16)
        idx = rng.choice(h * w, 500, replace=False)
        sp.reshape(-1)[idx] = np.rint(d.reshape(-1)[idx] * 1000).astype(np.uint16)
        Image.fromarray(sp).save(tmp_path / "sparse" / f"f{q}.png")
    gv, gf = MO.sphere_room_mesh(CENTER, RADIUS, ROOM_LO, ROOM_HI, 4)
    write_ply(tmp_path / "gt.ply", gv.astype(np.float32), gf)
    out = tmp_path / "mesh.ply"
    res = reconstruct.main(["--img_path", str(tmp_path / "img"), "--pose_path", str(tmp_path / "pose"),
                            "--intrinsics", ",".join(str(v) for v in K), "--voxel", "0.05", "--out", str(out),
                            "--synthetic_weights", "--mode", "direct", "--sparse_path", str(tmp_path / "sparse"),
                            "--gt_mesh", str(tmp_path / "gt.ply"), "--gt_cull", "--eval_thresholds", "0.05,0.1"])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    mm = res["mesh_metrics"]
    assert set(line["mesh_metrics"]) == set(mm) and mm["scenes"] == 1 and "fscore@0.1" in mm
    assert line["frames"] == 3 and line["vertices"] == res["vertices"]
    # with loop closure the culling uses LoopClosure.poses, the final poses of the used frames
    res = reconstruct.main(["--img_path", str(tmp_path / "img"), "--pose_path", str(tmp_path / "pose"), "--track",
                            "--photometric", "1e-2", "--loop_closure", "--intrinsics", ",".join(str(v) for v in K),
                            "--voxel", "0.05", "--out", str(out), "--synthetic_weights", "--mode", "direct",
                            "--sparse_path", str(tmp_path / "sparse"), "--gt_mesh", str(tmp_path / "gt.ply"),
                            "--gt_cull"])
    capsys.readouterr()
    mm = res["mesh_metrics"]
    assert res["frames_used"] >= 1 and res["keyframes"] >= 1 and mm["scenes"] == 1 and mm["gt_culled"] > 0
    got = evaluate_mesh.main(["--pred", str(out), "--gt", str(tmp_path / "gt.ply"), "--thresholds", "0.05"])
    assert got["scenes"] == 1 and got["pred_culled"] == got["gt_culled"] == 0
    assert set(json.loads(capsys.readouterr().out.strip().splitlines()[-1])) == set(got)
