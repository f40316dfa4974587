"""Camera tracking on the GPU (FrameTracker, ops.track_frame, reconstruct.track_and_integrate; csrc/track.cu).

- Oracle parity (oracle/track_oracle.py) on several image sizes, affine on and off, with NaN, 0 and negative
  predictions and holes in the reference: one iteration gives the oracle's correspondence count exactly and its pose and
  nodes within 1e-10; a full run agrees within 1e-7.
- Recovery of perturbed poses, scales and shifts against the exact analytic reference and against a fused TSDF model.
- Unposed reconstruction along a smooth path and pose refinement from noisy poses, through reconstruct.py's step.
- The failure statuses, determinism, CUDA-graph replay, the launch sequence, refusals before any launch and the CLI."""
import json

import numpy as np
import pytest
import torch

from oracle import track_oracle as TO
from oracle import volume_oracle as VO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)
SIZE, F = (120, 160), 150.0                 # at most 7.3 mm per pixel on the sphere
K = (F, F, (SIZE[1] - 1) / 2, (SIZE[0] - 1) / 2)
VOXEL = 0.05


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _depth(pose, size=SIZE, k=K):
    return VO.sphere_room_depth(k, pose, size, CENTER, RADIUS, ROOM_LO, ROOM_HI)


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(dev)


def _nodes(s, t):
    return torch.tensor([s, t], dtype=torch.float64, device=dev).reshape(1, 1, 1, 2)


def _aligner():
    import reconstruct
    from omnidata_b200.sparse import SparseDepthAligner
    return SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST)


@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("hw", [(37, 53), (48, 64), (61, 83)])
def test_matches_the_oracle(hw, affine):
    from omnidata_b200.track import FrameTracker
    h, w = hw
    rng = np.random.default_rng(h * 7 + affine)
    k = (0.9 * w, 0.9 * w, (w - 1) / 2 + 0.3, (h - 1) / 2 - 0.2)
    ref = TO.camera_path(1, CENTER, seed=h)[0]
    truth = TO.perturb(ref, 0.02, np.radians(1.5), rng)
    d_ref = _depth(ref, hw, k).astype(np.float32)
    d_ref[rng.random(hw) < 0.03] = 0.0                                     # holes in the model
    s1, t1 = (rng.uniform(0.6, 1.8), rng.uniform(-0.2, 0.2)) if affine else (1.0, 0.0)
    pred = (s1 * _depth(truth, hw, k) + t1).astype(np.float32)
    bad = rng.random(hw)
    pred[bad < 0.02] = np.nan
    pred[(bad >= 0.02) & (bad < 0.03)] = 0.0
    pred[(bad >= 0.03) & (bad < 0.04)] = -1.0
    init = (1 / s1 * 1.01, -t1 / s1 + 0.01) if affine else None
    for iters in (1, 20):
        tr = FrameTracker(affine=affine, iterations=iters)
        pose, nodes, rec = tr.track(_t(pred), _t(d_ref), k, ref, init_nodes=_nodes(*init) if affine else None)
        normals = tr._bufs["normals"][0].cpu().numpy()
        T, (s, t), orec = TO.track(pred, d_ref, k, ref, None, init, affine=affine, iterations=iters, normals=normals)
        rec = rec.cpu().numpy()
        tol = 1e-10 if iters == 1 else 1e-7
        print(f"{hw} affine={affine} iterations={iters}: {int(rec[0])} correspondences of {int(rec[7])}, status "
              f"{int(rec[1])}, {int(rec[4])} run; oracle {int(orec[4])}; pose diff "
              f"{np.abs(pose.cpu().numpy() - T).max():.2e}")
        assert rec[1] == 0 and orec[1] == 0
        if iters == 1:
            assert rec[0] == orec[0] and rec[7] == orec[7]
        assert rec[4] == orec[4]
        assert np.abs(pose.cpu().numpy() - T).max() <= tol
        assert np.abs(nodes.reshape(2).cpu().numpy() - np.array([s, t])).max() <= tol
        assert abs(rec[2] - orec[2]) <= 1e-9 and abs(rec[3] - orec[3]) <= 1e-12


def _recover(ref_depth, ref, truth, s1, t1, what):
    from omnidata_b200.track import FrameTracker
    pred = _t((s1 * _depth(truth) + t1).astype(np.float32))
    nodes0, rec0 = _aligner().fit(pred.unsqueeze(0), ref_depth.unsqueeze(0))
    assert int(rec0[0, 1]) == 0
    pose, nodes, rec = FrameTracker().track(pred, ref_depth, K, ref, init_nodes=nodes0.clone())
    rec = rec.cpu().numpy()
    dp, dr = TO.pose_error(pose.cpu().numpy(), truth)
    ds = abs(float(nodes[0, 0, 0, 0]) * s1 - 1)
    print(f"{what}: position {dp * 1e3:.3f} mm, rotation {np.degrees(dr):.4f} deg, |s s' - 1| {ds:.2e}, "
          f"{int(rec[4])} iterations, {int(rec[0])} correspondences, RMS {rec[2] * 1e3:.3f} mm, status {int(rec[1])}")
    assert rec[1] == 0
    return dp, dr, ds


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_recovery_against_exact_geometry(seed):
    """Walls are exact planes and the sphere's curvature under a 7 mm pixel is below 0.1 mm."""
    rng = np.random.default_rng(100 + seed)
    ref = TO.camera_path(1, CENTER, seed=seed)[0]
    truth = TO.perturb(ref, rng.uniform(0.0, 0.05), np.radians(rng.uniform(0.0, 3.0)), rng)
    dp, dr, ds = _recover(_t(_depth(ref).astype(np.float32)), ref, truth, rng.uniform(0.5, 2.0),
                          rng.uniform(-0.3, 0.3), f"exact reference, seed {seed}")
    assert dp < 2e-3 and dr < np.radians(0.1) and ds < 5e-3


FINE = 0.0125                               # the voxel of the model-based tests (single frames are accurate there)


def _fused_volume(voxel):
    from omnidata_b200.volume import TSDFVolume
    T = VO.orbit_poses(20, 1.2, CENTER)
    n = int(round(3.2 / voxel)) + 1
    vol = TSDFVolume((-1.6, -1.6, -1.6), voxel, (n, n, n), device=dev)
    vol.integrate(_t(np.stack([_depth(t) for t in T]).astype(np.float32)), K, T)
    return vol


def test_frame_to_model_recovery():
    """Against the raycast of a 257^3 volume with 12.5 mm voxels fused from 20 exact orbit frames: within a quarter
    voxel, and at most a fifth of the initial offset (a tracker that does nothing fails).  The error follows the model:
    measured 2.2-2.7 mm at 12.5 mm voxels, 3.8-5.8 mm at 25 mm and 7-18 mm at 50 mm, where the raycast lies a median 8 mm
    behind the exact surface."""
    vol = _fused_volume(FINE)
    for seed in range(3):
        rng = np.random.default_rng(200 + seed)
        ref = TO.camera_path(1, CENTER, seed=seed)[0]
        off = rng.uniform(0.0, 0.05)
        truth = TO.perturb(ref, off, np.radians(rng.uniform(0.0, 3.0)), rng)
        dp, dr, ds = _recover(vol.raycast(K, ref, SIZE), ref, truth, rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3),
                              f"fused model, voxel {FINE * 1e3} mm, seed {seed}")
        assert dp < FINE / 4 and dp < 0.2 * off and dr < np.radians(0.5) and ds < 5e-3


def test_chained_tracking_against_exact_geometry():
    """The unposed loop's tracking with a perfect model: every frame of the 48-frame path starts from the previous
    estimate and is tracked against the exact depth rendered there.  Errors do not accumulate, so this isolates the
    tracker from the fused model.  Most frames land within 0.2 mm and 0.01 degrees; frames 39-40 of this path see the
    sphere and essentially one wall, whose rotation about the wall's normal through the sphere's centre only a sliver
    of a second wall constrains, and come out 0.35 and 0.28 degrees off (the float64 oracle agrees)."""
    from omnidata_b200.track import FrameTracker
    rng = np.random.default_rng(17)
    path = TO.camera_path(48, CENTER, seed=3)
    aligner, tr = _aligner(), FrameTracker()
    last, errs = path[0], []
    for T in path[1:]:
        s1, t1 = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
        pred = _t((s1 * _depth(T) + t1).astype(np.float32)).unsqueeze(0)
        ref = _t(_depth(last).astype(np.float32))
        n0, _ = aligner.fit(pred, ref.unsqueeze(0))
        pose, _, rec = tr.track(pred, ref, K, last, init_nodes=n0.clone())
        assert int(rec[1]) == 0
        last = pose.cpu().numpy()
        errs.append(TO.pose_error(last, T))
    errs = np.array(errs)
    print(f"chained, exact model: position max {errs[:, 0].max() * 1e3:.3f} mm, rotation max "
          f"{np.degrees(errs[:, 1].max()):.4f} deg, median {np.degrees(np.median(errs[:, 1])):.4f} deg")
    assert errs[:, 0].max() < 1e-3 and errs[:, 1].max() < np.radians(0.5)
    assert np.median(errs[:, 1]) < np.radians(0.01)


def _room_bounds_in(T0, voxel):
    """origin and dims of a grid covering the room in the camera coordinates of T0."""
    corners = np.array([[x, y, z, 1.0] for x in (ROOM_LO[0], ROOM_HI[0]) for y in (ROOM_LO[1], ROOM_HI[1])
                        for z in (ROOM_LO[2], ROOM_HI[2])])
    c = (np.linalg.inv(T0) @ corners.T).T[:, :3]
    lo, hi = c.min(0) - voxel, c.max(0) + voxel
    return tuple(lo), tuple(int(np.ceil((b - a) / voxel)) + 1 for a, b in zip(lo, hi))


def _report_mesh_in_world(vol, T0, what):
    from test_volume_gpu import _sphere_part
    v, f, _ = vol.extract_mesh()
    R0, t0 = torch.from_numpy(T0[:3, :3]).float().to(dev), torch.from_numpy(T0[:3, 3]).float().to(dev)
    v, fs, r = _sphere_part(v @ R0.T + t0, f, vol.voxel)
    edges, mult = VO.mesh_edges(fs)
    err = np.abs(r[np.unique(fs)] - RADIUS)
    print(f"{what}: {len(fs)} sphere faces, watertight {bool(np.all(mult == 2))}, sphere distance mean "
          f"{err.mean() * 1e3:.1f} mm, max {err.max() * 1e3:.1f} mm (voxel {vol.voxel * 1e3:.0f} mm)")
    assert len(fs) > 0


def _path_run(path, voxel, size, f, noisy, seed):
    """reconstruct.py's loop over the path with per-frame scales and shifts and sparse depths on frame 0 only: unposed
    (noisy None: frame 0 at the identity, the grid in its camera coordinates) or refining noisy poses.  Returns the
    volume, the pose errors and, when refining, the input errors."""
    import reconstruct
    from omnidata_b200.track import FrameTracker
    from omnidata_b200.volume import TSDFVolume
    rng = np.random.default_rng(seed)
    h, w = size
    k = (f, f, (w - 1) / 2, (h - 1) / 2)
    T0 = path[0] if noisy is None else np.eye(4)
    if noisy is None:
        origin, dims = _room_bounds_in(T0, voxel)
    else:
        n = int(round(3.2 / voxel)) + 1
        origin, dims = (-1.6, -1.6, -1.6), (n, n, n)
    vol = TSDFVolume(origin, voxel, dims, device=dev)
    aligner = _aligner()
    trackers = {a: FrameTracker(affine=a) for a in (False, True)}
    last, errs, noise = np.eye(4), [], []
    for q, T in enumerate(path):
        truth = np.linalg.inv(T0) @ T
        d = _depth(T, size, k)
        s1, t1 = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
        pred = _t((s1 * d + t1).astype(np.float32)).unsqueeze(0)
        if q == 0:
            sp = np.zeros(size, np.float32)
            idx = rng.choice(d.size, 300, replace=False)
            sp.reshape(-1)[idx] = d.reshape(-1)[idx]
            rec, _ = reconstruct.align_and_integrate(vol, aligner, pred, k, truth, _t(sp).unsqueeze(0))
            assert int(rec[1]) == 0
            continue
        init = last if noisy is None else TO.perturb(T, noisy[0], noisy[1], rng)
        noise.append(TO.pose_error(init, truth))
        failure, pose, _ = reconstruct.track_and_integrate(vol, aligner, trackers, pred, k, init)
        assert failure is None, (q, failure)
        last = pose
        errs.append(TO.pose_error(pose, truth))
    return vol, T0, np.array(errs), np.array(noise)


def test_unposed_reconstruction():
    """Every frame of a 48-frame path is tracked (12.5 mm voxels).  The trajectory drifts more than the half voxel we
    aimed for: measured 13.5 mm and 0.39 degrees at most.  Each frame's error becomes part of the model the next frame
    is tracked against, so the weakly constrained views of test_chained_tracking_against_exact_geometry and the model's
    bias (test_frame_to_model_recovery) accumulate; the drift scales with the voxel (123, 36 and 13.5 mm at 50, 25 and
    12.5 mm).  The bound below is two voxels, against the 1.4 m the path travels (a tracker that does nothing is off by
    metres); the mesh is reported, not checked.  reconstruct.py documents the unposed mode as experimental."""
    vol, T0, errs, _ = _path_run(TO.camera_path(48, CENTER, seed=3), FINE, SIZE, F, None, 17)
    print(f"unposed: 48 frames, position error max {errs[:, 0].max() * 1e3:.2f} mm (last {errs[-1, 0] * 1e3:.2f}), "
          f"rotation max {np.degrees(errs[:, 1].max()):.3f} deg")
    assert errs[:, 0].max() < 2 * FINE and errs[:, 1].max() < np.radians(1.0)
    _report_mesh_in_world(vol, T0, "unposed")


def test_pose_refinement():
    """Frame 0's pose is exact (it fixes the model's frame); the others start 20 mm and 1.5 degrees off (320x240,
    12.5 mm voxels).  Every refined pose must be closer to the truth than its input, and the mean error at most half
    the input's: measured at most 14.8 mm, mean 6.8 mm.  The 2 mm we aimed for is not reached, for the reasons of
    test_unposed_reconstruction; reconstruct.py documents --track as experimental.  The mesh is reported, not
    checked."""
    vol, T0, errs, noise = _path_run(TO.camera_path(40, CENTER, seed=5), FINE, (240, 320), 2 * F,
                                     (0.02, np.radians(1.5)), 17)
    print(f"refined: position error max {errs[:, 0].max() * 1e3:.2f} mm, mean {errs[:, 0].mean() * 1e3:.2f} mm "
          f"(input {noise[:, 0].mean() * 1e3:.1f} mm); rotation max {np.degrees(errs[:, 1].max()):.3f} deg "
          f"(input {np.degrees(noise[:, 1].max()):.2f})")
    assert np.all(errs[:, 0] < noise[:, 0]) and errs[:, 0].mean() < 0.5 * noise[:, 0].mean()
    assert np.all(errs[:, 1] < noise[:, 1])
    _report_mesh_in_world(vol, T0, "refined")


def test_failure_statuses_return_the_initial_state():
    from omnidata_b200.track import FrameTracker
    from omnidata_b200.volume import TSDFVolume
    ref = TO.camera_path(1, CENTER)[0]
    init = TO.perturb(ref, 0.01, np.radians(0.5), np.random.default_rng(0))
    pred = _t(_depth(ref).astype(np.float32))
    empty = TSDFVolume((-1.6, -1.6, -1.6), VOXEL, (65, 65, 65), device=dev).raycast(K, ref, SIZE)
    eye = VO.look_at((0.0, 0.0, 0.0), (1.0, 0.0, 0.0))
    kw = (400.0, 400.0, K[2], K[3])
    wall = _t(VO.sphere_room_depth(kw, eye, SIZE, (0.0, 0.0, -40.0), 0.1, ROOM_LO, ROOM_HI).astype(np.float32))
    cases = [("no_overlap", pred, empty, K, ref, init, _nodes(1.0, 0.0)),
             ("degenerate", wall, wall, kw, eye, eye, _nodes(1.02, -0.01)),
             ("nonfinite", pred, _t(_depth(ref).astype(np.float32)), K, ref, init, _nodes(float("nan"), 0.0))]
    from omnidata_b200.track import STATUS
    for name, p, r, k, rp, ip, n0 in cases:
        pose, nodes, rec = FrameTracker().track(p, r, k, rp, ip, n0)
        rec = rec.cpu().numpy()
        assert STATUS[int(rec[1])] == name, (name, rec)
        assert np.array_equal(pose.cpu().numpy().view(np.int64), np.asarray(ip, np.float64).view(np.int64))
        assert torch.equal(nodes.view(torch.int64), n0.view(torch.int64))
        assert not np.isnan(pose.cpu().numpy()).any() and not np.isnan(rec[[0, 1, 2, 3, 4, 7]]).any()


def test_determinism_graph_capture_and_launches():
    from omnidata_b200 import _capi, ops
    from omnidata_b200.track import FrameTracker
    ref = TO.camera_path(1, CENTER)[0]
    truth = TO.perturb(ref, 0.03, np.radians(2.0), np.random.default_rng(4))
    pred, r = _t((1.3 * _depth(truth) - 0.1).astype(np.float32)), _t(_depth(ref).astype(np.float32))
    n0 = _nodes(0.78, 0.08)
    tr = FrameTracker(iterations=20)
    out = [t.clone() for t in tr.track(pred, r, K, ref, init_nodes=n0)]          # the first call at this shape
    torch.cuda.synchronize()
    a0, l0 = torch.cuda.memory_stats(dev)["allocation.all.allocated"], _capi.launch_count()
    again = tr.track(pred, r, K, ref, init_nodes=n0)
    torch.cuda.synchronize()
    launches = _capi.launch_count() - l0
    assert torch.cuda.memory_stats(dev)["allocation.all.allocated"] == a0
    for x, y in zip(out, again):
        assert torch.equal(x.view(torch.int64), y.view(torch.int64))
    l1 = _capi.launch_count()
    ops.track_frame(pred, r, tr._bufs["normals"], K, ref, ref, n0, True, 20, 1e-6, 0.02, 0.1, 0.1,
                    tr._bufs["workspace"], tr._bufs["pose"], tr._bufs["nodes"], tr._bufs["record"])
    assert _capi.launch_count() - l1 == 20 + 2                   # setup, 20 steps, output
    print(f"launches per FrameTracker.track: {launches} (depth_normals {launches - 22}, tracking 22)")
    for t in tr._bufs.values():
        if t.dtype == torch.float64:
            t.fill_(float("nan"))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = tr.track(pred, r, K, ref, init_nodes=n0)
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(out, res):
        assert torch.equal(x.view(torch.int64), y.view(torch.int64))


def test_refusals_before_any_launch():
    from omnidata_b200 import _capi
    from omnidata_b200.track import FrameTracker
    ref = np.eye(4)
    d = torch.ones(24, 32, device=dev)
    n0 = _nodes(1.0, 0.0)
    bad_rot = ref.copy()
    bad_rot[:3, :3] *= 1.01
    k = (30.0, 30.0, 15.5, 11.5)
    tr, metric = FrameTracker(), FrameTracker(affine=False)
    n = _capi.launch_count()
    calls = [
        lambda: tr.track(d, torch.ones(24, 31, device=dev), k, ref, init_nodes=n0),          # shape
        lambda: tr.track(d.double(), d, k, ref, init_nodes=n0),                             # dtype
        lambda: tr.track(d.cpu(), d.cpu(), k, ref, init_nodes=n0),                          # device
        lambda: tr.track(d, d, k, torch.from_numpy(ref).to(dev), init_nodes=n0),            # device pose
        lambda: tr.track(d, d, k, bad_rot, init_nodes=n0),                                  # not orthonormal
        lambda: tr.track(d, d, k, ref, bad_rot, init_nodes=n0),
        lambda: tr.track(d, d, (0.0, 30.0, 1.0, 1.0), ref, init_nodes=n0),                  # intrinsics
        lambda: tr.track(d, d, k, ref),                                                     # no init_nodes
        lambda: metric.track(d, d, k, ref, init_nodes=n0),                                  # init_nodes, metric
        lambda: tr.track(d, d, k, ref, init_nodes=n0.float()),
        lambda: tr.track(d, d, k, ref, init_nodes=n0.reshape(2)),
        lambda: FrameTracker(iterations=0),
        lambda: FrameTracker(max_dist=-1.0),
        lambda: FrameTracker(min_overlap=2.0),
    ]
    for call in calls:
        with pytest.raises((ValueError, _capi.OdbError)):
            call()
    assert _capi.launch_count() == n


def test_reconstruct_cli_without_poses(tmp_path, capsys):
    """Runs end to end with random weights and no poses; no claim on the mesh's quality."""
    import reconstruct
    from PIL import Image
    rng = np.random.default_rng(6)
    h = w = 384
    k = (300.0, 300.0, (w - 1) / 2, (h - 1) / 2)
    for sub in ("img", "sparse"):
        (tmp_path / sub).mkdir()
    for q, pose in enumerate(TO.camera_path(3, CENTER)):
        Image.fromarray(rng.integers(0, 255, (h, w, 3), dtype=np.uint8)).save(tmp_path / "img" / f"f{q}.png")
        if q == 0:
            d = VO.sphere_room_depth(k, pose, (h, w), CENTER, RADIUS, ROOM_LO, ROOM_HI)
            sp = np.zeros((h, w), np.uint16)
            idx = rng.choice(h * w, 500, replace=False)
            sp.reshape(-1)[idx] = np.rint(d.reshape(-1)[idx] * 1000).astype(np.uint16)
            Image.fromarray(sp).save(tmp_path / "sparse" / f"f{q}.png")
    out = tmp_path / "mesh.ply"
    res = reconstruct.main(["--img_path", str(tmp_path / "img"), "--intrinsics", ",".join(str(v) for v in k),
                            "--voxel", "0.05", "--bounds=-1.6,-1.6,0.1,1.6,1.6,3.3", "--out", str(out),
                            "--synthetic_weights", "--mode", "direct", "--sparse_path", str(tmp_path / "sparse"),
                            "--pose_out", str(tmp_path / "poses")])
    line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert line == res and res["frames"] == 3
    assert res["frames_used"] + len(res["frames_skipped"]) == 3
    written = sorted(p.name for p in (tmp_path / "poses").iterdir())
    assert len(written) == res["frames_used"]
    for p in written:
        assert reconstruct.load_pose(tmp_path / "poses" / p).shape == (4, 4)
    assert out.exists()
