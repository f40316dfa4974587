"""Loop closure end to end on the GPU (LoopClosure, reconstruct.py --loop_closure; omnidata_b200/loop.py over
csrc/track.cu, csrc/posegraph.cu and csrc/volume.cu).

- A closed 360-degree orbit of the analytic sphere-in-a-room scene, unposed at 12.5 mm voxels with per-frame scales
  and shifts and sparse depths on frame 0 only, tracked with the photometric term against a colour volume, run with
  and without LoopClosure in the same test: a loop edge is accepted near the end of the orbit, the last frame's, the
  largest and the mean position error fall, and the volume after the last closure is bit-identical to a fresh
  integration of the stored frames at the final poses.
- The 48-frame arc, which never revisits a place: no loop edge, and poses and volume bit-identical to the run without.
- A forced candidate between keyframes that look at opposite walls is rejected by verification.
- reconstruct.py --loop_closure end to end."""
import json

import numpy as np
import pytest
import torch

from oracle import color_volume_oracle as CO
from oracle import track_oracle as TO
from oracle import volume_oracle as VO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)
SIZE, F = (120, 160), 150.0
K = (F, F, (SIZE[1] - 1) / 2, (SIZE[0] - 1) / 2)
FINE = 0.0125
LAMBDA = 1e-2                               # the photometric weight of tests/test_track_rgbd_gpu.py


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _depth(pose, size=SIZE, k=K):
    return VO.sphere_room_depth(k, pose, size, CENTER, RADIUS, ROOM_LO, ROOM_HI)


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(dev)


def _rgb(pose):
    return _t(CO.sphere_room_rgb(K, pose, SIZE, CENTER, RADIUS, ROOM_LO, ROOM_HI).astype(np.float32))


def _run(path, seed, closure, lam=0.0):
    """test_track_gpu._path_run (unposed; with lam > 0 test_track_rgbd_gpu's, with a colour volume) with an optional
    LoopClosure: (volume, loop, final poses, errors of the final poses against the truth)."""
    import reconstruct
    from omnidata_b200.loop import LoopClosure
    from omnidata_b200.sparse import SparseDepthAligner
    from omnidata_b200.track import FrameTracker
    from omnidata_b200.volume import TSDFVolume
    from test_track_gpu import _room_bounds_in
    rng = np.random.default_rng(seed)
    T0 = path[0]
    origin, dims = _room_bounds_in(T0, FINE)
    vol = TSDFVolume(origin, FINE, dims, color=lam > 0, device=dev)
    aligner = SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST)
    trackers = {a: FrameTracker(affine=a, photometric=lam) for a in (False, True)}
    loop = LoopClosure(K, SIZE, photometric=lam) if closure else None
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
            rec, _ = reconstruct.align_and_integrate(vol, aligner, pred, K, np.eye(4), _t(sp).unsqueeze(0), rgb,
                                                     loop=loop)
            assert int(rec[1]) == 0
            poses.append(np.eye(4))
            continue
        failure, pose, _ = reconstruct.track_and_integrate(vol, aligner, trackers, pred, K, last, None, rgb, loop)
        assert failure is None, (q, failure)
        last = pose
        poses.append(pose)
    final = loop.poses if closure else np.stack(poses)
    errs = np.array([TO.pose_error(P, np.linalg.inv(T0) @ T) for P, T in zip(final, path)])
    return vol, loop, final, errs


def _fresh(vol, loop):
    from omnidata_b200.volume import TSDFVolume
    f = loop.frames
    fresh = TSDFVolume(vol.origin, vol.voxel, vol.dims, color=vol.color is not None, device=dev)
    fresh.integrate(loop._metres[:f], K, loop.poses, None if loop._rgb is None else loop._rgb[:f])
    return fresh


def test_closed_orbit():
    """The closed orbit with the photometric term (tracking and edges), with and without LoopClosure.  Measured: the
    last frame 5.4 -> 4.0 mm and the largest error 10.4 -> 6.9 mm, short of the halving aimed for (the 12.5 mm model's
    bias is 2-3 mm per frame); asserted: a loop near the end, a lower last and largest error, and the re-fusion."""
    path = TO.camera_path(240, CENTER, step_deg=1.5, seed=3)
    vol0, _, _, e0 = _run(path, 17, False, LAMBDA)
    vol1, loop, _, e1 = _run(path, 17, True, LAMBDA)
    print(f"closed orbit, 240 frames: {len(loop.keyframes)} keyframes, loops {loop.loops}, {loop.refusions} "
          f"re-fusions")
    for what, e in (("without", e0), ("with", e1)):
        print(f"  {what} loop closure: position error last {e[-1, 0] * 1e3:.2f} mm, max {e[:, 0].max() * 1e3:.2f} mm, "
              f"mean {e[:, 0].mean() * 1e3:.2f} mm; rotation max {np.degrees(e[:, 1].max()):.3f} deg")
    for what, v in (("without", vol0), ("with", vol1)):
        _, faces, _ = v.extract_mesh()
        f = faces.cpu().numpy().astype(np.int64)
        edges = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
        _, counts = np.unique(edges, axis=0, return_counts=True)
        print(f"  mesh {what}: {len(f)} faces, every edge shared by two faces (watertight): {bool((counts == 2).all())}")
    assert loop.loops and max(j for _, j in loop.loops) >= 200
    assert e1[-1, 0] < e0[-1, 0] and e1[:, 0].max() < e0[:, 0].max() and e1[:, 0].mean() < e0[:, 0].mean()
    assert torch.equal(vol1._data.view(torch.int32), _fresh(vol1, loop)._data.view(torch.int32))


def test_arc_without_revisit_is_unchanged():
    path = TO.camera_path(48, CENTER, seed=3)
    vol0, _, P0, _ = _run(path, 17, False)
    vol1, loop, P1, _ = _run(path, 17, True)
    print(f"48-frame arc: {len(loop.keyframes)} keyframes, loops {loop.loops}")
    assert loop.loops == [] and loop.refusions == 0
    assert np.array_equal(P0, P1)
    assert torch.equal(vol0._data.view(torch.int32), vol1._data.view(torch.int32))


def test_forced_candidate_on_different_walls_is_rejected():
    from omnidata_b200.loop import LoopClosure
    eye = np.array(CENTER)
    A = VO.look_at(eye + np.array([0.0, 0.0, 0.2]), eye + np.array([1.0, 0.0, 0.2]))
    B = VO.look_at(eye + np.array([0.0, 0.0, 0.2]), eye + np.array([-1.0, 0.0, 0.2]))
    loop = LoopClosure(K, SIZE, min_gap=1, radius=10.0, angle=180.0)
    assert not loop.add(_t(_depth(A)), A)
    assert not loop.add(_t(_depth(B)), B)
    assert loop.keyframes == [0, 1] and loop.loops == [] and loop.closures == 0
    assert np.array_equal(loop.poses, np.stack([A, B]))


def test_reconstruct_cli_loop_closure(tmp_path, capsys):
    """Runs end to end with random weights and no poses: the summary's loop-closure keys and the final poses."""
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
    res = reconstruct.main(["--img_path", str(tmp_path / "img"), "--intrinsics", ",".join(str(v) for v in k),
                            "--voxel", "0.05", "--bounds=-1.6,-1.6,0.1,1.6,1.6,3.3", "--out", str(tmp_path / "m.ply"),
                            "--synthetic_weights", "--mode", "direct", "--sparse_path", str(tmp_path / "sparse"),
                            "--loop_closure", "--photometric", str(LAMBDA), "--pose_out", str(tmp_path / "poses")])
    lines = capsys.readouterr().out.strip().splitlines()
    assert json.loads(lines[-1]) == res and res["frames"] == 3
    assert res["keyframes"] >= 1 and res["loops"] == [] and res["refusions"] == 0
    assert len(list((tmp_path / "poses").iterdir())) == res["frames_used"]
