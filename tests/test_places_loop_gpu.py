"""Place recognition and relocalisation end to end on the GPU (LoopClosure(places=True), reconstruct.py
--place_recognition; omnidata_b200/loop.py over csrc/places.cu, csrc/track.cu, csrc/posegraph.cu and csrc/volume.cu) on
the analytic sphere-in-a-room scene of tests/test_loop_gpu.py.

- Loops beyond the pose radius: the closed 240-frame orbit followed by its first 16 frames again, true metres and
  images at poses with injected drift that grows smoothly to 0.5 m and 3 degrees at the end (none at frame 0).  As
  reconstruct.py continues from the corrected pose after a closure, each later pose carries the last closure's
  correction.  Without places no loop is accepted; with them a loop to an early keyframe is accepted on the second
  pass and the solve removes the drift.  The orbit alone does not do: its height and aim wander, so the views near its
  end differ from its first ones as much as unrelated views do (dissimilarity about 0.8, DESIGN.md §6).
- Relocalisation: an unposed, photometric run over orbit frames 0-119, then a jump back to frames 20-59.  Without
  place recognition the tracker does not report the jump: every later frame tracks with status ok to a pose more
  than half a metre off (a failure relocalisation cannot see).  With it the first frame after the jump is relocalised,
  as reconstruct.py does after a failure, and every later frame is tracked from there, within a small multiple of
  the largest error before the jump; the relocalisation's edge is not proposed again as a loop.
- A covered lens: blank frames in the run fail their fit, relocalisation is tried and fails, the frames are skipped
  with status "relocalise: failed" and the run goes on from the last good pose.
- The 48-frame arc, which never revisits a place, with places=True.
- reconstruct.py --place_recognition end to end."""
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
LAMBDA = 1e-2
DRIFT = (0.5, 3.0)                          # metres, degrees at the last frame


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _depth(pose):
    return VO.sphere_room_depth(K, pose, SIZE, CENTER, RADIUS, ROOM_LO, ROOM_HI)


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(dev)


def _rgb(pose):
    return _t(CO.sphere_room_rgb(K, pose, SIZE, CENTER, RADIUS, ROOM_LO, ROOM_HI).astype(np.float32))


def _drift(s):
    """The world-frame drift at fraction s of the path: a turn of s * 3 degrees about a tilted axis through the origin
    and a shift of s * 0.5 m, both growing smoothly from none."""
    axis = np.array([0.2, 0.3, 1.0]) / np.linalg.norm([0.2, 0.3, 1.0])
    a = np.radians(DRIFT[1]) * s
    Kx = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    D = np.eye(4)
    D[:3, :3] = np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx
    D[:3, 3] = DRIFT[0] * s * np.array([0.6, -0.48, 0.64])
    return D


def _feed_drifted(path, places):
    from omnidata_b200.loop import LoopClosure
    loop = LoopClosure(K, SIZE, photometric=LAMBDA, places=places)
    n = len(path)
    drifted = [_drift(q / (n - 1)) @ T for q, T in enumerate(path)]
    C = np.eye(4)                   # the last closure's correction, carried onto the later poses
    for T, Td in zip(path, drifted):
        if loop.add(_t(_depth(T)), C @ Td, _rgb(T)):
            C = loop.poses[-1] @ np.linalg.inv(Td)
    return loop, np.stack(drifted)


def test_loops_beyond_the_pose_radius():
    orbit = TO.camera_path(240, CENTER, step_deg=1.5, seed=3)
    path = np.concatenate([orbit, orbit[:16]])
    loop0, drifted = _feed_drifted(path, False)
    loop1, _ = _feed_drifted(path, True)
    injected = np.array([TO.pose_error(A, B)[0] for A, B in zip(drifted, path)])
    kf = loop1.keyframes
    before = np.array([TO.pose_error(drifted[f], path[f])[0] for f in kf])
    after = np.array([TO.pose_error(loop1.poses[f], path[f])[0] for f in kf])
    print(f"drifted orbit: {len(kf)} keyframes; injected drift up to {injected.max() * 1e3:.1f} mm; loops without "
          f"places {loop0.loops}, with {loop1.loops}; keyframe position error max {before.max() * 1e3:.1f} -> "
          f"{after.max() * 1e3:.1f} mm, mean {before.mean() * 1e3:.1f} -> {after.mean() * 1e3:.1f} mm")
    assert loop0.loops == [] and loop0.closures == 0                # the premise: beyond the pose radius
    assert loop1.loops and max(j for _, j in loop1.loops) >= 240 and min(i for i, _ in loop1.loops) <= 20
    # measured on the H100: 454 -> 0.6 mm largest, 247 -> 0.4 mm mean
    assert after.max() < 0.1 * injected.max() and after.max() < 0.005


def _run(frames, places, seed=17, lost=(), blank=()):
    """test_loop_gpu._run's unposed photometric tracking with LoopClosure over the orbit frames given (indices into
    the 240-frame orbit), relocalising failed frames with places, the frames at the positions in `lost` as if their
    tracking had failed and those in `blank` seen through a covered lens (a flat prediction, a black image):
    (loop, per-frame (failure, error) list)."""
    import reconstruct
    from omnidata_b200.loop import LoopClosure
    from omnidata_b200.sparse import SparseDepthAligner
    from omnidata_b200.track import FrameTracker
    from omnidata_b200.volume import TSDFVolume
    from test_track_gpu import _room_bounds_in
    orbit = TO.camera_path(240, CENTER, step_deg=1.5, seed=3)
    rng = np.random.default_rng(seed)
    T0 = orbit[frames[0]]
    origin, dims = _room_bounds_in(T0, FINE)
    vol = TSDFVolume(origin, FINE, dims, color=True, device=dev)
    aligner = SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST)
    trackers = {a: FrameTracker(affine=a, photometric=LAMBDA) for a in (False, True)}
    loop = LoopClosure(K, SIZE, photometric=LAMBDA, places=places)
    last, out = np.eye(4), []
    for q, fi in enumerate(frames):
        T = orbit[fi]
        d = _depth(T)
        s1, t1 = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
        pred = _t((s1 * d + t1).astype(np.float32)).unsqueeze(0)
        rgb = _rgb(T)
        if q in blank:
            pred, rgb = torch.full_like(pred, 1.0), torch.zeros_like(rgb)
        if q == 0:
            sp = np.zeros(SIZE, np.float32)
            idx = rng.choice(d.size, 300, replace=False)
            sp.reshape(-1)[idx] = d.reshape(-1)[idx]
            rec, _ = reconstruct.align_and_integrate(vol, aligner, pred, K, np.eye(4), _t(sp).unsqueeze(0), rgb,
                                                     loop=loop)
            assert int(rec[1]) == 0
            out.append((None, 0.0))
            continue
        failure, pose = "track: lost", None
        if q not in lost:
            failure, pose, _ = reconstruct.track_and_integrate(vol, aligner, trackers, pred, K, last, None, rgb, loop)
        if failure is not None and places:
            failure, pose, _ = reconstruct.relocalise_and_integrate(vol, aligner, trackers, loop, pred, K, None, rgb)
            if failure is None:
                failure = "relocalised"
        if pose is not None:
            last = pose
        out.append((failure, None if pose is None else TO.pose_error(pose, np.linalg.inv(T0) @ T)[0]))
    return loop, out


def test_relocalisation_after_a_jump():
    frames = list(range(120)) + list(range(20, 60))
    loop0, r0 = _run(frames, False)
    loop1, r1 = _run(frames, True, lost=(120,))
    before = max(e for f, e in r1[:120] if f is None)
    after = [e for _, e in r1[120:]]
    print(f"jump 119 -> 20: without places {sum(f is not None for f, _ in r0[120:])} of 40 frames fail, the "
          f"smallest error after the jump {min(e for f, e in r0[120:] if e is not None):.3f} m; with places failures "
          f"{[(q, f) for q, (f, _) in enumerate(r1) if f not in (None,)]}; relocalisations {loop1.relocalisations}; "
          f"largest error before the jump {before * 1e3:.2f} mm, after "
          f"{max(e for e in after if e is not None) * 1e3:.2f} mm; loops {loop1.loops}")
    assert all(f is None for f, _ in r0[:120]) and all(f is None for f, _ in r1[:120])
    assert all(f is None and e > 0.5 for f, e in r0[120:])        # the premise: lost for the rest of the video
    assert r1[120][0] == "relocalised" and all(f is None for f, _ in r1[121:])
    assert loop1.relocalisations and loop1.relocalisations[0][1] == 120
    assert max(after) <= 3.0 * before
    assert (loop1.relocalisations[0][0], 120) not in loop1.loops        # its edge is not proposed again
    assert len(set(loop1._edges)) == len(loop1._edges)


def test_covered_lens_fails_relocalisation_and_the_run_goes_on():
    """reconstruct.py's trigger as it happens: blank frames fail their fit, relocalisation is tried and finds nothing,
    and the frames are skipped; the pending state stays clear and the following frames track as before."""
    frames = list(range(40))
    loop, r = _run(frames, True, blank=(20, 21, 22))
    print(f"covered lens at frames 20-22: {[(q, f) for q, (f, _) in enumerate(r) if f is not None]}")
    assert [f for f, _ in r[20:23]] == ["relocalise: failed"] * 3
    assert all(f is None for q, (f, _) in enumerate(r) if q not in (20, 21, 22))
    assert loop._reloc is None and loop.relocalisations == [] and loop.frames == 37
    assert max(e for f, e in r[23:]) < 0.02


def test_arc_without_revisit_with_places():
    loop, r = _run(list(range(48)), True)
    print(f"48-frame arc with places: {len(loop.keyframes)} keyframes, loops {loop.loops}, relocalisations "
          f"{loop.relocalisations}")
    assert all(f is None for f, _ in r)
    assert loop.loops == [] and loop.relocalisations == []


def test_reconstruct_cli_place_recognition(tmp_path, capsys):
    """Runs end to end with random weights and no poses: the summary has the relocalised frames."""
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
                            "--loop_closure", "--photometric", str(LAMBDA), "--place_recognition"])
    lines = capsys.readouterr().out.strip().splitlines()
    assert json.loads(lines[-1]) == res and res["frames"] == 3
    print(f"reconstruct --place_recognition: {res}")
    assert "relocalised" in res and set(res["relocalised"]) <= {"f1.png", "f2.png"}
    assert res["frames_used"] + len(res["frames_skipped"]) == 3
    assert all(s["status"] == "relocalise: failed" for s in res["frames_skipped"])
