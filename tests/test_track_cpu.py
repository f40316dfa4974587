"""Camera tracking on the CPU: the float64 oracle's SE(3) exponential against scipy's expm, its Jacobian against
central differences, recovery of a perturbed pose and a corrupted scale and shift on the analytic sphere-in-a-room
scene, the degenerate single-wall view, the chunk-partial fold ordered_sum8, the host-side refusals of FrameTracker, ops.track_frame and reconstruct.py, and
the ptxas check of csrc/track.cu (no spills or stack frames)."""
import re
import subprocess

import numpy as np
import pytest
import scipy.linalg
import torch

from oracle import sparse_oracle as SO
from oracle import track_oracle as TO
from oracle import volume_oracle as VO

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)
H, W = 60, 80
K = (60.0, 60.0, (W - 1) / 2, (H - 1) / 2)


def _depth(pose, size=(H, W), k=K):
    return VO.sphere_room_depth(k, pose, size, CENTER, RADIUS, ROOM_LO, ROOM_HI)


def _twist_matrix(xi):
    v, w = xi[:3], xi[3:]
    X = np.zeros((4, 4))
    X[:3, :3] = [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]
    X[:3, 3] = v
    return X


@pytest.mark.parametrize("theta", [0.0, 1e-8, 1e-4, 0.0099999, 0.01, 0.0100001, 0.3, 2.5])
def test_exponential_matches_expm(theta):
    rng = np.random.default_rng(int(theta * 1e7) % 1000)
    axis = rng.standard_normal(3)
    xi = np.concatenate([rng.uniform(-0.2, 0.2, 3), theta * axis / np.linalg.norm(axis)])
    R, u = TO.se3_exp(xi)
    E = scipy.linalg.expm(_twist_matrix(xi))
    assert np.abs(R - E[:3, :3]).max() <= 1e-12 and np.abs(u - E[:3, 3]).max() <= 1e-12


def test_jacobian_matches_central_differences():
    """e(T exp(xi), s, t) with the association held fixed: d e / d(xi, s, t) at 0 against the oracle's rows."""
    ref = TO.camera_path(1, CENTER)[0]
    rng = np.random.default_rng(1)
    T = TO.perturb(ref, 0.02, np.radians(1.5), rng)
    d_ref = _depth(ref).astype(np.float32)
    pred = (1.3 * _depth(T) - 0.1).astype(np.float32)
    normals = TO.model_normals(d_ref, K)
    s, t = 1 / 1.3 + 0.01, 0.1 / 1.3 - 0.02
    Rm, tm = TO.relative_pose(ref, T)
    A = TO.associate(pred, d_ref, normals, K, Rm, tm, s, t, 0.1, 0.02)
    corr = A["corr"]
    assert corr.sum() > 0.5 * corr.size

    def e_at(x):
        Re, u = TO.se3_exp(x[:6])
        Tn = np.eye(4)
        Tn[:3, :3] = T[:3, :3] @ Re
        Tn[:3, 3] = T[:3, :3] @ u + T[:3, 3]
        return TO.residual(pred, d_ref, normals, K, *TO.relative_pose(ref, Tn), s + x[6], t + x[7], A)[corr]

    for k in range(8):
        h = 1e-6
        dx = np.zeros(8)
        dx[k] = h
        fd = (e_at(dx) - e_at(-dx)) / (2 * h)
        assert np.abs(fd - A["J"][corr][:, k]).max() <= 1e-6 * max(1.0, np.abs(fd).max()), k


def _oracle_recovery(h, w):
    k = (float(w) * 0.75, float(w) * 0.75, (w - 1) / 2, (h - 1) / 2)
    ref = TO.camera_path(1, CENTER)[0]
    rng = np.random.default_rng(0)
    truth = TO.perturb(ref, 0.03, np.radians(2.0), rng)
    d_ref = _depth(ref, (h, w), k).astype(np.float32)
    pred = (1.7 * _depth(truth, (h, w), k) - 0.2).astype(np.float32)
    nodes, _ = SO.fit(pred, d_ref, robust=0.05, iterations=5)
    T, (s, t), rec = TO.track(pred, d_ref, k, ref, None, nodes.reshape(2), iterations=30)
    dp, dr = TO.pose_error(T, truth)
    print(f"oracle recovery at {w}x{h}: {dp * 1e3:.3f} mm, {np.degrees(dr):.4f} deg, s 1.7 - 1 = {s * 1.7 - 1:.2e}, "
          f"{int(rec[4])} iterations")
    assert rec[1] == TO.OK and rec[4] < 30
    assert abs(s * 1.7 - 1) < 1e-3 and abs(t - 0.2 / 1.7) < 2e-3
    return dp, dr


def test_ordered_sum8_adds_in_the_folds_order():
    """Inputs whose sum depends on the order: lane l adds parts l, l + 8, ... from 0.0, then lanes 0..7 in order."""
    big = 1e16                                   # big + 1.0 rounds back to big
    # lane 0: big + (-big) = 0, lanes 1..7: 1.0 each -> 7.0; added in index order every 1.0 is lost -> 0.0
    a = np.r_[big, [1.0] * 7, -big]
    # one part per lane: 7.0 from lanes 0..6 is added to lane 7's big at once; one at a time it would be lost
    b = np.r_[[1.0] * 7, big]
    assert TO.ordered_sum8(a) == 7.0
    assert TO.ordered_sum8(b) == 7.0 + big != big
    seq = 0.0
    for v in a:
        seq += v
    assert seq == 0.0                            # the plain ascending order gives another value
    cols = TO.ordered_sum8(np.stack([a, np.r_[b, 0.0]], 1))     # columns are independent
    assert cols.shape == (2,) and cols[0] == 7.0 and cols[1] == 7.0 + big
    assert TO.ordered_sum8(np.ones((3, 2, 2))).tolist() == [[3.0, 3.0], [3.0, 3.0]]


def test_oracle_recovers_pose_scale_and_shift():
    """A 3 cm, 2 degree perturbation and pred = 1.7 d - 0.2 from initial nodes fitted to the reference at ref_pose.

    The error is not 1e-6 even with the exact analytic reference: the minimum of the point-to-plane energy is not at the
    true pose.  Each frame point is paired with the nearest reference pixel, and the reference normal there is a finite
    difference: on the sphere the tangent plane at V_q misses Q by up to |Q - V_q|^2 / 2r, always on the same side, and
    pixels on the room's concave corners carry normals averaged across two walls.  Both effects shrink with the pixel
    footprint, and so does the error: 0.49 mm and 0.016 degrees at 80x60, 0.15 mm and 0.003 degrees at 160x120 (0.047 mm
    at 320x240), at the same field of view.  The test checks that it shrinks by at least a factor 2."""
    coarse = _oracle_recovery(H, W)
    fine = _oracle_recovery(2 * H, 2 * W)
    assert coarse[0] < 1e-3 and coarse[1] < np.radians(0.05)
    assert fine[0] < 0.5 * coarse[0] and fine[1] < 0.5 * coarse[1]


def test_single_wall_is_degenerate():
    eye = np.array([0.0, 0.0, 0.0])
    ref = VO.look_at(eye, eye + np.array([1.0, 0.0, 0.0]))            # facing the wall x = 1.5 squarely
    k = (200.0, 200.0, (W - 1) / 2, (H - 1) / 2)                        # a narrow view: the wall fills the frame
    d = VO.sphere_room_depth(k, ref, (H, W), (0.0, 0.0, -40.0), 0.1, ROOM_LO, ROOM_HI)
    assert np.allclose(d, d[H // 2, W // 2] / 1.0, rtol=0.2)
    for affine in (True, False):
        T, nodes, rec = TO.track(d.astype(np.float32), d.astype(np.float32), k, ref, None, (1.0, 0.0) if affine
                                 else None, affine=affine)
        assert rec[1] == TO.DEGENERATE and np.array_equal(T, ref)


def test_tracker_refusals():
    from omnidata_b200 import _capi, ops
    from omnidata_b200.track import FrameTracker
    bad = [dict(affine=1), dict(iterations=0), dict(iterations=101), dict(iterations=2.5), dict(tol=0.0),
           dict(tol=float("nan")), dict(robust=-1.0), dict(max_dist=float("inf")), dict(min_overlap=0.0),
           dict(min_overlap=1.5)]
    for kw in bad:
        with pytest.raises(ValueError):
            FrameTracker(**kw)
        args = dict(affine=True, iterations=20, tol=1e-6, robust=0.02, max_dist=0.1, min_overlap=0.1)
        args.update(kw)
        with pytest.raises(_capi.OdbError):
            ops.check_track_params("t", *args.values())
    tr = FrameTracker()
    cpu = torch.zeros(H, W)
    with pytest.raises(ValueError):
        tr.track(cpu, cpu, K, np.eye(4), init_nodes=torch.zeros(1, 1, 1, 2, dtype=torch.float64))
    with pytest.raises(_capi.OdbError):
        ops.track_frame(cpu, cpu, torch.zeros(3, H, W), K, np.eye(4), np.eye(4), None, False, 20, 1e-6, 0.02, 0.1, 0.1,
                        torch.zeros(8, dtype=torch.float64), torch.zeros(4, 4, dtype=torch.float64),
                        torch.zeros(1, 1, 1, 2, dtype=torch.float64), torch.zeros(8, dtype=torch.float64))


def test_reconstruct_tracking_arguments(tmp_path):
    import reconstruct
    base = ["--img_path", "i", "--intrinsics", "500,500,319.5,239.5", "--voxel", "0.02", "--bounds=-1,-1,-1,1,1,1",
            "--out", "m.ply", "--synthetic_weights", "--sparse_path", "s"]
    a = reconstruct.parse_args(base)
    assert a.pose_path is None and not a.track and a.pose_out is None
    a = reconstruct.parse_args(base + ["--pose_path", "p", "--track", "--pose_out", str(tmp_path / "new")])
    assert a.track and a.pose_out == str(tmp_path / "new")
    (tmp_path / "file.txt").write_text("x")
    for argv in (base + ["--track"],                                             # nothing to refine
                 base + ["--pose_out", str(tmp_path / "file.txt")],              # a file, not a directory
                 base[:-2]):                                                     # frame 0 still needs sparse depths
        with pytest.raises(SystemExit):
            reconstruct.parse_args(argv)


def test_track_kernels_do_not_spill(tmp_path):
    """csrc/track.cu compiled as the build compiles it (without fast-math): no stack frame, no spills."""
    from omnidata_b200 import build
    assert "track.cu" in build.SOURCES and "track.cu" not in build.FAST_MATH_SOURCES
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "track.cu"), "-o",
           str(tmp_path / "track.o")]
    try:
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600).stdout
    except FileNotFoundError:
        pytest.skip("nvcc not available")
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert len(frames) >= 3, out
    assert all(f == ("0", "0", "0") for f in frames), out
