"""The photometric tracking term and the coloured raycast on the CPU: the float64 oracle's photometric Jacobian against
central differences, its luminance and Sobel gradient against a direct numpy restatement, the textured single wall
(degenerate without the term, solved with it), the host-side refusals of FrameTracker, ops.track_frame,
ops.tsdf_raycast_color and reconstruct.py, and the ptxas check of csrc/volume.cu (no spills or stack frames; track.cu's
is tests/test_track_cpu.py's)."""
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import color_volume_oracle as CO
from oracle import photometric_oracle as PO
from oracle import track_oracle as TO
from oracle import volume_oracle as VO

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)
H, W = 60, 80
K = (60.0, 60.0, (W - 1) / 2, (H - 1) / 2)


def _scene(pose, size=(H, W), k=K):
    return (VO.sphere_room_depth(k, pose, size, CENTER, RADIUS, ROOM_LO, ROOM_HI),
            CO.sphere_room_rgb(k, pose, size, CENTER, RADIUS, ROOM_LO, ROOM_HI).astype(np.float32))


def test_texture_is_smooth_and_varies():
    """Colours lie in [0.05, 0.95]; the luminance changes by a few percent per pixel at the tests' resolution."""
    d, c = _scene(TO.camera_path(1, CENTER)[0], (120, 160), (150.0, 150.0, 79.5, 59.5))
    assert c.min() >= 0.05 and c.max() <= 0.95
    Y = PO.luminance(c)
    step = np.abs(np.diff(Y, axis=1))
    assert np.median(step) > 2e-3 and np.percentile(step[np.abs(np.diff(d, axis=1)) < 0.05], 99) < 0.1


def test_luminance_and_sobel_match_numpy():
    ref = TO.camera_path(1, CENTER)[0]
    d, c = _scene(ref)
    d = d.astype(np.float32)
    rng = np.random.default_rng(0)
    d[rng.random(d.shape) < 0.02] = 0.0                               # holes
    c[:, rng.random(d.shape) < 0.02] = np.nan                         # no colour
    normals = TO.model_normals(d, K)
    ig = PO.intensity_gradient(d, c, normals)
    cd = c.astype(np.float64)
    Y = 0.299 * cd[0] + 0.587 * cd[1] + 0.114 * cd[2]
    usable = (d > 0) & np.isfinite(cd).all(0) & np.isfinite(normals).all(0)
    assert np.array_equal(np.isfinite(ig[0]), usable)
    assert np.abs(ig[0][usable] - Y[usable]).max() <= 1e-7
    gu = np.full((H, W), np.nan)
    gv = np.full((H, W), np.nan)
    for y in range(1, H - 1):
        for x in range(1, W - 1):
            win = np.s_[y - 1:y + 2, x - 1:x + 2]
            if usable[win].all() and np.all(np.abs(d[win].astype(np.float64) - float(d[y, x])) <= 0.05 * d[y, x]):
                Yw = Y[win]
                gu[y, x] = ((Yw[:, 2] - Yw[:, 0]) * np.array([1.0, 2.0, 1.0])).sum() / 8.0
                gv[y, x] = ((Yw[2, :] - Yw[0, :]) * np.array([1.0, 2.0, 1.0])).sum() / 8.0
    for got, want in ((ig[1], gu), (ig[2], gv)):
        assert np.array_equal(np.isfinite(got), np.isfinite(want))
        ok = np.isfinite(want)
        assert ok.sum() > 0.5 * ok.size and np.abs(got[ok] - want[ok]).max() <= 1e-7


def test_gradient_is_undefined_across_depth_steps():
    """depth_normals keeps one-sided normals at a depth step, so the gradient's own step test has to keep the sphere's
    silhouette out: every window that straddles it has no gradient."""
    ref = TO.camera_path(1, CENTER)[0]
    d, c = _scene(ref)
    d = d.astype(np.float32)
    normals = TO.model_normals(d, K)
    ig = PO.intensity_gradient(d, c, normals)
    step = np.zeros((H, W), bool)
    jump = np.abs(np.diff(d.astype(np.float64), axis=1)) > 0.2
    step[:, 1:] |= jump
    step[:, :-1] |= jump
    assert step.sum() > 20
    assert np.isfinite(normals[:, step].sum(0)).any()           # the normals alone would let these through
    grown = step.copy()
    grown[1:, :] |= step[:-1, :]
    grown[:-1, :] |= step[1:, :]
    assert not np.isfinite(ig[1][grown]).any() and not np.isfinite(ig[2][grown]).any()


def test_photometric_jacobian_matches_central_differences():
    """e_c(T exp(xi), s, t) with the association (bilinear base, interpolated intensity and gradient) held fixed:
    d e_c / d(xi, s, t) at 0 against the oracle's rows."""
    ref = TO.camera_path(1, CENTER)[0]
    T = TO.perturb(ref, 0.02, np.radians(1.5), np.random.default_rng(1))
    d_ref, c_ref = _scene(ref)
    d_ref = d_ref.astype(np.float32)
    d, rgb = _scene(T)
    pred = (1.3 * d - 0.1).astype(np.float32)
    normals = TO.model_normals(d_ref, K)
    ig = PO.intensity_gradient(d_ref, c_ref, normals)
    s, t = 1 / 1.3 + 0.01, 0.1 / 1.3 - 0.02
    Rm, tm = TO.relative_pose(ref, T)
    A = PO.associate(pred, d_ref, normals, K, Rm, tm, s, t, 0.1, 0.02)
    Ph = PO.photometric(A, rgb, ig, K, Rm, 0.1)
    corr = Ph["corr"]
    assert corr.sum() > 0.5 * A["corr"].sum()

    def e_at(x):
        Re, u = TO.se3_exp(x[:6])
        Tn = np.eye(4)
        Tn[:3, :3] = T[:3, :3] @ Re
        Tn[:3, 3] = T[:3, :3] @ u + T[:3, 3]
        return PO.photometric_residual(pred, rgb, K, *TO.relative_pose(ref, Tn), s + x[6], t + x[7], Ph)[corr]

    for k in range(8):
        h = 1e-6
        dx = np.zeros(8)
        dx[k] = h
        fd = (e_at(dx) - e_at(-dx)) / (2 * h)
        assert np.abs(fd - Ph["J"][corr][:, k]).max() <= 1e-6 * max(1.0, np.abs(fd).max()), k


def _wall(pose, k):
    d = VO.sphere_room_depth(k, pose, (H, W), (0.0, 0.0, -40.0), 0.1, ROOM_LO, ROOM_HI).astype(np.float32)
    c = CO.sphere_room_rgb(k, pose, (H, W), (0.0, 0.0, -40.0), 0.1, ROOM_LO, ROOM_HI).astype(np.float32)
    return d, c


def test_textured_single_wall_is_solved_with_the_term():
    eye = np.zeros(3)
    ref = VO.look_at(eye, eye + np.array([1.0, 0.0, 0.0]))            # facing the wall x = 1.5 squarely
    k = (200.0, 200.0, (W - 1) / 2, (H - 1) / 2)
    d, c = _wall(ref, k)
    T, _, rec = TO.track(d, d, k, ref, None, None, affine=False)
    assert rec[1] == TO.DEGENERATE and np.array_equal(T, ref)
    T, _, rec = PO.track(d, d, k, ref, c, c, affine=False, photometric=1e-2)
    assert rec[1] == TO.OK and len(rec) == 11 and rec[8] > 0.8 * rec[0]
    truth = TO.perturb(ref, 0.02, np.radians(1.5), np.random.default_rng(3))
    dt, ct = _wall(truth, k)
    T, _, rec = PO.track(dt, d, k, ref, ct, c, affine=False, photometric=1e-2, iterations=30)
    dp, dr = TO.pose_error(T, truth)
    assert rec[1] == TO.OK and dp < 1e-3 and dr < np.radians(0.01)


def test_photometric_refusals():
    from omnidata_b200 import _capi, ops
    from omnidata_b200.track import FrameTracker
    for kw in (dict(photometric=-1e-3), dict(photometric=float("nan")), dict(photometric=float("inf")),
               dict(photometric=True), dict(photometric_robust=0.0), dict(photometric_robust=float("nan"))):
        with pytest.raises(ValueError):
            FrameTracker(**kw)
        args = dict(photometric=1e-3, photometric_robust=0.1)
        args.update(kw)
        with pytest.raises(_capi.OdbError):
            ops.check_photometric("t", *args.values())
    cpu = torch.zeros(H, W)
    rgb = torch.zeros(3, H, W)
    n0 = torch.zeros(1, 1, 1, 2, dtype=torch.float64)
    geo, photo = FrameTracker(), FrameTracker(photometric=1e-2)
    with pytest.raises(ValueError, match="photometric"):
        geo.track(cpu, cpu, K, np.eye(4), init_nodes=n0, rgb=rgb, ref_rgb=rgb)     # rgb without the term
    with pytest.raises(ValueError, match="photometric"):
        photo.track(cpu, cpu, K, np.eye(4), init_nodes=n0)                         # the term without rgb
    with pytest.raises(ValueError, match="photometric"):
        photo.track(cpu, cpu, K, np.eye(4), init_nodes=n0, rgb=rgb)                # no ref_rgb
    with pytest.raises(ValueError, match="rgb must be"):
        photo.track(cpu, cpu, K, np.eye(4), init_nodes=n0, rgb=torch.zeros(3, H, W - 1), ref_rgb=rgb)
    with pytest.raises(ValueError, match="ref_rgb must be"):
        photo.track(cpu, cpu, K, np.eye(4), init_nodes=n0, rgb=rgb, ref_rgb=torch.zeros(1, H, W))
    ws = torch.zeros(8, dtype=torch.float64)
    with pytest.raises(_capi.OdbError):                                            # rgb without lambda
        ops.track_frame(cpu, cpu, torch.zeros(3, H, W), K, np.eye(4), np.eye(4), None, False, 20, 1e-6, 0.02, 0.1,
                        0.1, ws, torch.zeros(4, 4, dtype=torch.float64), n0, torch.zeros(8, dtype=torch.float64),
                        rgb, rgb, rgb, 0.0, 0.1)
    with pytest.raises(_capi.OdbError):                                            # lambda without rgb
        ops.track_frame(cpu, cpu, torch.zeros(3, H, W), K, np.eye(4), np.eye(4), None, False, 20, 1e-6, 0.02, 0.1,
                        0.1, ws, torch.zeros(4, 4, dtype=torch.float64), n0, torch.zeros(11, dtype=torch.float64),
                        photometric=1e-2)
    with pytest.raises(_capi.OdbError):                                            # no colour planes
        ops.tsdf_raycast_color(torch.zeros(4, 4, 4), torch.zeros(4, 4, 4), None, (4, 4, 4), (0, 0, 0), 0.1, K,
                               np.eye(4), 0.05, cpu, rgb)


def test_reconstruct_colour_arguments():
    import reconstruct
    base = ["--img_path", "i", "--intrinsics", "500,500,319.5,239.5", "--voxel", "0.02", "--bounds=-1,-1,-1,1,1,1",
            "--out", "m.ply", "--synthetic_weights", "--sparse_path", "s"]
    a = reconstruct.parse_args(base)
    assert not a.color and a.photometric is None
    assert reconstruct.parse_args(base + ["--color"]).color
    a = reconstruct.parse_args(base + ["--photometric", "1e-3"])
    assert a.color and a.photometric == 1e-3
    a = reconstruct.parse_args(base + ["--pose_path", "p", "--track", "--photometric", "1e-3"])
    assert a.color and a.track
    assert reconstruct.parse_args(base + ["--pose_path", "p", "--color"]).color
    for argv in (base + ["--pose_path", "p", "--photometric", "1e-3"],          # posed, nothing is tracked
                 base + ["--photometric", "0"], base + ["--photometric", "-1"], base + ["--photometric", "nan"]):
        with pytest.raises(SystemExit):
            reconstruct.parse_args(argv)


def test_volume_kernels_do_not_spill(tmp_path):
    """csrc/volume.cu compiled as the build compiles it (without fast-math), both raycast instantiations included: no
    stack frame, no spills."""
    from omnidata_b200 import build
    assert "volume.cu" in build.SOURCES and "volume.cu" not in build.FAST_MATH_SOURCES
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "volume.cu"), "-o",
           str(tmp_path / "volume.o")]
    try:
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600).stdout
    except FileNotFoundError:
        pytest.skip("nvcc not available")
    assert len(re.findall(r"tsdf_raycast_kernelILb[01]E", out)) >= 2, out
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert len(frames) >= 7, out
    assert all(f == ("0", "0", "0") for f in frames), out
