"""Depth-normal fusion without a GPU: the float64 oracle (oracle/fusion_oracle.py) on seeded piecewise-planar scenes
(tilted planes separated by depth steps, no creases, so every kept edge is exact), depth_normals' analytic cases, the
configuration refusals, the evaluate.py flag rules, and the ptxas check of csrc/fusion.cu (no spills or stack frames)."""
import re
import subprocess

import numpy as np
import pytest

from oracle import fusion_oracle as FO

K = (60.0, 60.0, 31.5, 23.5)                      # 48 x 64 images


def _scene(seed=0):
    return FO.planes_scene(48, 64, K, seed)


def test_exact_normals_without_shift_keep_the_depth():
    z, c = _scene()
    r = FO.fuse(z, c, K, shift=False)
    assert r["status"] == FO.STATUS_OK and r["n"] == 48 * 64 and r["kept"] > 0
    assert np.max(np.abs(r["z"] - z)) <= 1e-12


def test_the_bordered_solve_matches_the_eliminated_operator():
    z, c = _scene(1)
    a = z + 0.01 * np.random.default_rng(2).standard_normal(z.shape)
    for shift in (True, False):
        r = FO.fuse(a, c, K, shift=shift)
        mv, b, _ = FO.system(a, c, K, shift=shift)
        assert np.linalg.norm(b - mv(r["z"])) <= 1e-12 * np.linalg.norm(b)


def test_shift_is_recovered_to_the_kappa_bound():
    z, c = _scene()
    r = FO.fuse(z + 0.5, c, K)
    err_t, err_z = abs(r["t"] + 0.5), np.max(np.abs(r["z"] - z) / z)
    kappa = FO.KAPPA
    try:
        FO.KAPPA = 1e-12
        r0 = FO.fuse(z + 0.5, c, K)
    finally:
        FO.KAPPA = kappa
    err_z0 = np.max(np.abs(r0["z"] - z) / z)
    print(f"kappa 1e-6: t error {err_t:.1e}, z {err_z:.1e} relative; kappa 1e-12: z {err_z0:.1e}")
    # the error is the ridge's bias alone: it falls with kappa in proportion
    assert err_t <= 1e-3 and err_z <= 1e-3 and err_z0 <= 1e-6 * err_z * 1.1 + 1e-12


def test_fronto_parallel_scene_stays_finite():
    a = 3.0 + 0.01 * np.random.default_rng(3).standard_normal((48, 64))
    c = np.stack([np.full((48, 64), 0.5), np.full((48, 64), 0.5), np.ones((48, 64))])
    r = FO.fuse(a, c, K)
    assert np.isfinite(r["z"]).all() and abs(r["t"]) <= 1e-6


def test_normal_sign_and_axes():
    z, c = _scene()
    a = z + 0.5
    r = FO.fuse(a, c, K)
    neg = FO.fuse(a, 1.0 - c, K)                               # n -> -n
    assert np.max(np.abs(neg["z"] - r["z"])) <= 1e-12 and neg["kept"] == r["kept"]
    flipped = FO.fuse(a, c, K, axes=(-1, -1, -1))              # one axis sign wrong
    assert np.max(np.abs(flipped["z"] - r["z"])) > 1e-3 and abs(flipped["t"] + 0.5) > 1e-2


def test_high_frequency_noise_is_reduced():
    z, c = _scene(4)
    noise = 0.01 * np.random.default_rng(5).standard_normal(z.shape)
    r = FO.fuse(z + noise, c, K)
    ratio = np.sqrt(np.mean((r["z"] - z) ** 2)) / np.sqrt(np.mean(noise ** 2))
    print(f"RMS error after / before fusion: {ratio:.3f}")
    assert ratio <= 0.65                                       # 0.614 measured on this scene


def test_status_rules():
    z, c = _scene()
    assert FO.fuse(z, c, K, mask=np.zeros(z.shape))["status"] == FO.STATUS_EMPTY
    r = FO.fuse(np.full(z.shape, 2.0), c, K)
    assert r["status"] == FO.STATUS_FLAT and np.isnan(r["z"]).all()
    a = z.copy()
    a[3:6, 4:9] = np.nan
    c2 = c.copy()
    c2[1, 20:24, 30:33] = np.nan
    r = FO.fuse(a, c2, K)
    assert r["n"] == 48 * 64 - 15 and np.array_equal(np.isnan(r["z"]), np.isnan(a))


def test_depth_normals_analytic_cases():
    flat = np.full((8, 10), 2.0)
    out = FO.depth_normals(flat, K)
    assert np.array_equal(out[:, 4, 5], np.array([0.5, 0.5, 1.0], np.float32))
    assert np.array_equal(out, np.broadcast_to(np.array([0.5, 0.5, 1.0], np.float32)[:, None, None], out.shape))
    n = np.array([0.3, -0.2, -1.0])
    n /= np.linalg.norm(n)
    rx, ry = FO.rays(20, 30, K)
    r = np.stack(np.broadcast_arrays(rx[None, :], ry[:, None], np.ones((20, 30))))
    z = 2.0 * n[2] / np.tensordot(n, r, 1)                     # n . X = 2 n_z < 0: facing the camera
    got = 2.0 * FO.depth_normals(z, K, jump=1.0).astype(np.float64) - 1.0
    want = np.array([1.0, -1.0, -1.0]) * n
    assert np.max(np.abs(got - want[:, None, None])) <= 1.2e-7      # the fp32 rounding of the encoding only
    # the same in fp64: the oracle's arithmetic before the final rounding gives the analytic normal to 1e-12
    X = z * r
    tx, ty = X[:, 5, 7] - X[:, 5, 5], X[:, 6, 6] - X[:, 4, 6]
    m = np.cross(ty, tx)
    m /= np.linalg.norm(m)
    assert np.max(np.abs(m - n)) <= 1e-12
    assert np.isnan(FO.depth_normals(np.ones((1, 1)), K)).all()
    assert np.isnan(FO.depth_normals(np.arange(7.0)[None], K)).all()
    step = np.ones((10, 12))
    step[:, 6:] = 3.0                                          # a step: edges across it are dropped
    out = FO.depth_normals(step, K)
    assert np.isfinite(out).all() and np.array_equal(out[:, :, 5], out[:, :, 2])


def test_configuration_refusals():
    from omnidata_b200.fusion import DepthNormalFusion
    DepthNormalFusion()
    DepthNormalFusion(weight=1.0, shift=False, jump=0.1, iterations=1, tol=1e-3, axes=(1, 1, 1))
    for kw in ({"weight": 0.0}, {"weight": float("nan")}, {"shift": 1}, {"jump": 0.0}, {"jump": float("inf")},
               {"iterations": 0}, {"iterations": 10001}, {"iterations": 2.5}, {"tol": 0.0}, {"tol": 1.0},
               {"axes": (1, -1)}, {"axes": (1, 0, -1)}, {"axes": (True, -1, -1)}):
        with pytest.raises(ValueError):
            DepthNormalFusion(**kw)


def test_input_refusals_before_any_launch():
    import torch
    from omnidata_b200.fusion import DepthNormalFusion, depth_normals
    fus = DepthNormalFusion()
    d, n = torch.zeros(1, 8, 8), torch.zeros(1, 3, 8, 8)
    for intr in ((0.0, 1.0, 0.0, 0.0), (1.0, -1.0, 0.0, 0.0), (1.0, 1.0, float("nan"), 0.0), (1.0, 1.0, 0.0),
                 "abc"):
        with pytest.raises(ValueError):
            fus.fit(d, n, intr)
        with pytest.raises(ValueError):
            depth_normals(d, intr)
    with pytest.raises(ValueError):
        fus.fit(d, torch.zeros(1, 3, 8, 9), (1.0, 1.0, 0.0, 0.0))
    with pytest.raises(ValueError):
        fus.fit(d, n, (1.0, 1.0, 0.0, 0.0), torch.ones(1, 8, 9))
    with pytest.raises(ValueError):
        depth_normals(d, (1.0, 1.0, 0.0, 0.0), axes=(1, 2, 1))


def test_evaluate_flag_rules():
    import evaluate
    base = ["--task", "depth", "--img_path", "i", "--gt_path", "g", "--synthetic_weights"]
    a = evaluate.parse_args(base + ["--fuse_normals", "--intrinsics", "500,500,319.5,239.5"])
    assert a.fuse_normals and a.intrinsics == (500.0, 500.0, 319.5, 239.5) and a.fusion_weight == 0.1
    assert not a.no_shift
    a = evaluate.parse_args(base + ["--fuse_normals", "--intrinsics", "1,1,0,0", "--fusion_weight", "2", "--no_shift"])
    assert a.fusion_weight == 2.0 and a.no_shift
    a = evaluate.parse_args(base)
    assert not a.fuse_normals and a.intrinsics is None
    ck = ["--task", "depth", "--img_path", "i", "--gt_path", "g", "--checkpoint", "c"]
    evaluate.parse_args(ck + ["--fuse_normals", "--intrinsics", "1,1,0,0", "--normal_checkpoint", "n"])
    for argv in (base + ["--fuse_normals"], base + ["--intrinsics", "1,1,0,0"], base + ["--no_shift"],
                 base + ["--fusion_weight", "1"], base + ["--normal_checkpoint", "n"],
                 base + ["--fuse_normals", "--intrinsics", "0,1,0,0"], base + ["--fuse_normals", "--intrinsics", "1,1"],
                 base + ["--fuse_normals", "--intrinsics", "1,1,0,0", "--fusion_weight", "0"],
                 base + ["--fuse_normals", "--intrinsics", "1,1,0,0", "--normal_checkpoint", "n"],
                 ck + ["--fuse_normals", "--intrinsics", "1,1,0,0"],
                 ["--task", "normal", "--img_path", "i", "--gt_path", "g", "--synthetic_weights", "--fuse_normals",
                  "--intrinsics", "1,1,0,0"]):
        with pytest.raises(SystemExit):
            evaluate.parse_args(argv)


def test_fusion_kernels_do_not_spill(tmp_path):
    """csrc/fusion.cu compiled as the build compiles it (without fast-math): no stack frame, no spills."""
    from omnidata_b200 import build
    assert "fusion.cu" in build.SOURCES and "fusion.cu" not in build.FAST_MATH_SOURCES
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "fusion.cu"), "-o",
           str(tmp_path / "fusion.o")]
    try:
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600).stdout
    except FileNotFoundError:
        pytest.skip("nvcc not available")
    kernels = 0
    for line in out.splitlines():
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            kernels += 1
            assert m.groups() == ("0", "0", "0"), line
    assert kernels >= 8, out
