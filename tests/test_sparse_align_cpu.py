"""Sparse metric alignment without a GPU: the float64 oracle (oracle/sparse_oracle.py) against compute_scale_and_shift,
exact recovery of affine fields, robustness to gross outliers, the status rules, the configuration refusals, the
evaluate.py flag rules, and the ptxas check of csrc/sparse.cu (no kernel spills or stack frames)."""
import math
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import metrics_oracle, reference_loader
from oracle import sparse_oracle as SO


def _scene(h, w, seed, density=0.05):
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
    depth = (2.0 + 3.0 * yy + np.sin(4 * xx) + 0.2 * rng.standard_normal((h, w))).astype(np.float32)
    sparse = np.where(rng.random((h, w)) < density, depth, 0.0).astype(np.float32)
    return depth, sparse


def test_global_fit_is_compute_scale_and_shift():
    depth, sparse = _scene(48, 64, 0)
    rng = np.random.default_rng(1)
    pred = (0.3 * depth - 0.1 + 0.05 * rng.standard_normal(depth.shape)).astype(np.float32)
    nodes, rec = SO.fit(pred, sparse)
    v = SO.points(sparse, None, 1e-3, math.inf)
    p, y = torch.from_numpy(pred[v]).double(), torch.from_numpy(sparse[v]).double()
    s, t, _ = metrics_oracle.scale_shift(p, y)
    assert rec[1] == SO.STATUS_OK and rec[0] == v.sum()
    assert abs(nodes[0, 0, 0] - float(s)) <= 1e-12 * abs(float(s))
    assert abs(nodes[0, 0, 1] - float(t)) <= 1e-12 * abs(float(t))
    if reference_loader.reference_available():
        import importlib
        reference_loader._prepare_path()
        midas = importlib.import_module("losses.midas_loss")
        rs, rt = midas.compute_scale_and_shift(torch.from_numpy(pred)[None].double(),
                                               torch.from_numpy(sparse)[None].double(),
                                               torch.from_numpy(v)[None].double())
        assert abs(nodes[0, 0, 0] - float(rs[0])) <= 1e-12 * abs(float(rs[0]))
        assert abs(nodes[0, 0, 1] - float(rt[0])) <= 1e-12 * abs(float(rt[0]))


@pytest.mark.parametrize("grid", [(1, 1), (2, 3), (4, 4), (1, 7)])
@pytest.mark.parametrize("smooth", [1e-3, 0.1, 10.0])
def test_uniform_fields_are_recovered_exactly(grid, smooth):
    rng = np.random.default_rng(2)
    S, T = 2.5, -0.75
    pred = (rng.integers(64, 256, (40, 56)) / 64).astype(np.float32)      # S a + T is exact in fp32
    sparse = np.where(rng.random(pred.shape) < 0.2, pred * np.float32(S) + np.float32(T), 0).astype(np.float32)
    nodes, rec = SO.fit(pred, sparse, grid=grid, smooth=smooth)
    assert rec[1] == SO.STATUS_OK
    assert np.abs(nodes[..., 0] - S).max() <= 1e-10 * S and np.abs(nodes[..., 1] - T).max() <= 1e-10


def test_bilinear_node_fields_are_recovered_as_smoothing_vanishes():
    h, w, grid = 48, 64, (3, 4)
    rng = np.random.default_rng(3)
    true = np.stack([1.0 + 0.5 * rng.random(grid), 0.3 * rng.standard_normal(grid)], -1)
    S, T = SO.fields(true, h, w)
    pred = (1.0 + rng.random((h, w))).astype(np.float32)
    sparse = np.where(rng.random((h, w)) < 0.3, S * pred + T, 0.0)
    errs = []
    for lam in (1e-2, 1e-3, 1e-4, 1e-5):
        nodes, _ = SO.fit(pred, sparse, grid=grid, smooth=lam)
        errs.append(np.abs(nodes - true).max())
    print("node error per smooth 1e-2..1e-5:", errs)
    for e0, e1 in zip(errs, errs[1:]):
        assert 5.0 <= e0 / e1 <= 20.0                               # falls in proportion to smooth
    assert errs[-1] < 1e-4


def test_huber_irls_ignores_gross_outliers():
    h, w = 64, 80
    rng = np.random.default_rng(4)
    pred = (0.5 + rng.random((h, w))).astype(np.float32)
    s_true, t_true = 3.0, 0.4
    depth = s_true * pred.astype(np.float64) + t_true
    take = rng.random((h, w)) < 0.05
    sparse = np.where(take, depth * (1.0 + 0.01 * rng.standard_normal((h, w))), 0.0)
    ys, xs = np.nonzero(take)
    bad = rng.choice(ys.size, ys.size // 10, replace=False)
    sparse[ys[bad], xs[bad]] *= 3.0                                    # 10 % of the points scaled x3
    bound = 0.015                                   # relative error of the fitted map over the prediction's range
    robust, rec = SO.fit(pred, sparse, robust=0.02, iterations=10)
    plain, _ = SO.fit(pred, sparse)
    a = np.array([0.5, 1.5])
    err = lambda n: np.max(np.abs(n[0, 0, 0] * a + n[0, 0, 1] - (s_true * a + t_true)) / (s_true * a + t_true))
    print(f"relative error: Huber {err(robust):.2e}, least squares {err(plain):.2e}; down-weighted {rec[3]:.3f}")
    assert err(robust) <= bound and err(plain) >= 10 * bound
    assert rec[3] >= 0.09


def test_disparity_space_fits_inverse_depth():
    rng = np.random.default_rng(5)
    pred = rng.choice(np.array([0.125, 0.375, 0.875, 1.875], np.float32), (32, 40))
    disp = 2.0 * pred.astype(np.float64) + 0.25                          # 0.5, 1, 2, 4: exact depths 2 .. 0.25
    sparse = np.where(rng.random((32, 40)) < 0.2, 1.0 / disp, 0.0).astype(np.float32)
    nodes, rec = SO.fit(pred, sparse, space="disparity", max_depth=100.0)
    assert rec[1] == SO.STATUS_OK and abs(nodes[0, 0, 0] - 2.0) < 1e-12 and abs(nodes[0, 0, 1] - 0.25) < 1e-12
    out = SO.apply(pred, nodes, space="disparity", max_depth=100.0)
    assert np.allclose(out, 1.0 / disp, rtol=1e-12)


def test_status_rules_and_nan_reach():
    pred = np.full((8, 8), 0.5, np.float32)
    sparse = np.zeros((8, 8), np.float32)
    nodes, rec = SO.fit(pred, sparse)
    assert rec[1] == SO.STATUS_NO_POINTS and np.isnan(nodes).all() and np.isnan(SO.apply(pred, nodes)).all()
    sparse[2, 3] = 4.0
    assert SO.fit(pred, sparse)[1][1] == SO.STATUS_NO_POINTS
    sparse[5, 1] = 2.0
    nodes, rec = SO.fit(pred, sparse)                                    # all a equal on V
    assert rec[1] == SO.STATUS_DEGENERATE and np.isnan(nodes).all()
    pred[0, 0] = 1.0
    sparse[0, 0] = 3.0
    pred[7, 7] = np.nan                                                  # off V
    nodes, rec = SO.fit(pred, sparse)
    out = SO.apply(pred, nodes)
    assert rec[1] == SO.STATUS_OK and np.isnan(out[7, 7]) and np.isfinite(np.delete(out.ravel(), 63)).all()
    pred[2, 3] = np.inf                                                  # on V
    nodes, rec = SO.fit(pred, sparse)
    assert rec[1] == SO.STATUS_NONFINITE and np.isnan(nodes).all()


def test_metric_depth_metrics_oracle_clamps_only():
    pred = np.array([[0.5, 2.0], [50.0, np.nan]], np.float32)
    gt = np.array([[1.0, 2.0], [10.0, 0.0]], np.float32)
    rec = SO.depth_image_metric(pred, gt, max_depth=20.0)
    d = np.array([0.5, 2.0, 20.0])
    g = np.array([1.0, 2.0, 10.0])
    assert rec["n"] == 3 and abs(rec["abs_rel"] - np.mean(np.abs(d - g) / g)) < 1e-15 and rec["c1"] == 1


def test_configuration_refusals():
    from omnidata_b200.sparse import SparseDepthAligner
    SparseDepthAligner()
    SparseDepthAligner(grid=(16, 12), robust=0.1)
    for kw in ({"space": "log"}, {"space": "disparity"}, {"grid": (0, 3)}, {"grid": (33, 32)}, {"grid": 4},
               {"grid": (2, 2), "smooth": 0.0}, {"smooth": float("nan")}, {"iterations": 3},
               {"robust": 0.0}, {"robust": -1.0}, {"robust": 0.1, "iterations": 1},
               {"robust": 0.1, "iterations": 33}, {"robust": 0.1, "iterations": 2.5}, {"min_depth": -1.0},
               {"min_depth": 2.0, "max_depth": 1.0}):
        with pytest.raises(ValueError):
            SparseDepthAligner(**kw)
    from omnidata_b200.metrics import DepthMetrics
    DepthMetrics(align=False)
    with pytest.raises(ValueError):
        DepthMetrics(space="disparity", max_depth=10.0, align=False)


def test_input_refusals_before_any_launch():
    from omnidata_b200 import _capi
    from omnidata_b200.sparse import SparseDepthAligner
    al = SparseDepthAligner(grid=(4, 4))
    with pytest.raises((_capi.OdbError, ValueError)):
        al.fit(torch.zeros(1, 8, 8), torch.zeros(1, 8, 8))                # CPU tensors: no CPU path
    with pytest.raises(ValueError):
        al._check_grid("fit", 3, 8)


def test_evaluate_flag_rules():
    import evaluate
    base = ["--task", "depth", "--img_path", "i", "--gt_path", "g", "--synthetic_weights"]
    a = evaluate.parse_args(base + ["--sparse_points", "200"])
    assert a.sparse_points == 200 and a.sparse_grid == (1, 1) and a.huber is None and a.sparse_seed == 0
    a = evaluate.parse_args(base + ["--sparse_path", "s", "--sparse_grid", "4x3", "--huber", "0.1",
                                    "--huber_iterations", "7", "--sparse_smooth", "0.5"])
    assert a.sparse_grid == (4, 3) and a.huber == 0.1 and a.huber_iterations == 7 and a.sparse_smooth == 0.5
    assert evaluate.parse_args(base).sparse_points is None
    for extra in (["--sparse_points", "10", "--sparse_path", "s"], ["--sparse_grid", "2x2"], ["--huber", "0.1"],
                  ["--huber_iterations", "3"], ["--sparse_smooth", "1"], ["--sparse_seed", "3"],
                  ["--sparse_points", "0"], ["--sparse_points", "5", "--huber_iterations", "3"]):
        with pytest.raises(SystemExit):
            evaluate.parse_args(base + extra)
    with pytest.raises(SystemExit):
        evaluate.parse_args(["--task", "normal", "--img_path", "i", "--gt_path", "g", "--synthetic_weights",
                             "--sparse_points", "10"])


def test_sample_points_is_seeded_by_stem():
    import evaluate
    gt = np.full((20, 30), 2.0, np.float32)
    gt[:5] = np.nan
    a = evaluate.sample_sparse(gt, 50, 0, "img_0", 1e-3, math.inf)
    b = evaluate.sample_sparse(gt, 50, 0, "img_0", 1e-3, math.inf)
    c = evaluate.sample_sparse(gt, 50, 0, "img_1", 1e-3, math.inf)
    assert np.array_equal(a, b) and not np.array_equal(a, c)
    assert (a > 0).sum() == 50 and np.all(a[:5] == 0) and np.all(a[a > 0] == 2.0)
    assert (evaluate.sample_sparse(gt, 10 ** 6, 0, "x", 1e-3, math.inf) > 0).sum() == 15 * 30


def test_sparse_kernels_do_not_spill(tmp_path):
    """csrc/sparse.cu compiled as the build compiles it (without fast-math): no stack frame, no spills."""
    from omnidata_b200 import build
    nvcc = build._nvcc()
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "sparse.cu"), "-o",
           str(tmp_path / "sparse.o")]
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
    assert kernels >= 5, out
