"""Depth-boundary errors without a GPU: the float64 oracle (oracle/boundary_oracle.py) on hand-built edge maps and
hysteresis cases, the refusals of BoundaryMetrics, the evaluate.py flag rules, and the compiler report of
csrc/boundary.cu (no kernel spills or stack frames)."""
import math
import os
import re
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import boundary_oracle as O

ROOT = Path(__file__).resolve().parents[1]


def _lines(h, w, cols):
    e = np.zeros((h, w), dtype=np.uint8)
    e[:, cols] = 1
    return e


# ------------------------------------------------------------------------------------------ oracle: scoring
@pytest.mark.parametrize("k", [1, 2, 5, 9, 10, 14])
def test_vertical_lines_k_apart(k):
    gt = _lines(30, 40, [10])
    pred = _lines(30, 40, [10 + k])
    r = O.score(pred, gt, max_dist=10.0)
    if k < 10:
        assert r["acc"] == float(k) and r["comp"] == float(k) and not r["no_pred"] and r["n_a"] == 30
    else:
        assert r["acc"] == 10.0 and r["comp"] == 10.0 and r["no_pred"] and r["n_a"] == 0
    assert r["n_gt"] == r["n_pred"] == 30 and not r["no_gt"]


def test_perfect_edges_score_zero():
    e = _lines(20, 20, [3, 11])
    e[5, :] = 1
    r = O.score(e, e)
    assert r["acc"] == 0.0 and r["comp"] == 0.0


def test_no_ground_truth_edges_excludes_the_image():
    empty = np.zeros((16, 16), dtype=np.uint8)
    r = O.score(_lines(16, 16, [4]), empty)
    assert r["no_gt"] and math.isnan(r["acc"]) and math.isnan(r["comp"])
    other = O.score(_lines(16, 16, [6]), _lines(16, 16, [4]))
    d = O.boundary_dataset([r, other])
    assert d["images"] == 2 and d["no_gt_edges"] == 1 and d["dbe_acc"] == 2.0 and d["dbe_comp"] == 2.0


def test_distances_are_exact_squares():
    e = np.zeros((7, 9), dtype=np.uint8)
    e[2, 3] = 1
    d2 = O.distance2(e)
    yy, xx = np.indices(e.shape)
    assert np.array_equal(d2, (yy - 2) ** 2 + (xx - 3) ** 2)
    assert (O.distance2(np.zeros((3, 4))) == O.NO_EDGE).all()
    assert (O.distance2(np.ones((3, 4))) == 0).all()


# ------------------------------------------------------------------------------------------ oracle: hysteresis
def test_weak_chain_touching_strong_is_kept():
    weak = np.zeros((8, 12), dtype=bool)
    strong = np.zeros_like(weak)
    weak[2, 1:6] = True                          # a horizontal chain
    weak[3, 6] = weak[4, 7] = True               # continued diagonally only
    strong[5, 8] = True                          # touching the chain's end only diagonally
    out = O.hysteresis(weak, strong)
    assert out[2, 1:6].all() and out[3, 6] and out[4, 7] and out[5, 8]
    assert out.sum() == 8


def test_weak_chain_without_strong_is_dropped():
    weak = np.zeros((8, 12), dtype=bool)
    strong = np.zeros_like(weak)
    weak[1, 1:5] = True
    weak[6, 2:10] = True
    strong[6, 9] = True
    out = O.hysteresis(weak, strong)
    assert not out[1].any() and out[6, 2:10].all() and out.sum() == 8


def test_detector_finds_a_step_and_is_scale_invariant():
    g = np.full((32, 40), 2.0, dtype=np.float32)
    g[:, 20:] = 6.0
    v = O.valid_set(g)
    e = O.edges(g, v)
    cols = np.nonzero(e.any(0))[0]
    assert e.sum() > 0 and set(cols) <= {19, 20}
    assert np.array_equal(O.edges(g * 8.0, v), e)
    assert O.edges(np.full_like(g, 3.0), v).sum() == 0                  # a flat map has no edges
    bad = g.copy()
    bad[4, 4] = np.nan
    assert O.edges(bad, v).sum() == 0                                   # nor one not finite on V


# ------------------------------------------------------------------------------------------ configuration
def test_boundary_metric_configuration_refusals():
    from omnidata_b200.metrics import BoundaryMetrics
    for kw in ({"sigma": 0.0}, {"sigma": 4.5}, {"sigma": math.nan}, {"low": math.nan}, {"high": math.inf},
               {"low": -0.1}, {"low": 0.3, "high": 0.2}, {"max_dist": 0.0}, {"max_dist": math.inf},
               {"min_depth": -1.0}, {"min_depth": 5.0, "max_depth": 5.0}):
        with pytest.raises(ValueError):
            BoundaryMetrics(**kw)
    m = BoundaryMetrics(sigma=4.0, low=0.0, high=0.0)
    out = m.compute()
    assert out["images"] == 0 and math.isnan(out["dbe_acc"]) and math.isnan(out["dbe_comp"])


def test_cli_boundary_flag_rules(tmp_path):
    sys.path.insert(0, str(ROOT))
    import evaluate
    base = ["--img_path", str(tmp_path), "--gt_path", str(tmp_path), "--synthetic_weights"]
    with pytest.raises(SystemExit):
        evaluate.parse_args(["--task", "normal", "--boundary"] + base)
    with pytest.raises(SystemExit):
        evaluate.parse_args(["--task", "depth", "--edge_path", str(tmp_path)] + base)
    a = evaluate.parse_args(["--task", "depth", "--boundary", "--edge_path", str(tmp_path), "--mode", "guided",
                             "--guided_size", "384x384", "--flip"] + base)
    assert a.boundary and a.edge_path == str(tmp_path)
    assert not evaluate.parse_args(["--task", "depth"] + base).boundary
    np.save(tmp_path / "e.npy", np.array([[0, 2], [1, 0]]))
    assert evaluate.load_edges(tmp_path / "e.npy").tolist() == [[0, 1], [1, 0]]


# ------------------------------------------------------------------------------------------ compiler report
def test_boundary_kernels_do_not_spill(tmp_path):
    from omnidata_b200 import build
    nvcc = build._nvcc()
    if not ((os.path.isabs(nvcc) and os.path.exists(nvcc)) or shutil.which(nvcc)):
        pytest.skip("nvcc not found")
    assert "boundary.cu" in build.SOURCES and "boundary.cu" not in build.FAST_MATH_SOURCES
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "boundary.cu"), "-o",
           str(tmp_path / "boundary.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    found, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            found[cur] = tuple(int(x) for x in m.groups())
            cur = None
    names = ("edge_stats_kernel", "smooth_h_kernel", "smooth_v_kernel", "sobel_nms_kernel", "hysteresis_init_kernel",
             "ccl_merge_kernel", "ccl_resolve_kernel", "edge_select_kernel", "edt_col_kernel", "edt_row_kernel",
             "chamfer_kernel", "boundary_fold_kernel")
    assert all(any(n in k for k in found) for n in names), sorted(found)
    assert all(v == (0, 0, 0) for v in found.values()), found
