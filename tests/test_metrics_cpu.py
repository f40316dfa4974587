"""Evaluation metrics without a GPU: the float64 oracle (oracle/metrics_oracle.py) on hand-built cases, the
rank-order fold of DepthMetrics / NormalMetrics.all_reduce in a world-size-2 gloo group, the refusals of the metric
configuration, the CLI's ground-truth readers, and the compiler report of csrc/metrics.cu (no kernel spills)."""
import math
import os
import re
import shutil
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from oracle import metrics_oracle as O

ROOT = Path(__file__).resolve().parents[1]


def _rand(shape, seed, lo=0.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(shape, generator=g, dtype=torch.float64) * (hi - lo) + lo


# ------------------------------------------------------------------------------------------ oracle: depth
@pytest.mark.parametrize("space", ["depth", "disparity"])
def test_perfect_prediction(space):
    g = _rand((40, 50), 0, 0.5, 10.0)
    p = g if space == "depth" else 1.0 / g
    r = O.depth_image(p, g, space=space, max_depth=20.0)
    assert r["n"] == 2000 and not r["degenerate"]
    assert r["abs_rel"] < 1e-12 and r["rmse"] < 1e-11 and r["rmse_log"] < 1e-12
    assert r["c1"] == r["c2"] == r["c3"] == 2000
    d = O.depth_dataset([r])
    assert d["delta1"] == 1.0 and d["images"] == 1 and d["pixels"] == 2000


@pytest.mark.parametrize("space", ["depth", "disparity"])
def test_affine_distortion_is_recovered(space):
    g = _rand((30, 30), 1, 1.0, 8.0)
    y = g if space == "depth" else 1.0 / g
    p = (y - 0.3) / 2.5                                      # y = 2.5 p + 0.3
    r = O.depth_image(p, g, space=space, max_depth=100.0)
    assert abs(r["s"] - 2.5) < 1e-10 and abs(r["t"] - 0.3) < 1e-10
    assert r["abs_rel"] < 1e-12 and r["c1"] == 900


def test_alignment_is_least_squares():
    g = _rand((20, 20), 2, 1.0, 5.0)
    p = _rand((20, 20), 3)
    r = O.depth_image(p, g)
    A = torch.stack([p.reshape(-1), torch.ones(400, dtype=torch.float64)], 1)
    sol = torch.linalg.lstsq(A, g.reshape(-1, 1)).solution.reshape(-1)
    assert abs(r["s"] - float(sol[0])) < 1e-10 and abs(r["t"] - float(sol[1])) < 1e-10


def test_valid_set_and_clamp():
    g = torch.tensor([[0.0, 1e-4, 2.0, float("nan")], [float("inf"), 3.0, 50.0, 4.0]], dtype=torch.float64)
    mask = torch.tensor([[1, 1, 1, 1], [1, 1, 1, 0]], dtype=torch.uint8)
    v = O.depth_valid(g.reshape(-1), mask.reshape(-1), 1e-3, 10.0)
    assert v.tolist() == [False, False, True, False, False, True, False, False]
    p = torch.tensor([[0.0, 0.0, -5.0, 0.0], [0.0, 1.0, 0.0, 0.0]], dtype=torch.float64)
    r = O.depth_image(p, g, mask, max_depth=10.0)
    assert r["n"] == 2                                        # the fit is exact on two points; nothing to clamp
    assert r["abs_rel"] < 1e-12


def test_empty_and_single_pixel_masks():
    g, p = _rand((8, 8), 4, 1.0, 3.0), _rand((8, 8), 5)
    empty = O.depth_image(p, g, torch.zeros(8, 8, dtype=torch.uint8))
    assert empty["n"] == 0 and math.isnan(empty["abs_rel"]) and not empty["degenerate"]
    one = torch.zeros(8, 8, dtype=torch.uint8)
    one[3, 4] = 1
    single = O.depth_image(p, g, one)
    assert single["n"] == 1 and single["degenerate"] and single["s"] == 0.0 and single["t"] == 0.0
    # aligned to 0, clamped to min_depth: AbsRel = |1e-3 - g| / g
    assert abs(single["abs_rel"] - abs(1e-3 - float(g[3, 4])) / float(g[3, 4])) < 1e-15
    full = O.depth_image(p, g)
    d = O.depth_dataset([empty, single, full])
    assert (d["images"], d["excluded"], d["degenerate"], d["pixels"]) == (2, 1, 1, 65)
    assert d["abs_rel"] == (single["abs_rel"] + full["abs_rel"]) / 2


def test_nonfinite_prediction_gives_nan():
    g, p = _rand((6, 6), 6, 1.0, 3.0), _rand((6, 6), 7)
    p[2, 2] = float("nan")
    r = O.depth_image(p, g)
    assert r["nonfinite"] == 1 and all(math.isnan(r[k]) for k in ("abs_rel", "sq_rel", "rmse", "rmse_log", "c1"))
    d = O.depth_dataset([O.depth_image(_rand((6, 6), 8), g), r])
    assert math.isnan(d["abs_rel"]) and d["images"] == 2


# ------------------------------------------------------------------------------------------ oracle: normals
def _encode(v):
    return (v + 1.0) / 2.0


def test_rotated_normals_give_their_angles():
    angles = torch.tensor([0.0, 5.0, 11.0, 11.5, 20.0, 25.0, 29.0, 45.0, 90.0, 179.0], dtype=torch.float64)
    rad = angles * math.pi / 180.0
    gt = torch.stack([torch.zeros(10), torch.zeros(10), torch.ones(10)]).double().reshape(1, 3, 1, 10)
    pred = torch.stack([torch.sin(rad), torch.zeros(10), torch.cos(rad)]).reshape(1, 3, 1, 10)
    th, bad = O.normal_angles(_encode(pred), _encode(gt))
    assert bad == 0 and torch.allclose(th, angles, atol=1e-10, rtol=0)
    d = O.normal_dataset([th])
    assert (d["n_11.25"], d["n_22.5"], d["n_30"]) == (3, 5, 7)
    assert d["pct_30"] == 70.0 and abs(d["mean"] - float(angles.mean())) < 1e-10
    # lower median of 10: rank 4 -> 20 degrees; its bin is floor(4096 * 20 +- rounding)
    assert d["median_bin"] in (20 * 4096 - 1, 20 * 4096) and abs(d["median"] - 20.0) <= 1.0 / 4096
    assert int(O.histogram(th).sum()) == 10


def test_degenerate_normals_are_excluded_and_nonfinite_counted():
    gt = _encode(torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)).reshape(1, 3, 1, 1).repeat(1, 1, 1, 4)
    pred = gt.clone()
    pred[0, :, 0, 1] = 0.5                                   # decodes to the zero vector: excluded
    pred[0, 0, 0, 2] = float("nan")                          # non-finite angle: counted, excluded
    mask = torch.tensor([[[1, 1, 1, 0]]], dtype=torch.uint8)
    th, bad = O.normal_angles(pred, gt, mask)
    assert th.tolist() == [0.0] and bad == 1
    d = O.normal_dataset([th], bad)
    assert d["pixels"] == 1 and d["median_bin"] == 0 and d["nonfinite"] == 1
    assert O.normal_dataset([])["median_bin"] == -1


# ------------------------------------------------------------------------------------------ configuration
def test_depth_metric_configuration_refusals():
    from omnidata_b200.metrics import DepthMetrics
    with pytest.raises(ValueError):
        DepthMetrics(space="disparity")
    with pytest.raises(ValueError):
        DepthMetrics(space="log")
    with pytest.raises(ValueError):
        DepthMetrics(min_depth=-1.0)
    with pytest.raises(ValueError):
        DepthMetrics(min_depth=5.0, max_depth=5.0)
    m = DepthMetrics(space="disparity", max_depth=80.0)
    assert m.compute()["images"] == 0 and math.isnan(m.compute()["abs_rel"])


# ------------------------------------------------------------------------------------------ all_reduce
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _depth_state(records):
    """The state depth_fold_kernel leaves after folding `records` in order."""
    sums = torch.zeros(7, dtype=torch.float64)
    counts = torch.zeros(4, dtype=torch.int64)
    for r in records:
        if r["n"] == 0:
            counts[1] += 1
            continue
        vals = [r["abs_rel"], r["sq_rel"], r["rmse"], r["rmse_log"]] + [r[f"c{k}"] / r["n"] for k in (1, 2, 3)]
        for q in range(7):
            sums[q] += vals[q]
        counts[0] += 1
        counts[2] += int(r["degenerate"])
        counts[3] += r["n"]
    return sums, counts


def _dataset():
    recs, thetas = [], []
    for i in range(6):
        g, p = _rand((16, 16), 10 + i, 1.0, 4.0), _rand((16, 16), 20 + i)
        mask = (_rand((16, 16), 30 + i) > 0.3).to(torch.uint8) if i != 2 else torch.zeros(16, 16, dtype=torch.uint8)
        recs.append(O.depth_image(p, g, mask))
        thetas.append(_rand((100 + 10 * i,), 40 + i, 0.0, 60.0))
    return recs, thetas


def _reduce_worker(rank, world, port, out):
    sys.path.insert(0, str(ROOT))
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    from omnidata_b200 import parallel
    from omnidata_b200.metrics import DepthMetrics, NormalMetrics
    parallel.init_from_env("gloo")
    recs, thetas = _dataset()
    lo, hi = parallel.shard_range(len(recs), rank, world)
    dm = DepthMetrics()
    st = dm._state_on(torch.device("cpu"))
    st["sums"][:], st["counts"][:] = _depth_state(recs[lo:hi])
    nm = NormalMetrics()
    ns = nm._state_on(torch.device("cpu"))
    th = torch.cat(thetas[lo:hi])
    ns["sums"][:] = torch.tensor([float(th.sum()), float((th * th).sum())], dtype=torch.float64)
    ns["counts"][:] = torch.tensor([th.numel(), rank, int((th < 11.25).sum()), int((th < 22.5).sum()),
                                    int((th < 30).sum())])
    ns["hist"][:] = O.histogram(th)
    dm.all_reduce()
    nm.all_reduce()
    out.put((rank, {k: v.tolist() for k, v in dm._state.items()}, {k: v.tolist() for k, v in nm._state.items()}))
    torch.distributed.destroy_process_group()


def test_world2_gloo_all_reduce_folds_in_rank_order():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_reduce_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((r, (d, n)) for r, d, n in (q.get(timeout=120) for _ in procs))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res[0] == res[1]                                  # every rank holds the same folded state
    (d, n) = res[0]
    recs, thetas = _dataset()
    sums, counts = _depth_state(recs)                        # a single-process fold of all images in order
    assert d["counts"] == counts.tolist()
    assert all(abs(a - b) <= 1e-12 * abs(b) for a, b in zip(d["sums"], sums.tolist()))
    th = torch.cat(thetas)
    assert n["counts"] == [th.numel(), 1, int((th < 11.25).sum()), int((th < 22.5).sum()), int((th < 30).sum())]
    assert n["hist"] == O.histogram(th).tolist()
    assert abs(n["sums"][0] - float(th.sum())) <= 1e-12 * float(th.sum())


# ------------------------------------------------------------------------------------------ CLI readers
def test_cli_ground_truth_readers(tmp_path):
    from PIL import Image
    sys.path.insert(0, str(ROOT))
    import evaluate
    v = np.array([[512, 1024], [65535, 256]], dtype=np.uint16)
    Image.fromarray(v).save(tmp_path / "d.png")
    d = evaluate.load_gt(tmp_path / "d.png", "depth", 512.0, 65535)
    assert d[0, 0] == 1.0 and d[0, 1] == 2.0 and np.isnan(d[1, 0]) and d[1, 1] == 0.5
    rgb = np.zeros((2, 3, 3), dtype=np.uint8)
    rgb[..., 2] = 255
    Image.fromarray(rgb).save(tmp_path / "n.png")
    n = evaluate.load_gt(tmp_path / "n.png", "normal", 512.0, 65535)
    assert n.shape == (3, 2, 3) and n[2].min() == 1.0 and n[0].max() == 0.0
    np.save(tmp_path / "n.npy", rgb.astype(np.float32) / 255.0)
    assert np.array_equal(evaluate.load_gt(tmp_path / "n.npy", "normal", 512.0, 65535), n)
    np.save(tmp_path / "m.npy", np.array([[0, 3]]))
    assert evaluate.load_mask(tmp_path / "m.npy").tolist() == [[0, 1]]


# ------------------------------------------------------------------------------------------ compiler report
def test_metric_kernels_do_not_spill(tmp_path):
    from omnidata_b200 import build
    nvcc = build._nvcc()
    if not ((os.path.isabs(nvcc) and os.path.exists(nvcc)) or shutil.which(nvcc)):
        pytest.skip("nvcc not found")
    assert "metrics.cu" in build.SOURCES and "metrics.cu" not in build.FAST_MATH_SOURCES
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / "metrics.cu"), "-o",
           str(tmp_path / "metrics.o")]
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
    names = ("depth_moments_kernel", "depth_error_kernel", "depth_fold_kernel", "slab_reduce_kernel",
             "normal_angle_kernel", "normal_fold_kernel", "normal_median_kernel")
    assert all(any(n in k for k in found) for n in names), sorted(found)
    assert all(v == (0, 0, 0) for v in found.values()), found
