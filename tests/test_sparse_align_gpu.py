"""Sparse metric alignment on the GPU (SparseDepthAligner, csrc/sparse.cu).

- Kernels on guarded buffers (oracle/guard.py checked_launch: every output written, nothing else touched, a second run
  bit-identical) against the float64 oracle (oracle/sparse_oracle.py): nodes within 1e-9 relative, the output within
  1 fp32 ulp of the oracle's value rounded once; grids 1x1 to 32x32 and 1x1024, sizes 2x2 to 3024x4032 and widths not
  divisible by 4, 1 and 2 points to dense maps, every mask kind, depth and disparity, robust on and off.
- Status rules and NaN reach; batch independence and repeat runs; CUDA-graph replay; no synchronisation and no
  allocation beyond the output after the first call at a shape.
- End to end with synthetic weights (hybrid, bf16): the aligner on GuidedPredictor and TiledPredictor output against the
  oracle applied to that same prediction; DepthMetrics(align=False) against its oracle; evaluate.py --sparse_points."""
import json
import math

import numpy as np
import pytest
import torch

from oracle import sparse_oracle as SO
from oracle.guard import Guarded, checked_launch

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _scene(b, h, w, seed, density, offset=0.2):
    """pred (a relative prediction), sparse (metres, 0 = none): depth varies over the image and the map from pred to
    depth drifts slowly across it, with 1 % noise on the points."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
    pred = (offset + rng.random((b, h, w)) * 0.5 + 0.5 * yy + 0.3 * xx).astype(np.float32)
    depth = (2.0 + 0.5 * xx) * pred + 0.3 + 0.2 * yy
    depth *= 1.0 + 0.01 * rng.standard_normal((b, h, w))
    if isinstance(density, int):                                      # exactly this many points per image
        take = np.zeros((b, h * w), bool)
        for i in range(b):
            take[i, rng.choice(h * w, density, replace=False)] = True
        take = take.reshape(b, h, w)
    else:
        take = rng.random((b, h, w)) < density
    return pred, np.where(take, depth, 0.0).astype(np.float32)


def _mask(kind, b, h, w, seed):
    if kind is None:
        return None
    m = np.random.default_rng(seed).random((b, h, w)) < 0.8
    return torch.from_numpy(m.astype(np.float32) if kind == "f32" else m if kind == "bool" else m.astype(np.uint8))


def _guarded(arr, gen, dtype=torch.float32):
    g = Guarded(arr.numel(), dtype, gen)
    v = g.contiguous(*arr.shape)
    v.copy_(arr.to(dev))
    return g, v


def _check_against_oracle(pred, sparse, mask, grid, space, robust, max_depth, nodes, rec, out):
    kw = dict(grid=grid, space=space, smooth=0.1, robust=robust, min_depth=1e-3, max_depth=max_depth)
    worst_node = worst_ulp = 0.0
    for i in range(pred.shape[0]):
        m = None if mask is None else mask[i].numpy()
        want, wrec = SO.fit(pred[i], sparse[i], m, **kw)
        assert rec[i, 1] == wrec[1] and rec[i, 0] == wrec[0], (i, rec[i], wrec)
        got = nodes[i].cpu().numpy()
        scale = np.abs(want).max()
        worst_node = max(worst_node, float(np.abs(got - want).max() / scale))
        # the residual RMS to 1e-6 relative, or to rounding where the fit is exact (two points)
        assert abs(rec[i, 2] - wrec[2]) <= 1e-6 * wrec[2] + 1e-12 and abs(rec[i, 3] - wrec[3]) <= 0.01
        d = SO.apply(pred[i], want, space=space, min_depth=1e-3, max_depth=max_depth).astype(np.float32)
        o = out[i].cpu().numpy()
        ulp = np.spacing(np.abs(d))
        worst_ulp = max(worst_ulp, float(np.max(np.abs(o.astype(np.float64) - d) / ulp)))
    print(f"grid {grid} {space} robust {robust}: nodes {worst_node:.1e} relative, output {worst_ulp:.0f} ulp")
    assert worst_node <= 1e-9 and worst_ulp <= 1.0


CASES = [  # (b, h, w, grid, density, mask, space, robust)
    (2, 2, 2, (1, 1), 1.0, None, "depth", None),
    (3, 37, 51, (2, 3), 0.05, "u8", "depth", None),
    (2, 96, 128, (8, 6), 0.05, "bool", "disparity", 0.05),
    (2, 384, 384, (32, 32), 1.0, "f32", "depth", 0.05),
    (1, 40, 1030, (1, 1024), 1.0, None, "depth", None),
    (2, 384, 384, (1, 1), 2, None, "depth", None),
    (2, 384, 384, (16, 12), 0.001, "u8", "depth", 0.05),
    (1, 3024, 4032, (1, 1), 200, None, "depth", None),
    (1, 3024, 4032, (16, 12), 0.05, None, "disparity", 0.05),
    (1, 3024, 4032, (1, 1), 1.0, None, "depth", 0.05),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}x{c[1]}x{c[2]}-g{c[3][0]}x{c[3][1]}-{c[4]}-{c[5]}-"
                                                     f"{c[6]}-{c[7]}")
def test_fit_and_apply_match_the_oracle(case):
    from omnidata_b200 import _capi, ops
    b, h, w, grid, density, mkind, space, robust = case
    pred, sparse = _scene(b, h, w, sum(grid) + h + w, density)
    mask = _mask(mkind, b, h, w, 3)
    max_depth = 50.0 if space == "disparity" else math.inf
    gen = torch.Generator(device=dev).manual_seed(1)
    gp, p = _guarded(torch.from_numpy(pred), gen)
    gs, s = _guarded(torch.from_numpy(sparse), gen)
    bufs = [gp, gs]
    m = None if mask is None else mask.to(dev)
    ws = torch.empty(-(-ops.sparse_align_workspace_bytes(b, h, w, grid) // 8), dtype=torch.float64, device=dev)
    gn = Guarded(b * grid[0] * grid[1] * 2 + b * _capi.SPARSE_RECORD, torch.float64, gen)
    nodes = gn.view((b, *grid, 2), (grid[0] * grid[1] * 2, grid[1] * 2, 2, 1))
    rec = gn.view((b, _capi.SPARSE_RECORD), (_capi.SPARSE_RECORD, 1), b * grid[0] * grid[1] * 2)
    go = Guarded(b * h * w, torch.float32, gen)
    out = go.contiguous(b, h, w)
    sp = _capi.SPACE_DISPARITY if space == "disparity" else _capi.SPACE_DEPTH
    rb, it = (0.0, 1) if robust is None else (robust, 5)

    def launch():
        ops.sparse_align_fit(p, s, m, grid, sp, 1e-3, max_depth, 0.1, rb, it, ws, nodes, rec)
        ops.sparse_align_apply(p, nodes, out, sp, 1e-3, max_depth)
    nodes_c, rec_c, out_c = checked_launch(bufs + [gn, go], [nodes, rec, out], launch)
    _check_against_oracle(pred, sparse, mask, grid, space, robust, max_depth, nodes_c, rec_c.cpu().numpy(), out_c)


def test_status_rules_and_nan_reach():
    from omnidata_b200.sparse import STATUS, SparseDepthAligner
    pred, sparse = _scene(5, 33, 47, 9, 0.1)
    sparse[0] = 0.0                                                    # no points
    sparse[1] = 0.0
    sparse[1, 4, 5] = 3.0                                              # one point
    pred[2] = 0.5                                                      # all a equal on V
    ys, xs = np.nonzero(sparse[3])
    pred[3, ys[0], xs[0]] = np.nan                                     # NaN on V
    ys, xs = np.nonzero(sparse[4] == 0)
    pred[4, ys[0], xs[0]] = np.nan                                     # NaN off V
    for grid in ((1, 1), (3, 4)):
        al = SparseDepthAligner(grid=grid)
        p, s = torch.from_numpy(pred).to(dev), torch.from_numpy(sparse).to(dev)
        nodes, rec = al.fit(p, s)
        out = al.apply(p, nodes).cpu()
        rec = rec.cpu()
        assert [STATUS[int(v)] for v in rec[:, 1]] == ["no_points", "no_points", "degenerate", "nonfinite", "ok"]
        assert torch.isnan(out[:4]).all() and torch.isnan(rec[:4, 2]).all()
        bad = torch.isnan(out[4])
        assert int(bad.sum()) == 1 and bool(bad[ys[0], xs[0]])


def test_batch_split_and_repeat_runs_give_the_same_bits():
    from omnidata_b200.sparse import SparseDepthAligner
    pred, sparse = _scene(17, 120, 164, 11, 0.05)
    p, s = torch.from_numpy(pred).to(dev), torch.from_numpy(sparse).to(dev)
    al = SparseDepthAligner(grid=(4, 6), robust=0.05)
    nodes, rec = (t.clone() for t in al.fit(p, s))
    out = al.apply(p, nodes)
    for parts in ([1] * 17, [5, 12]):
        o, got = 0, []
        for k in parts:
            n, _ = al.fit(p[o:o + k], s[o:o + k])
            got.append(al.apply(p[o:o + k], n))
            assert torch.equal(n, nodes[o:o + k])
            o += k
        assert torch.equal(torch.cat(got), out)
    n2, r2 = al.fit(p, s)
    assert torch.equal(n2, nodes) and torch.equal(r2, rec) and torch.equal(al.apply(p, n2), out)


def test_graph_replay_no_sync_no_alloc():
    from omnidata_b200.sparse import SparseDepthAligner
    pred, sparse = _scene(3, 200, 300, 12, 0.05)
    p, s = torch.from_numpy(pred).to(dev), torch.from_numpy(sparse).to(dev)
    al = SparseDepthAligner(grid=(8, 12), robust=0.05)
    want = al(p, s)
    torch.cuda.synchronize()
    n0 = torch.cuda.memory_stats()["allocation.all.allocated"]
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = al(p, s)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.cuda.memory_stats()["allocation.all.allocated"] - n0 == 1    # the output
    assert torch.equal(out, want)
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        al(p, s)
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(graph):
        static = al(p, s)
    static.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, want)


def _model():
    from omnidata_b200.model import DPTDepthModel
    from oracle import weights
    m = DPTDepthModel(backbone="vitb_rn50_384", num_channels=1, non_negative=False)
    m.load_state_dict(weights.make_state_dict(0, 1), strict=True)
    return m.to(dev).eval()


@pytest.mark.parametrize("which", ["guided", "tiled"])
def test_on_predictor_output(which):
    from omnidata_b200.guided import GuidedPredictor
    from omnidata_b200.sparse import SparseDepthAligner
    from omnidata_b200.tiled import TiledPredictor
    model = _model()
    g = torch.Generator().manual_seed(13)
    x = (torch.rand(1, 3, 600, 900, generator=g) * 2 - 1).to(dev)
    with torch.no_grad():
        pred = GuidedPredictor(model, size=(384, 512))(x) if which == "guided" else \
            TiledPredictor(model, tile=(384, 384), overlap=64)(x)
    pred = pred.float().contiguous()
    rng = np.random.default_rng(14)
    pc = pred.cpu().numpy()
    sparse = np.where(rng.random(pc.shape) < 0.02, 3.0 * (pc - pc.min()) + 1.0, 0.0).astype(np.float32)
    for grid, robust in (((1, 1), None), ((6, 8), 0.05)):
        al = SparseDepthAligner(grid=grid, robust=robust)
        nodes, rec = al.fit(pred, torch.from_numpy(sparse).to(dev))
        out = al.apply(pred, nodes)
        _check_against_oracle(pc, sparse, None, grid, "depth", robust, math.inf, nodes, rec.cpu().numpy(), out)


def test_metric_depth_metrics_match_the_oracle():
    from omnidata_b200.metrics import DepthMetrics
    rng = np.random.default_rng(15)
    gt = (1.0 + 9.0 * rng.random((3, 50, 70))).astype(np.float32)
    gt[0, :5] = np.nan
    pred = (gt * (1.0 + 0.1 * rng.standard_normal(gt.shape))).astype(np.float32)
    pred[1, 3, 3] = 30.0
    mask = torch.from_numpy(rng.random(gt.shape) < 0.9)
    met = DepthMetrics(max_depth=20.0, align=False)
    rec = met.update(torch.from_numpy(pred).to(dev), torch.from_numpy(gt).to(dev), mask.to(dev)).cpu().numpy()
    for i in range(3):
        want = SO.depth_image_metric(pred[i], gt[i], mask[i].numpy(), max_depth=20.0)
        assert rec[i, 0] == want["n"] and rec[i, 8] == 1.0 and rec[i, 9] == 0.0 and rec[i, 10] == 0.0
        for q, k in enumerate(("abs_rel", "sq_rel", "rmse", "rmse_log")):
            assert abs(rec[i, 1 + q] - want[k]) <= 1e-10 * abs(want[k]), (k, rec[i, 1 + q], want[k])
        for q in range(3):
            assert rec[i, 5 + q] == want[f"c{q + 1}"]


def test_cli_sparse_points(tmp_path, capsys):
    import evaluate
    from PIL import Image
    img, gtd = tmp_path / "img", tmp_path / "gt"
    img.mkdir()
    gtd.mkdir()
    rng = np.random.default_rng(16)
    for i in range(2):
        g = (1.0 + 5.0 * rng.random((384, 384))).astype(np.float32)
        Image.fromarray((g / 6.0 * 255).astype(np.uint8)).convert("RGB").save(img / f"im{i}.png")
        np.save(gtd / f"im{i}.npy", g)
    base = ["--task", "depth", "--img_path", str(img), "--gt_path", str(gtd), "--synthetic_weights", "--mode",
            "direct", "--max_depth", "10"]
    plain = evaluate.main(base)
    capsys.readouterr()
    assert "sparse" not in plain
    ret = evaluate.main(base + ["--sparse_points", "200"])
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert set(ret) - set(plain) == {"sparse"} and json.dumps(printed["sparse"]) == json.dumps(ret["sparse"])
    assert json.dumps(ret["metrics"]) == json.dumps(plain["metrics"])
    sp = ret["sparse"]
    assert sp["records"]["ok"] + sp["records"]["degenerate"] == 2 and sp["records"]["mean_points"] == 200.0
    assert sp["metrics"]["images"] == 2 and sp["grid"] == [1, 1]
