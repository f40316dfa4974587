"""Depth-boundary errors on the GPU (omnidata_b200/metrics.py BoundaryMetrics, csrc/boundary.cu) against the float64
oracle (oracle/boundary_oracle.py):

- seeded piecewise-planar scenes with noise at 2x2 ... 3024x4032, every mask kind: edge maps bit for bit, record counts
  equal and accuracy / completeness to 1e-12 relative, with ground-truth edges detected and given;
- squared distance transforms equal scipy's exactly (empty, single-pixel, all-edge, sparse and dense maps, w = 65535);
  hysteresis equals scipy.ndimage.label on a spiral covering the image and on random masks at densities 0.3-0.6;
  the outputs are written exactly and nothing around them is touched (guard bands);
- exact cases (pred = gt, pred x 2^k, a NaN on V), batch splits and repeats bit-identical, a captured update replays to
  the eager bits and allocates nothing, refusals before any launch, and evaluate.py --boundary against the API."""
import json
import math

import numpy as np
import pytest
import torch

from oracle import boundary_oracle as O

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
GUARD = 64 * 1024


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def scene(b, h, w, seed, regions=12):
    """[b,h,w] fp32 depth: Voronoi regions, each a plane, with bars 1-3 px wide in front and 1 % noise."""
    g = _gen(seed)
    yy = torch.arange(h, device=dev, dtype=torch.float32).view(1, h, 1) / max(h, w)
    xx = torch.arange(w, device=dev, dtype=torch.float32).view(1, 1, w) / max(h, w)
    out = torch.empty(b, h, w, device=dev)
    for i in range(b):
        seeds = torch.rand(regions, 2, generator=g, device=dev) * torch.tensor([h, w], device=dev) / max(h, w)
        d = (yy - seeds[:, 0].view(-1, 1, 1)) ** 2 + (xx - seeds[:, 1].view(-1, 1, 1)) ** 2
        lab = d.argmin(0)
        coef = torch.rand(regions, 3, generator=g, device=dev) * torch.tensor([4.0, 2.0, 2.0], device=dev) + \
            torch.tensor([1.0, -1.0, -1.0], device=dev)
        z = coef[lab, 0] + coef[lab, 1] * yy[0] + coef[lab, 2] * xx[0]
        for k in range(3):
            wd = k + 1
            x0 = int(torch.randint(0, max(w - wd, 1), (1,), generator=g, device=dev))
            y0 = int(torch.randint(0, max(h - wd, 1), (1,), generator=g, device=dev))
            z[:, x0:x0 + wd] = 0.8
            z[y0:y0 + wd, :] = 0.9
        out[i] = z
    noise = 1.0 + 0.01 * torch.randn(b, h, w, generator=g, device=dev)
    return (out * noise).clamp_min(0.05).contiguous()


def prediction(gt, seed):
    """A distorted prediction: affine, shifted by one column, smoothed rows, noisier."""
    p = 0.5 * gt.roll(1, dims=2) + 0.3
    p = (p + p.roll(1, dims=1)) / 2
    return (p + 0.02 * torch.randn(gt.shape, generator=_gen(seed), device=dev)).contiguous()


def _mask(kind, b, h, w, seed):
    if kind == "none":
        return None
    m = torch.rand(b, h, w, generator=_gen(seed), device=dev) > 0.02
    m[:, h // 3:h // 3 + max(h // 8, 1), w // 4:w // 4 + max(w // 6, 1)] = False          # a hole
    return {"uint8": m.to(torch.uint8), "bool": m, "fp32": m.float()}[kind]


def _close(a, b, rel=1e-12):
    if math.isnan(b):
        return math.isnan(a)
    return abs(a - b) <= rel * abs(b) + 1e-300


def _check_records(rec, want):
    for i, r in enumerate(want):
        row = O.record_row(r)
        got = rec[i].tolist()
        assert got[2:] == row[2:], (i, got, row)
        for q in range(2):
            assert _close(got[q], row[q]), (i, q, got[q], row[q])


def _check_dataset(got, want):
    for k, v in want.items():
        assert (got[k] == v) if isinstance(v, int) else _close(got[k], v), (k, got[k], v)


def _np(t):
    return None if t is None else t.cpu().numpy()


SIZES = [(2, 2), (3, 3), (97, 131), (384, 384), (1080, 1920), (3024, 4032)]
MASKS = ["none", "uint8", "bool", "fp32"]


@pytest.mark.parametrize("mask_kind", MASKS)
@pytest.mark.parametrize("h,w", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_edges_and_records_match_oracle(h, w, mask_kind):
    from omnidata_b200.metrics import BoundaryMetrics
    b = 1 if h * w > 1e6 else 2
    g = scene(b, h, w, h + 7 * w)
    p = prediction(g, h * w)
    m = _mask(mask_kind, b, h, w, h + w)
    bm = BoundaryMetrics()
    e = bm.edges(g, m).cpu().numpy()
    mi = [None if m is None else _np(m[i]) for i in range(b)]
    for i in range(b):
        want = O.edges(_np(g[i]), O.valid_set(_np(g[i]), mi[i]))
        assert np.array_equal(e[i], want), (i, int((e[i] != want).sum()))
    if h * w >= 384 * 384:
        assert e.sum() > 0
    rec = bm.update(p, g, m).cpu()
    want = [O.boundary_image(_np(p[i]), _np(g[i]), mi[i]) for i in range(b)]
    _check_records(rec, want)
    _check_dataset(bm.compute(), O.boundary_dataset(want))
    given = torch.rand(b, 1, h, w, generator=_gen(5), device=dev) < 0.01           # [B,1,H,W] bool edge maps
    bg = BoundaryMetrics(max_dist=4.0)
    rec = bg.update(p.unsqueeze(1), g, m, gt_edges=given).cpu()
    want = [O.boundary_image(_np(p[i]), _np(g[i]), mi[i], _np(given[i]), max_dist=4.0) for i in range(b)]
    _check_records(rec, want)
    _check_dataset(bg.compute(), O.boundary_dataset(want))


# ------------------------------------------------------------------------------------------ stages on guarded buffers
def _guarded(shape, dtype, seed):
    """(full buffer with GUARD bytes of random bands on both sides, the [shape] view between them)."""
    n = int(np.prod(shape))
    es = torch.tensor([], dtype=dtype).element_size()
    pad = GUARD // es
    full = torch.randint(0, 120, (n + 2 * pad,), generator=_gen(seed), device=dev).to(dtype)
    return full, full[pad:pad + n].view(shape)


def _bands_intact(full, before, n):
    pad = (full.numel() - n) // 2
    assert torch.equal(full[:pad], before[:pad]) and torch.equal(full[pad + n:], before[pad + n:])


def _run_guarded(launch, shape, out_dtype):
    from omnidata_b200 import ops
    b, h, w = shape
    nws = -(-ops.boundary_workspace_bytes(b, h, w) // 8)
    wfull, ws = _guarded((nws,), torch.float64, 1)
    ofull, out = _guarded(shape, out_dtype, 2)
    wb, ob = wfull.clone(), ofull.clone()
    launch(ws, out)
    torch.cuda.synchronize()
    _bands_intact(wfull, wb, nws)
    _bands_intact(ofull, ob, b * h * w)
    first = out.clone()
    launch(ws, out)
    assert torch.equal(out, first)
    return first


def _dist2(edges):
    from omnidata_b200 import ops
    return _run_guarded(lambda ws, out: ops.edge_distance2(edges, ws, out), tuple(edges.shape),
                        torch.int64).cpu().numpy()


@pytest.mark.parametrize("h,w", [(1, 1), (2, 2), (3, 3), (97, 131), (384, 384), (2, 65535), (1080, 1920)])
def test_distance_transform_is_exact(h, w):
    cases = [np.zeros((h, w), np.uint8), np.ones((h, w), np.uint8)]
    one = np.zeros((h, w), np.uint8)
    one[h // 2, w // 3] = 1
    cases.append(one)
    corner = np.zeros((h, w), np.uint8)
    corner[h - 1, w - 1] = 1
    cases.append(corner)
    rng = np.random.default_rng(h * w)
    for dens in (1e-4, 0.01, 0.3):
        cases.append((rng.random((h, w)) < dens).astype(np.uint8))
    e = torch.from_numpy(np.stack(cases)).to(dev)
    got = _dist2(e)
    for i, c in enumerate(cases):
        assert np.array_equal(got[i], O.distance2(c)), i
    assert (got[0] == O.NO_EDGE).all() and (got[1] == 0).all()
    bools = _dist2(e[2:4].bool())
    assert np.array_equal(bools, got[2:4])


def _spiral(h, w):
    """A one-pixel-wide spiral with one-pixel gaps, covering the image: one component of about h w / 2 pixels."""
    a = np.zeros((h, w), np.uint8)
    y, x, dy, dx = 0, 0, 0, 1
    a[0, 0] = 1
    while True:
        for _ in range(2):                                          # straight on, else turn clockwise
            ny, nx, fy, fx = y + dy, x + dx, y + 2 * dy, x + 2 * dx
            if 0 <= ny < h and 0 <= nx < w and not a[ny, nx] and not (0 <= fy < h and 0 <= fx < w and a[fy, fx]):
                y, x = ny, nx
                a[y, x] = 1
                break
            dy, dx = dx, -dy
        else:
            return a


def _hysteresis(ws_in):
    from omnidata_b200 import ops
    return _run_guarded(lambda ws, out: ops.edge_hysteresis(ws_in, ws, out), tuple(ws_in.shape),
                        torch.uint8).cpu().numpy()


@pytest.mark.parametrize("h,w", [(257, 263), (1024, 1024)])
def test_hysteresis_on_a_spiral(h, w):
    from scipy import ndimage
    sp = _spiral(h, w)
    lab, n = ndimage.label(sp, structure=np.ones((3, 3), int))
    weak = sp.astype(bool)
    strong = np.zeros_like(weak)
    ys, xs = np.nonzero(sp)
    assert n == 1 and sp.sum() > h * w // 3
    strong[ys[-1], xs[-1]] = True                                   # one strong pixel
    flags = torch.from_numpy((weak | strong).astype(np.uint8) | (strong.astype(np.uint8) << 1)).to(dev)
    got = _hysteresis(flags[None])[0]
    want = O.hysteresis(weak, strong)
    assert np.array_equal(got, want)
    assert got.sum() == (lab == lab[ys[-1], xs[-1]]).sum()


@pytest.mark.parametrize("density", [0.3, 0.4, 0.45, 0.5, 0.6])
def test_hysteresis_on_random_masks(density):
    rng = np.random.default_rng(int(density * 100))
    b, h, w = 3, 512, 700
    weak = rng.random((b, h, w)) < density
    strong = weak & (rng.random((b, h, w)) < 0.002)
    flags = torch.from_numpy(weak.astype(np.uint8) | (strong.astype(np.uint8) << 1)).to(dev)
    got = _hysteresis(flags)
    for i in range(b):
        assert np.array_equal(got[i], O.hysteresis(weak[i], strong[i])), i


def test_depth_edges_on_guarded_buffers():
    from omnidata_b200 import ops
    g = scene(2, 97, 131, 3)
    m = _mask("uint8", 2, 97, 131, 4)
    got = _run_guarded(lambda ws, out: ops.depth_edges(g, m, math.sqrt(2.0), 0.1, 0.2, 1e-3, math.inf, ws, out),
                       (2, 97, 131), torch.uint8).cpu().numpy()
    for i in range(2):
        assert np.array_equal(got[i], O.edges(_np(g[i]), O.valid_set(_np(g[i]), _np(m[i]))))


# ------------------------------------------------------------------------------------------ exact cases
def test_exact_cases():
    from omnidata_b200.metrics import BoundaryMetrics
    g = scene(3, 200, 260, 9)
    bm = BoundaryMetrics()
    rec = bm.update(g, g).cpu()
    assert (rec[:, 0] == 0).all() and (rec[:, 1] == 0).all() and (rec[:, 2] > 0).all()
    assert bm.compute()["dbe_acc"] == 0.0 and bm.compute()["dbe_comp"] == 0.0
    p = prediction(g, 10)
    ref = BoundaryMetrics().update(p, g).cpu()
    for k in (-3, 1, 5):
        assert torch.equal(BoundaryMetrics().update(p * 2.0 ** k, g).cpu(), ref), k
    bad = p.clone()
    bad[1, 100, 100] = float("nan")
    bn = BoundaryMetrics()
    rec = bn.update(bad, g).cpu()
    assert math.isnan(rec[1, 0]) and math.isnan(rec[1, 1]) and rec[1, 5] == 1.0
    assert not math.isnan(rec[0, 0]) and not math.isnan(rec[2, 1])
    out = bn.compute()
    assert math.isnan(out["dbe_acc"]) and math.isnan(out["dbe_comp"]) and out["images"] == 3
    flat = BoundaryMetrics()
    rec = flat.update(g, torch.full_like(g, 2.0)).cpu()
    assert (rec[:, 6] == 1).all() and flat.compute()["no_gt_edges"] == 3 and math.isnan(flat.compute()["dbe_acc"])


# ------------------------------------------------------------------------------------------ determinism
def _split(splits, p, g, m):
    from omnidata_b200.metrics import BoundaryMetrics
    bm = BoundaryMetrics()
    i = 0
    for n in splits:
        bm.update(p[i:i + n], g[i:i + n], m[i:i + n])
        i += n
    return bm


def test_batch_split_and_repeat_are_bit_identical():
    g = scene(17, 120, 150, 11)
    p = prediction(g, 12)
    m = _mask("uint8", 17, 120, 150, 13)
    ref = _split([17], p, g, m)
    assert ref.compute()["images"] == 17 and ref.compute()["no_gt_edges"] < 17
    for s in ([1] * 17, [5, 12], [17]):
        other = _split(s, p, g, m)
        for k in ref._state:
            assert torch.equal(other._state[k], ref._state[k]), (s, k)
        assert json.dumps(other.compute()) == json.dumps(ref.compute())


def test_cuda_graph_replay_equals_eager_and_allocates_nothing():
    from omnidata_b200.metrics import BoundaryMetrics
    g = scene(4, 96, 128, 21)
    p = prediction(g, 22)
    m = _mask("fp32", 4, 96, 128, 23)
    for edges in (None, torch.rand(4, 96, 128, generator=_gen(24), device=dev) < 0.02):
        eager = BoundaryMetrics()
        eager.update(p, g, m, edges)
        eager.update(p, g, m, edges)
        cap = BoundaryMetrics()
        cap.update(p, g, m, edges)
        bufs = {k: v.data_ptr() for k, v in cap._bufs.items()}
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        cap.update(p, g, m, edges)
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() == before
        assert {k: v.data_ptr() for k, v in cap._bufs.items()} == bufs
        cap.reset()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(graph, stream=s):
                cap.update(p, g, m, edges)
        torch.cuda.current_stream().wait_stream(s)
        graph.replay()
        graph.replay()
        torch.cuda.synchronize()
        for k in eager._state:
            assert torch.equal(cap._state[k], eager._state[k]), k
        assert json.dumps(cap.compute()) == json.dumps(eager.compute())


def test_refusals_before_any_launch():
    from omnidata_b200 import _capi
    from omnidata_b200.metrics import BoundaryMetrics
    g = scene(2, 32, 48, 31)
    p = prediction(g, 32)
    n0 = _capi.launch_count()
    bm = BoundaryMetrics()
    e = torch.zeros(2, 32, 48, dtype=torch.uint8, device=dev)
    bad = [(p.cpu(), g.cpu(), None, None), (p.double(), g, None, None), (p, g[:, :31], None, None),
           (p, g, torch.ones(2, 32, 48, dtype=torch.int32, device=dev), None), (p[:0], g[:0], None, None),
           (p, g, None, e.float()), (p, g, None, e[:, :31]), (p, g, None, e.cpu()),
           (p, g, None, e.transpose(1, 2).contiguous().transpose(1, 2)),
           (torch.zeros(1, 65536, 1, device=dev), torch.zeros(1, 65536, 1, device=dev), None, None),
           (torch.zeros(1, 1, 65536, device=dev), torch.zeros(1, 1, 65536, device=dev), None, None)]
    for a, b_, m, ed in bad:
        with pytest.raises((ValueError, _capi.OdbError)):
            bm.update(a, b_, m, ed)
    with pytest.raises((ValueError, _capi.OdbError)):
        bm.edges(p.double())
    assert bm._state is None and _capi.launch_count() == n0


# ------------------------------------------------------------------------------------------ evaluate.py
def _write_dataset(root):
    from PIL import Image
    img, gtd, edd = root / "img", root / "gt", root / "edges"
    for d in (img, gtd, edd):
        d.mkdir()
    rng = np.random.default_rng(0)
    for i in range(3):
        g = _np(scene(1, 384, 384, 50 + i)[0])
        rgb = (np.clip(g / g.max(), 0, 1)[..., None] * rng.uniform(0.5, 1.0, 3) * 255).astype(np.uint8)
        Image.fromarray(rgb).save(img / f"im{i}.png")
        np.save(gtd / f"im{i}.npy", g.astype(np.float32))
        e = (rng.random((384, 384)) < 0.01).astype(np.uint8) * 255
        if i == 1:
            Image.fromarray(e).save(edd / f"im{i}.png")
        else:
            np.save(edd / f"im{i}.npy", e > 0)
    return img, gtd, edd


def test_cli_boundary_equals_api(tmp_path, capsys):
    import evaluate
    from pathlib import Path
    from omnidata_b200.metrics import BoundaryMetrics
    img, gtd, edd = _write_dataset(tmp_path)
    model = evaluate.build_model("depth", "vitb_rn50_384", None, True, "bf16", dev)
    base = ["--task", "depth", "--img_path", str(img), "--gt_path", str(gtd), "--synthetic_weights", "--mode",
            "direct", "--max_depth", "10"]
    plain = evaluate.main(base)
    capsys.readouterr()
    assert "boundary" not in plain
    for extra in ([], ["--edge_path", str(edd)]):
        ret = evaluate.main(base + ["--boundary"] + extra)
        printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
        assert json.dumps(printed["metrics"]) == json.dumps(plain["metrics"])
        api = BoundaryMetrics(max_depth=10.0)
        for p in sorted(Path(img).iterdir()):
            gt = evaluate.load_gt(gtd / (p.stem + ".npy"), "depth", 512.0, 65535)
            pred = evaluate.predict(model, evaluate.image_tensor(p, "depth").to(dev), "direct", (384, 384), 64,
                                    p.name)
            edges = None
            if extra:
                edges = torch.from_numpy(evaluate.load_edges(next(edd.glob(p.stem + ".*")))).unsqueeze(0).to(dev)
            api.update(pred, torch.from_numpy(gt).unsqueeze(0).to(dev), None, edges)
        want = dict(api.compute(), edges="given" if extra else "detected")
        assert json.dumps(printed["boundary"]) == json.dumps(want) == json.dumps(ret["boundary"])
        assert want["images"] == 3 and want["gt_edge_pixels"] > 0
