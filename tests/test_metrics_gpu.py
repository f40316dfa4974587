"""Evaluation metrics on the GPU (omnidata_b200/metrics.py, csrc/metrics.cu) against the float64 oracle
(oracle/metrics_oracle.py, evaluated on the device in float64):

- depth: per-image records and dataset values to 1e-10 relative, delta counts equal, at 1x2 ... 3024x4032, full / empty /
  1 % / single-pixel masks, both spaces, with and without max_depth; a NaN prediction on a valid pixel gives NaN;
- normals: mean and RMSE to 1e-10 relative, threshold counts, the histogram and the median bin equal;
- a batch of 17, 17 batches of 1 and 5 + 12 leave bit-identical state; repeat runs are bit-identical; an update
  captured in a CUDA graph equals eager and nothing is allocated after the first call at a shape;
- every refusal raises before any launch;
- end to end on synthetic-weight models in bf16 (model(x), TiledPredictor) and through evaluate.py."""
import json
import math

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as O

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _close(a, b, rel=1e-10, floor=1e-14):
    if isinstance(b, float) and math.isnan(b):
        return isinstance(a, float) and math.isnan(a)
    return abs(a - b) <= rel * abs(b) + floor


SIZES = [(1, 2), (7, 5), (384, 384), (1080, 1920), (3024, 4032)]
MASKS = ["full", "empty", "random1pct", "single"]
CONFIGS = [("depth", math.inf), ("depth", 10.0), ("disparity", 10.0)]


def _mask(kind, b, h, w, seed):
    if kind == "full":
        return None
    if kind == "empty":
        return torch.zeros(b, h, w, dtype=torch.uint8, device=dev)
    if kind == "single":
        m = torch.zeros(b, h, w, dtype=torch.float32, device=dev)       # the fp32 mask dtype
        m[:, h // 2, w // 2] = 1.0
        return m
    m = torch.rand(b, h, w, generator=_gen(seed), device=dev) < 0.01
    m[:, 0, 0] = True                                                     # at least one pixel at the tiny sizes
    return m                                                              # bool, passed as uint8


def _depth_data(b, h, w, seed):
    g = torch.rand(b, h, w, generator=_gen(seed), device=dev) * 11.5 + 0.5
    p = 0.3 / g + 0.02 * torch.rand(b, h, w, generator=_gen(seed + 1), device=dev)   # a noisy disparity-like map
    return p.contiguous(), g.contiguous()


def _depth_records(p, g, m, space, max_depth):
    return [O.depth_image(p[i], g[i], None if m is None else m[i], space=space, min_depth=1e-3, max_depth=max_depth)
            for i in range(p.shape[0])]


def _check_records(rec, want):
    fields = ("n", "abs_rel", "sq_rel", "rmse", "rmse_log", "c1", "c2", "c3", "s", "t", "degenerate", "nonfinite")
    for i, w in enumerate(want):
        got = rec[i].tolist()
        for q, f in enumerate(fields):
            wv = float(w[f])
            if f in ("n", "c1", "c2", "c3", "degenerate", "nonfinite"):
                assert (math.isnan(wv) and math.isnan(got[q])) or got[q] == wv, (i, f, got[q], wv)
            else:
                assert _close(got[q], wv, floor=1e-12 if f in ("s", "t") else 1e-14), (i, f, got[q], wv)


def _check_dataset(got, want):
    for k, v in want.items():
        if isinstance(v, int):
            assert got[k] == v, (k, got[k], v)
        else:
            assert _close(got[k], v), (k, got[k], v)


@pytest.mark.parametrize("mask_kind", MASKS)
@pytest.mark.parametrize("h,w", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_depth_matches_oracle(h, w, mask_kind):
    from omnidata_b200.metrics import DepthMetrics
    b = 1 if h * w > 4e6 else 2
    p, g = _depth_data(b, h, w, h + 3 * w)
    m = _mask(mask_kind, b, h, w, h * w)
    for space, max_depth in CONFIGS:
        dm = DepthMetrics(space=space, max_depth=None if math.isinf(max_depth) else max_depth)
        rec = dm.update(p, g, m).cpu()
        want = _depth_records(p, g, m, space, max_depth)
        _check_records(rec, want)
        _check_dataset(dm.compute(), O.depth_dataset(want))
        if mask_kind == "single":                           # det = 0, unless max_depth leaves the pixel out of V
            out = dm.compute()
            assert out["degenerate"] + out["excluded"] == b and out["degenerate"] >= 1
        if mask_kind == "empty":
            assert dm.compute()["excluded"] == b and math.isnan(dm.compute()["abs_rel"])


def test_depth_nan_prediction_gives_nan():
    from omnidata_b200.metrics import DepthMetrics
    p, g = _depth_data(3, 40, 60, 5)
    p[1, 10, 20] = float("nan")
    dm = DepthMetrics()
    rec = dm.update(p, g).cpu()
    assert rec[1, 11] == 1.0 and all(math.isnan(v) for v in rec[1, 1:8].tolist())
    assert not any(math.isnan(v) for v in rec[0, :8].tolist() + rec[2, :8].tolist())
    out = dm.compute()
    assert math.isnan(out["abs_rel"]) and math.isnan(out["delta1"]) and out["images"] == 3
    _check_records(rec, _depth_records(p, g, None, "depth", math.inf))


def _normal_data(b, h, w, seed):
    gv = torch.randn(b, 3, h, w, generator=_gen(seed), device=dev)
    gv = gv / gv.norm(dim=1, keepdim=True)
    pv = gv + 0.4 * torch.randn(b, 3, h, w, generator=_gen(seed + 1), device=dev)
    pv = pv / pv.norm(dim=1, keepdim=True)
    return ((pv + 1) / 2).contiguous(), ((gv + 1) / 2).contiguous()


@pytest.mark.parametrize("mask_kind", MASKS)
@pytest.mark.parametrize("h,w", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_normals_match_oracle(h, w, mask_kind):
    from omnidata_b200.metrics import NormalMetrics
    b = 1 if h * w > 4e6 else 2
    p, g = _normal_data(b, h, w, 7 * h + w)
    m = _mask(mask_kind, b, h, w, h + w)
    nm = NormalMetrics()
    nm.update(p, g, m)
    got = nm.compute()
    th, bad = O.normal_angles(p, g, m)
    want = O.normal_dataset([th], bad)
    for k in ("pixels", "nonfinite", "n_11.25", "n_22.5", "n_30", "median_bin"):
        assert got[k] == want[k], (k, got[k], want[k])
    for k in ("mean", "rmse", "median", "pct_11.25", "pct_22.5", "pct_30"):
        assert _close(got[k], want[k]), (k, got[k], want[k])
    assert torch.equal(nm._state["hist"].cpu(), O.histogram(th))


def _depth_split(splits, p, g, m):
    from omnidata_b200.metrics import DepthMetrics
    dm = DepthMetrics(space="disparity", max_depth=10.0)
    i = 0
    for n in splits:
        dm.update(p[i:i + n], g[i:i + n], None if m is None else m[i:i + n])
        i += n
    return dm


def _normal_split(splits, p, g, m):
    from omnidata_b200.metrics import NormalMetrics
    nm = NormalMetrics()
    i = 0
    for n in splits:
        nm.update(p[i:i + n], g[i:i + n], m[i:i + n])
        i += n
    return nm


def test_batch_split_and_repeat_are_bit_identical():
    p, g = _depth_data(17, 100, 130, 11)
    m = (torch.rand(17, 100, 130, generator=_gen(12), device=dev) > 0.2).to(torch.uint8)
    pn, gn = _normal_data(17, 100, 130, 13)
    for split, data in ((_depth_split, (p, g, m)), (_normal_split, (pn, gn, m))):
        ref = split([17], *data)
        for s in ([1] * 17, [5, 12], [17]):
            other = split(s, *data)
            for k in ref._state:
                assert torch.equal(other._state[k], ref._state[k]), (split.__name__, s, k)
            assert json.dumps(other.compute()) == json.dumps(ref.compute())


def test_cuda_graph_replay_equals_eager_and_allocates_nothing():
    from omnidata_b200.metrics import DepthMetrics, NormalMetrics
    p, g = _depth_data(4, 96, 128, 21)
    pn, gn = _normal_data(4, 96, 128, 22)
    m = (torch.rand(4, 1, 96, 128, generator=_gen(23), device=dev) > 0.1).float()
    for cls, args in ((DepthMetrics, (p, g, m)), (NormalMetrics, (pn, gn, m))):
        eager = cls()
        eager.update(*args)
        eager.update(*args)
        cap = cls()
        cap.update(*args)                                   # first call at the shape: buffers and state allocated
        bufs = {k: v.data_ptr() for k, v in cap._bufs.items()}
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        cap.update(*args)
        torch.cuda.synchronize()
        assert torch.cuda.memory_allocated() == before
        assert {k: v.data_ptr() for k, v in cap._bufs.items()} == bufs
        cap.reset()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(graph, stream=s):
                cap.update(*args)
        torch.cuda.current_stream().wait_stream(s)
        graph.replay()
        graph.replay()
        torch.cuda.synchronize()
        for k in eager._state:
            assert torch.equal(cap._state[k], eager._state[k]), (cls.__name__, k)
        assert json.dumps(cap.compute()) == json.dumps(eager.compute())


def test_refusals_before_any_launch():
    from omnidata_b200 import _capi
    from omnidata_b200.metrics import DepthMetrics, NormalMetrics
    p, g = _depth_data(2, 32, 48, 31)
    pn, gn = _normal_data(2, 32, 48, 32)
    n0 = _capi.launch_count()
    with pytest.raises(ValueError):
        DepthMetrics(space="disparity")
    dm, nm = DepthMetrics(), NormalMetrics()
    bad_depth = [(p.cpu(), g.cpu(), None), (p.bfloat16(), g, None), (p, g.double(), None), (p, g[:, :31], None),
                 (p.transpose(1, 2).contiguous().transpose(1, 2), g, None), (p[:, None].expand(2, 2, 32, 48), g, None),
                 (p, g, torch.ones(2, 32, 48, dtype=torch.int32, device=dev)), (p, g, torch.ones(2, 32, 47, device=dev)),
                 (p, g, torch.ones(2, 2, 32, 48, device=dev)), (p[:0], g[:0], None), (p, g, torch.ones(2, 32, 48, dtype=torch.uint8))]
    for a, b, m in bad_depth:
        with pytest.raises((ValueError, _capi.OdbError)):
            dm.update(a, b, m)
    for a, b, m in [(pn[:, :1], gn[:, :1], None), (pn, gn[:, :, :31], None), (pn.cpu(), gn.cpu(), None),
                    (pn, gn, torch.ones(2, 3, 32, 48, device=dev)), (p, g, None)]:
        with pytest.raises((ValueError, _capi.OdbError)):
            nm.update(a, b, m)
    assert dm._state is None and nm._state is None          # refused before anything was allocated or launched
    assert _capi.launch_count() == n0


# ------------------------------------------------------------------------------------------ end to end
def _model(c):
    from omnidata_b200.model import DPTDepthModel
    from oracle import weights
    m = DPTDepthModel(num_channels=c, non_negative=False)
    m.load_state_dict(weights.make_state_dict(0, c), strict=True)
    return m.to(dev).eval()


@pytest.mark.parametrize("c", [1, 3])
def test_model_and_tiled_predictions_end_to_end(c):
    from omnidata_b200.metrics import DepthMetrics, NormalMetrics
    from omnidata_b200.tiled import TiledPredictor
    model = _model(c)
    x = torch.rand(4, 3, 384, 384, generator=_gen(41), device=dev) * 2 - 1
    xt = torch.rand(1, 3, 600, 900, generator=_gen(42), device=dev) * 2 - 1
    with torch.no_grad():
        preds = [model(x).float().clamp(0, 1).contiguous(),
                 TiledPredictor(model, tile=(384, 384), overlap=64)(xt).float().clamp(0, 1).contiguous()]
    for pred in preds:
        b, h, w = pred.shape[0], pred.shape[-2], pred.shape[-1]
        if c == 1:
            assert pred.shape == (b, h, w)
            g = torch.rand(b, h, w, generator=_gen(h), device=dev) * 5 + 0.5
            for space in ("depth", "disparity"):
                dm = DepthMetrics(space=space, max_depth=10.0)
                rec = dm.update(pred, g).cpu()
                want = _depth_records(pred, g, None, space, 10.0)
                _check_records(rec, want)
                _check_dataset(dm.compute(), O.depth_dataset(want))
        else:
            _, g = _normal_data(b, h, w, h + 1)
            nm = NormalMetrics()
            nm.update(pred, g)
            got = nm.compute()
            th, bad = O.normal_angles(pred, g)
            want = O.normal_dataset([th], bad)
            assert got["median_bin"] == want["median_bin"] and got["n_30"] == want["n_30"]
            assert _close(got["mean"], want["mean"]) and _close(got["rmse"], want["rmse"])


def _write_dataset(root, sizes, task):
    from PIL import Image
    img, gtd = root / "img", root / "gt"
    img.mkdir()
    gtd.mkdir()
    rng = np.random.default_rng(0)
    for i, (h, w) in enumerate(sizes):
        Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).save(img / f"im{i}.png")
        if task == "depth":
            if i == 2:
                v = rng.integers(256, 4096, (h, w)).astype(np.uint16)
                v[:4] = 65535                                          # no depth
                Image.fromarray(v).save(gtd / f"im{i}.png")
            else:
                np.save(gtd / f"im{i}.npy", rng.uniform(0.5, 8.0, (h, w)).astype(np.float32))
        else:
            n = rng.normal(size=(h, w, 3))
            n /= np.linalg.norm(n, axis=-1, keepdims=True)
            enc = (n + 1) / 2
            if i == 2:
                Image.fromarray((enc * 255).astype(np.uint8)).save(gtd / f"im{i}.png")
            else:
                np.save(gtd / f"im{i}.npy", enc.astype(np.float32).transpose(2, 0, 1))
    return img, gtd


@pytest.mark.parametrize("task", ["depth", "normal"])
def test_cli_equals_api(tmp_path, capsys, task):
    import evaluate
    from omnidata_b200.metrics import DepthMetrics, NormalMetrics
    from pathlib import Path
    img, gtd = _write_dataset(tmp_path, [(384, 384), (320, 448), (256, 288)], task)
    model = evaluate.build_model(task, "vitb_rn50_384", None, True, "bf16", dev)
    for mode in ("tiled", "direct"):
        argv = ["--task", task, "--img_path", str(img), "--gt_path", str(gtd), "--synthetic_weights", "--mode", mode]
        if task == "depth":
            argv += ["--max_depth", "10", "--space", "disparity"]
        ret = evaluate.main(argv)
        line = capsys.readouterr().out.strip().splitlines()[-1]
        printed = json.loads(line)
        assert printed["images"] == 3 and printed["mode"] == mode and printed["precision"] == "bf16"
        api = DepthMetrics(space="disparity", max_depth=10.0) if task == "depth" else NormalMetrics()
        for p in sorted(Path(img).iterdir()):
            gpath = next(gtd.glob(p.stem + ".*"))
            gt = evaluate.load_gt(gpath, task, 512.0, 65535)
            pred = evaluate.predict(model, evaluate.image_tensor(p, task).to(dev), mode, (384, 384), 64, p.name)
            api.update(pred, torch.from_numpy(np.ascontiguousarray(gt)).unsqueeze(0).to(dev))
        want = api.compute()
        assert json.dumps(printed["metrics"]) == json.dumps(want) == json.dumps(ret["metrics"])
    from PIL import Image
    odd = tmp_path / "odd"
    odd.mkdir()
    Image.fromarray(np.zeros((500, 500, 3), dtype=np.uint8)).save(odd / "big.png")
    np.save(odd / "big.npy", np.ones((500, 500) if task == "depth" else (3, 500, 500), dtype=np.float32))
    with pytest.raises(ValueError, match="big.png"):
        evaluate.main(["--task", task, "--img_path", str(odd), "--gt_path", str(odd), "--synthetic_weights",
                       "--mode", "direct"])
