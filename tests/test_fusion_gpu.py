"""Depth-normal fusion on the GPU (DepthNormalFusion, depth_normals; csrc/fusion.cu).

- depth_normals on guarded buffers against the float64 oracle (oracle/fusion_oracle.py): within 1 fp32 ulp, NaN at the
  same pixels, at 1x1 to 3024x4032, widths not divisible by 4 and every mask kind.
- The fusion with tol 1e-10 against the oracle's exact solve of the bordered energy: z within 1e-7 relative, t within
  1e-7, |V| and the kept edges exactly; at 3024x4032 the residual of the oracle's operator M.
- Status rules, NaN normals and depths, batch independence, repeat runs, CUDA-graph replay, no synchronisation and no
  allocation beyond the output after the first call.
- End to end with synthetic weights (hybrid, bf16) and evaluate.py --fuse_normals."""
import json

import numpy as np
import pytest
import torch

from oracle import fusion_oracle as FO
from oracle.guard import Guarded, bits

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _intr(h, w):
    f = 0.9 * max(h, w)
    return (f, f, (w - 1) / 2, (h - 1) / 2)


def _scene(b, h, w, seed, noise=0.0, shift=0.0):
    """depth fp32 [b,h,w] (piecewise-planar, plus seeded noise and a shift) and its exact normals fp32 [b,3,h,w]"""
    K = _intr(h, w)
    zs, cs = [], []
    rng = np.random.default_rng(seed)
    for i in range(b):
        z, c = FO.planes_scene(h, w, K, seed * 100 + i)
        zs.append(z + shift + noise * rng.standard_normal((h, w)))
        cs.append(c)
    return np.stack(zs).astype(np.float32), np.stack(cs).astype(np.float32), K


def _mask(kind, b, h, w, seed):
    if kind is None:
        return None
    m = np.random.default_rng(seed).random((b, h, w)) < 0.9
    return torch.from_numpy(m.astype(np.float32) if kind == "f32" else m if kind == "bool" else m.astype(np.uint8))


def _guarded_out(shape, gen):
    g = Guarded(int(np.prod(shape)), torch.float32, gen)
    return g, g.contiguous(*shape)


def _guards_intact(g, snap, out):
    changed = bits(g.t) != bits(snap)
    assert not bool((changed & ~g.mask([out])).any()), "a write outside the output"


@pytest.mark.parametrize("shape,mkind", [((1, 1, 1), None), ((2, 1, 37), "u8"), ((1, 2, 2), None),
                                         ((2, 384, 384), "bool"), ((1, 37, 53), "f32"), ((1, 1080, 1920), None),
                                         ((1, 3024, 4032), "u8")], ids=str)
def test_depth_normals_match_the_oracle(shape, mkind):
    from omnidata_b200 import ops
    b, h, w = shape
    depth, _, K = _scene(b, h, w, 1, noise=1e-3)
    mask = _mask(mkind, b, h, w, 2)
    gen = torch.Generator(device=dev).manual_seed(3)
    g, out = _guarded_out((b, 3, h, w), gen)
    ws = torch.empty(-(-ops.depth_normals_workspace_bytes(b, h, w) // 8), dtype=torch.float64, device=dev)
    d = torch.from_numpy(depth).to(dev)
    m = None if mask is None else mask.to(dev)
    snap = g.t.clone()
    ops.depth_normals(d, m, K, (1, -1, -1), 0.02, ws, out)
    torch.cuda.synchronize()
    _guards_intact(g, snap, out)
    first = out.clone()
    ops.depth_normals(d, m, K, (1, -1, -1), 0.02, ws, out)
    assert torch.equal(bits(out), bits(first))
    got = first.cpu().numpy()
    worst = 0.0
    for i in range(b):
        want = FO.depth_normals(depth[i], K, mask=None if mask is None else mask[i].numpy())
        assert np.array_equal(np.isnan(got[i]), np.isnan(want))
        fin = np.isfinite(want)
        if fin.any():
            ulp = np.spacing(np.abs(want[fin])).astype(np.float64)
            worst = max(worst, float(np.max(np.abs(got[i][fin].astype(np.float64) - want[fin]) / ulp)))
    print(f"{shape} {mkind}: {worst:.0f} ulp, {np.isnan(got).mean():.3f} NaN")
    assert worst <= 1.0
    if h * w == 1 or h == 1:
        assert np.isnan(got).all()


CASES = [  # (b, h, w, mask, shift, noise, shifted input)
    (1, 48, 64, None, False, 0.0, 0.0),
    (2, 48, 64, None, True, 0.0, 0.5),
    (2, 61, 83, "u8", True, 0.01, 0.0),
    (1, 200, 300, "f32", True, 0.01, 0.5),
    (1, 256, 384, "bool", False, 0.01, 0.0),
    (1, 512, 512, None, True, 0.01, 0.0),
]


@pytest.mark.parametrize("case", CASES, ids=str)
def test_fusion_matches_the_exact_solve(case):
    from omnidata_b200.fusion import DepthNormalFusion
    b, h, w, mkind, shift, noise, off = case
    depth, normals, K = _scene(b, h, w, 4, noise=noise, shift=off)
    mask = _mask(mkind, b, h, w, 5)
    fus = DepthNormalFusion(shift=shift, tol=1e-10, iterations=10000)
    out, rec = fus.fit(torch.from_numpy(depth).to(dev), torch.from_numpy(normals).to(dev), K,
                       None if mask is None else mask.to(dev))
    out, rec = out.cpu().numpy(), rec.cpu().numpy()
    for i in range(b):
        want = FO.fuse(depth[i], normals[i], K, shift=shift, mask=None if mask is None else mask[i].numpy())
        assert rec[i, 0] == want["n"] and rec[i, 2] == want["kept"] and rec[i, 1] == 0, (rec[i], want["n"])
        fin = np.isfinite(want["z"])
        assert np.array_equal(np.isfinite(out[i]), fin)
        err = np.max(np.abs(out[i][fin] - want["z"][fin]) / np.abs(want["z"][fin]))
        print(f"{case}: {int(rec[i, 3])} iterations, z {err:.1e} relative, t {rec[i, 5]:.9f} vs {want['t']:.9f}")
        assert err <= 1e-7 and abs(rec[i, 5] - want["t"]) <= 1e-7 and rec[i, 4] <= 1e-10


def test_full_resolution_residual():
    from omnidata_b200.fusion import DepthNormalFusion
    h, w = 3024, 4032
    depth, normals, K = _scene(1, h, w, 6, noise=0.01)
    fus = DepthNormalFusion()
    out, rec = fus.fit(torch.from_numpy(depth).to(dev), torch.from_numpy(normals).to(dev), K)
    out, rec = out.cpu().numpy()[0].astype(np.float64), rec.cpu().numpy()[0]
    mv, bvec, v = FO.system(depth[0], normals[0], K)
    res = np.linalg.norm(bvec - mv(out)) / np.linalg.norm(bvec)
    # the floor that rounding z to fp32 alone puts on the residual: M applied to a half-ulp perturbation
    sign = np.where(np.random.default_rng(7).random(out.shape) < 0.5, -0.5, 0.5)
    floor = np.linalg.norm(mv(out + sign * np.spacing(out.astype(np.float32)).astype(np.float64)) - mv(out)) / \
        np.linalg.norm(bvec)
    print(f"3024x4032: {int(rec[3])} iterations, record |r|/|b| {rec[4]:.2e}, oracle residual {res:.2e}, fp32 "
          f"rounding floor {floor:.2e}")
    assert rec[1] == 0 and rec[4] <= 1e-8 and res <= 10 * 1e-8 + 2 * floor


def test_status_rules_and_nan_inputs():
    from omnidata_b200.fusion import STATUS, DepthNormalFusion
    depth, normals, K = _scene(5, 40, 56, 8, noise=0.01)
    mask = np.ones((5, 40, 56), np.uint8)
    mask[0] = 0                                                     # V empty
    depth[1] = 2.5                                                  # a constant on V
    depth[3, 5:9, 7:30] = np.nan                                    # NaN depths leave V
    normals[3, 1, 20:30, 3:9] = np.nan                              # NaN normals drop their edges
    d, n, m = (torch.from_numpy(t).to(dev) for t in (depth, normals, mask))
    out, rec = DepthNormalFusion(tol=1e-10, iterations=10000).fit(d, n, K, m)
    out, rec = out.cpu().numpy(), rec.cpu().numpy()
    assert [STATUS[int(s)] for s in rec[:, 1]] == ["empty", "flat", "converged", "converged", "converged"]
    assert np.isnan(out[:2]).all() and np.isnan(rec[:2, 4]).all() and np.isnan(rec[:2, 5]).all()
    want = FO.fuse(depth[3], normals[3], K, mask=mask[3])
    assert rec[3, 0] == want["n"] == 40 * 56 - 4 * 23 and rec[3, 2] == want["kept"]
    assert np.array_equal(np.isnan(out[3]), np.isnan(depth[3]))
    out1, rec1 = DepthNormalFusion(iterations=1).fit(d, n, K, m)
    rec1 = rec1.cpu().numpy()
    assert (rec1[2:, 1] == 3).all() and (rec1[2:, 3] == 1).all() and np.isfinite(out1.cpu().numpy()[2]).all()


def test_batch_split_and_repeat_runs_give_the_same_bits():
    from omnidata_b200.fusion import DepthNormalFusion
    depth, normals, K = _scene(3, 96, 128, 9)
    depth[0] += 0.3                                                 # converges after a different number of iterations
    depth[1] += 0.01 * np.random.default_rng(10).standard_normal((96, 128)).astype(np.float32)
    d, n = torch.from_numpy(depth).to(dev), torch.from_numpy(normals).to(dev)
    fus = DepthNormalFusion()
    out, rec = (t.clone() for t in fus.fit(d, n, K))
    iters = rec[:, 3].cpu().tolist()
    print("iterations per image:", iters)
    assert len(set(iters)) == 3
    for i in range(3):
        o, r = fus.fit(d[i:i + 1], n[i:i + 1], K)
        assert torch.equal(bits(o), bits(out[i:i + 1])) and torch.equal(bits(r), bits(rec[i:i + 1]))
    o, r = fus.fit(d, n, K)
    assert torch.equal(bits(o), bits(out)) and torch.equal(bits(r), bits(rec))


def test_graph_replay_no_sync_no_alloc():
    from omnidata_b200.fusion import DepthNormalFusion
    depth, normals, K = _scene(2, 120, 160, 11, noise=0.01)
    d, n = torch.from_numpy(depth).to(dev), torch.from_numpy(normals).to(dev)
    fus = DepthNormalFusion(iterations=300)
    want = fus(d, n, K)
    torch.cuda.synchronize()
    n0 = torch.cuda.memory_stats()["allocation.all.allocated"]
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = fus(d, n, K)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.cuda.memory_stats()["allocation.all.allocated"] - n0 == 1    # the output
    assert torch.equal(bits(out), bits(want))
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fus(d, n, K)
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(graph):
        static = fus(d, n, K)
    static.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(static), bits(want))


def _models():
    from omnidata_b200.model import DPTDepthModel
    from oracle import weights
    out = []
    for c in (1, 3):
        m = DPTDepthModel(backbone="vitb_rn50_384", num_channels=c)
        m.load_state_dict(weights.make_state_dict(0, c), strict=True)
        out.append(m.to(dev).eval())
    return out


@pytest.mark.parametrize("which", ["direct", "tiled"])
def test_on_predictor_output(which):
    from omnidata_b200.fusion import DepthNormalFusion, depth_normals
    from omnidata_b200.tiled import TiledPredictor
    depth_model, normal_model = _models()
    h, w = (384, 384) if which == "direct" else (1080, 1920)
    g = torch.Generator().manual_seed(13)
    x = torch.rand(1, 3, h, w, generator=g).to(dev)
    with torch.no_grad():
        run = (lambda m, v: m(v)) if which == "direct" else \
            (lambda m, v: TiledPredictor(m, tile=(384, 384), overlap=64)(v))
        depth = run(depth_model, x * 2 - 1).float().clamp(0, 1).contiguous().reshape(1, h, w)
        normals = run(normal_model, x).float().clamp(0, 1).contiguous()
    K = _intr(h, w)
    fused, rec = DepthNormalFusion().fit(depth, normals, K)
    dn, nn, fz, rec = depth.cpu().numpy()[0], normals.cpu().numpy()[0], fused.cpu().numpy()[0], rec.cpu().numpy()[0]
    right, down, v = FO.edges(dn, nn, K)
    assert rec[0] == v.sum() and rec[2] == FO.kept_edges(right, down)
    mv, bvec, _ = FO.system(dn, nn, K)
    res = np.linalg.norm(bvec - mv(fz.astype(np.float64))) / np.linalg.norm(bvec)
    print(f"{which}: status {int(rec[1])}, {int(rec[3])} iterations, {int(rec[2])} kept edges, record |r|/|b| "
          f"{rec[4]:.1e}, oracle residual of the fp32 output {res:.1e}")
    assert rec[1] in (0, 3) and np.isfinite(fz[v]).all() and res <= max(1e-5, 10 * rec[4])
    if which == "direct":
        want = FO.fuse(dn, nn, K)
        fin = np.isfinite(want["z"])
        scale = np.abs(want["z"][fin]).max()
        if rec[1] == 0:
            assert np.max(np.abs(fz[fin] - want["z"][fin])) <= 1e-5 * scale
    got = depth_normals(depth, K).cpu().numpy()[0]
    want = FO.depth_normals(dn, K)
    assert np.array_equal(np.isnan(got), np.isnan(want))


def test_cli_fuse_normals(tmp_path, capsys):
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
            "direct"]
    plain = evaluate.main(base)
    capsys.readouterr()
    assert "fusion" not in plain
    ret = evaluate.main(base + ["--fuse_normals", "--intrinsics", "345.6,345.6,191.5,191.5"])
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert set(ret) - set(plain) == {"fusion"} and json.dumps(printed["fusion"]) == json.dumps(ret["fusion"])
    assert json.dumps(ret["metrics"]) == json.dumps(plain["metrics"])
    f = ret["fusion"]
    assert sum(f["records"][k] for k in ("converged", "empty", "flat", "not_converged")) == 2
    assert f["metrics"]["images"] == 2 and set(f["consistency"]) == {"pred", "fused"}
    print(json.dumps(f))
