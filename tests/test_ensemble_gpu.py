"""Test-time ensembles on the GPU (EnsemblePredictor, csrc/ensemble.cu).

- Kernels on guarded buffers (oracle/guard.py checked_launch: every output written, nothing else touched, a second run
  bit-identical) against the float64 oracle (oracle/ensemble_oracle.py): the Gram to fp64 rounding, the solve to 1e-9,
  the depth merge and the normal merge bit for bit (the normal spread, through atan2, to 2 fp32 ulp).
- EnsemblePredictor: K = 1 is the model's own output; the members are the model's predictions of the resized and
  mirrored input; flip-equivariant stubs merge to the unflipped prediction; composition with TiledPredictor; batch 3
  equals three batch-1 calls; repeat calls and CUDA-graph replay give the eager bits; the merge neither synchronises
  nor allocates beyond its outputs; the refusals raise before any launch."""
import pytest
import torch
import torch.nn.functional as F

from oracle import ensemble_oracle as E
from oracle.guard import Guarded, checked_launch

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _members(K, B, C, H, W, seed, nan=False):
    """Members that look like depth: one smooth map per image, each member an affine map of it plus noise."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    base = 1.5 + torch.sin(3 * xx[None] + torch.rand(B, 1, 1, generator=g) * 3) * torch.cos(2 * yy[None])
    s = torch.rand(K, B, 1, 1, 1, generator=g) * 1.5 + 0.5
    t = torch.randn(K, B, 1, 1, 1, generator=g)
    m = (base[None, :, None] - t) / s + 0.02 * torch.randn(K, B, C, H, W, generator=g)
    if C == 3:
        m = torch.rand(K, B, C, H, W, generator=g) * 1.2 - 0.1                  # normals: [0, 1] and a little outside
        m[:, :, :, :2, :2] = 0.5                                                # |mean| = 0 somewhere
    if nan:
        m[1, 0, 0, 0, 1] = float("nan")
        m[K - 1, B - 1, 0, H - 1, 0] = float("inf")
    return m


def _flips(K):
    return sum(1 << k for k in range(1, K, 2))


GEOMS = [(2, 2, 384, 384), (3, 1, 1080, 1920), (6, 1, 3024, 4032), (16, 2, 97, 131), (5, 3, 100, 1001),
         (4, 1, 33, 18)]
IDS = [f"K{k}-{b}x{h}x{w}" for k, b, h, w in GEOMS]


@pytest.mark.parametrize("K,B,H,W", GEOMS, ids=IDS)
def test_gram_matches_oracle(K, B, H, W):
    from omnidata_b200 import ops
    flips = _flips(K)
    nq = (K + 1) * (K + 2) // 2
    m = _members(K, B, 1, H, W, seed=H + W, nan=True)
    g = _gen(K)
    bm, bg = Guarded(m.numel(), torch.float32, g), Guarded(B * nq, torch.float64, g)
    nws = ops.ensemble_gram_workspace_bytes(K, B, H, W) // 8
    bw = Guarded(nws, torch.float64, g)
    members, gram, ws = bm.contiguous(K, B, 1, H, W), bg.contiguous(B, nq), bw.contiguous(nws)
    members.copy_(m)
    got, wsc = checked_launch([bm, bg, bw], [gram, ws], lambda: ops.ensemble_gram(members, flips, gram, ws))
    want = E.gram(m, flips)
    err = float(((got.cpu() - want).abs() / want.abs().clamp_min(1.0)).max())
    print(f"gram K={K} {B}x{H}x{W}: max relative error {err:.2e}")
    assert err <= 1e-12
    assert torch.equal(got[:, -1].cpu(), want[:, -1])                          # n: exact


@pytest.mark.parametrize("K", [1, 2, 3, 6, 16])
def test_solve_matches_dense_float64(K):
    from omnidata_b200 import ops
    B = 3
    nq = (K + 1) * (K + 2) // 2
    m = _members(K, B, 1, 60, 70, seed=K)
    want_g = E.gram(m, 0)
    g = _gen(K + 100)
    bg, bs = Guarded(B * nq, torch.float64, g), Guarded(B * K * 2, torch.float64, g)
    gram, st = bg.contiguous(B, nq), bs.contiguous(B, K, 2)
    gram.copy_(want_g)
    got, = checked_launch([bg, bs], [st], lambda: ops.ensemble_align_solve(gram, st))
    want = E.solve(want_g, K)
    err = float((got.cpu() - want).norm() / want.norm())
    print(f"solve K={K}: relative error {err:.2e}")
    assert err <= 1e-9


def _same(a, b):
    """Bit for bit, NaN where NaN."""
    a, b = a.cpu(), b.cpu()
    return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a.nan_to_num(), b.nan_to_num())


def _solve_on_device(members, flips):
    from omnidata_b200 import ops
    K, B, _, H, W = members.shape
    gram = torch.empty(B, (K + 1) * (K + 2) // 2, device=dev, dtype=torch.float64)
    ws = torch.empty(ops.ensemble_gram_workspace_bytes(K, B, H, W) // 8, device=dev, dtype=torch.float64)
    st = torch.empty(B, K, 2, device=dev, dtype=torch.float64)
    ops.ensemble_gram(members, flips, gram, ws)
    ops.ensemble_align_solve(gram, st)
    return st


@pytest.mark.parametrize("K,B,H,W", GEOMS, ids=IDS)
def test_depth_merge_bit_for_bit(K, B, H, W):
    from omnidata_b200 import ops
    flips = _flips(K)
    m = _members(K, B, 1, H, W, seed=3 * H + W)
    g = _gen(K + H)
    bm, bo, bp = (Guarded(m.numel(), torch.float32, g), Guarded(B * H * W, torch.float32, g),
                  Guarded(B * H * W, torch.float32, g))
    members, out, spread = bm.contiguous(K, B, 1, H, W), bo.contiguous(B, H, W), bp.contiguous(B, H, W)
    members.copy_(m)
    st = _solve_on_device(members, flips)
    got, sp = checked_launch([bm, bo, bp], [out, spread],
                             lambda: ops.ensemble_merge_depth(members, flips, st, out, spread))
    want, wsp = E.merge_depth(m, flips, st.cpu())
    assert _same(got, want) and _same(sp, wsp)
    assert float((st.cpu() - E.solve(E.gram(m, flips), K)).norm() / st.norm()) <= 1e-9
    alone = torch.empty(B, H, W, device=dev)                                  # without the spread: the same output
    ops.ensemble_merge_depth(members, flips, st, alone)
    assert _same(alone, got)


def test_depth_merge_non_finite_pixels():
    from omnidata_b200 import ops
    K, B, H, W = 3, 2, 40, 52
    m = _members(K, B, 1, H, W, seed=9, nan=True).to(dev)
    st = _solve_on_device(m, 0b010)
    out, spread = torch.empty(B, H, W, device=dev), torch.empty(B, H, W, device=dev)
    ops.ensemble_merge_depth(m, 0b010, st, out, spread)
    want, wsp = E.merge_depth(m.cpu(), 0b010, st.cpu())
    assert _same(out, want) and _same(spread, wsp)
    assert int(torch.isnan(spread).sum()) == 2 and float(out[0, 0, W - 2]) == float(m[0, 0, 0, 0, W - 2])


@pytest.mark.parametrize("K,B,H,W", GEOMS, ids=IDS)
def test_normal_merge_bit_for_bit(K, B, H, W):
    from omnidata_b200 import ops
    flips = _flips(K)
    m = _members(K, B, 3, H, W, seed=H + 5 * W)
    g = _gen(K + W)
    bm, bo, bp = (Guarded(m.numel(), torch.float32, g), Guarded(B * 3 * H * W, torch.float32, g),
                  Guarded(B * H * W, torch.float32, g))
    members, out, spread = bm.contiguous(K, B, 3, H, W), bo.contiguous(B, 3, H, W), bp.contiguous(B, H, W)
    members.copy_(m)
    got, sp = checked_launch([bm, bo, bp], [out, spread], lambda: ops.ensemble_merge_normal(members, flips, out, spread))
    want, wsp = E.merge_normal(m, flips)
    assert _same(got, want)
    ulp = torch.finfo(torch.float32).eps * wsp.abs().clamp_min(torch.finfo(torch.float32).tiny)
    err = float(((sp.cpu() - wsp).abs() / ulp).max())
    print(f"normal spread K={K} {B}x{H}x{W}: max error {err:.2f} ulp")
    assert err <= 2.0


# ------------------------------------------------------------------------------------------ EnsemblePredictor
def _model(c, backbone="vitb_rn50_384"):
    from omnidata_b200 import synthetic
    from omnidata_b200.model import DPTDepthModel, state_dict_spec
    from oracle import weights
    sd = weights.make_state_dict(0, c) if backbone == "vitb_rn50_384" else \
        synthetic.make_state_dict(0, c, spec=state_dict_spec(c, backbone=backbone))
    m = DPTDepthModel(backbone=backbone, num_channels=c, non_negative=False)
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(c):
        if c not in cache:
            cache.clear()
            torch.cuda.empty_cache()
            cache[c] = _model(c)
        return cache[c]
    return get


def _image(b, h, w, seed=0):
    g = torch.Generator().manual_seed(seed + h + 7 * w)
    return (torch.rand(b, 3, h, w, generator=g) * 2 - 1).to(dev)


@pytest.mark.parametrize("precision", ["bf16", "fp32", "fp8"])
def test_one_member_is_the_model(models, precision):
    from omnidata_b200.ensemble import EnsemblePredictor
    model = models(1)
    model.precision = precision
    try:
        x = _image(2, 384, 512)
        with torch.no_grad():
            want = model(x)
        ens = EnsemblePredictor(model, flip=False)
        assert torch.equal(ens(x), want)
        out, spread = ens(x, return_spread=True)
        assert torch.equal(out, want) and float(spread.abs().max()) == 0.0
    finally:
        model.precision = "bf16"


def _expected_members(predictor, x, sizes, C):
    """model(resize(x)) and model(flip(resize(x))), resized back, as EnsemblePredictor documents them."""
    from omnidata_b200 import ops
    B, _, H, W = x.shape
    out = []
    with torch.no_grad():
        for size in sizes:
            h, w = size or (H, W)
            xs = x
            if (h, w) != (H, W):
                xs = torch.empty(B, 3, h, w, device=dev)
                ops.resize_bilinear(x, xs)
            for xin in (xs, torch.flip(xs, dims=(3,))):
                y = predictor(xin).float().reshape(B, C, h, w).contiguous()
                if (h, w) != (H, W):
                    back = torch.empty(B, C, H, W, device=dev)
                    ops.resize_bilinear(y, back)
                    y = back
                out.append(y)
    return torch.stack(out)


@pytest.mark.parametrize("c,b,h,w,sizes", [(1, 2, 384, 384, [None, (320, 448)]), (3, 2, 384, 384, [None, (320, 448)]),
                                           (1, 1, 512, 768, [(384, 576), None, (640, 960)])])
def test_members_are_model_predictions_and_merge_matches_oracle(models, c, b, h, w, sizes):
    from omnidata_b200.ensemble import EnsemblePredictor
    model = models(c)
    ens = EnsemblePredictor(model, sizes=sizes, flip=True, max_batch=1)
    x = _image(b, h, w, seed=c)
    members = ens.member_predictions(x).clone()
    assert torch.equal(members, _expected_members(model, x, sizes, c))
    out, spread = ens(x, return_spread=True)
    assert torch.equal(ens.member_predictions(x), members)                     # repeat calls: the same bits
    if c == 1:
        st = _solve_on_device(members, ens.flips)
        want, wsp = E.merge_depth(members.cpu(), ens.flips, st.cpu())
    else:
        want, wsp = E.merge_normal(members.cpu(), ens.flips)
    assert _same(out, want)
    assert tuple(out.shape) == ((b, h, w) if c == 1 else (b, 3, h, w)) and tuple(spread.shape) == (b, h, w)
    if c == 1:
        assert _same(spread, wsp)


class _DepthStub:
    """A flip-equivariant depth predictor (pointwise in x)."""
    num_channels = 1

    def __call__(self, x):
        return x[:, 0] * 2.0 + x[:, 1] * x[:, 2]


class _NormalStub:
    """A flip-equivariant normal predictor: n_x from a central horizontal difference (odd under mirroring), quantised so
    that 0.5 +- v is exact in fp32; n_y, n_z pointwise."""
    num_channels = 3

    def __call__(self, x):
        p = F.pad(x[:, :1], (1, 1, 0, 0), mode="replicate")
        d = p[..., 2:] - p[..., :-2]
        vx = torch.round(torch.tanh(d) * 256) / 1024
        return torch.cat([0.5 + vx, 0.5 + 0.25 * x[:, 1:2], 0.6 + 0.1 * x[:, 2:3]], 1)


def test_flip_equivariant_stubs_merge_to_the_unflipped_prediction():
    from omnidata_b200 import ops
    from omnidata_b200.ensemble import EnsemblePredictor
    x = _image(2, 70, 91, seed=4)
    d = EnsemblePredictor(_DepthStub(), flip=True)
    out, spread = d(x, return_spread=True)
    assert torch.equal(out, _DepthStub()(x)) and float(spread.max()) == 0.0
    n = EnsemblePredictor(_NormalStub(), flip=True)
    out, spread = n(x, return_spread=True)
    one = torch.empty_like(out)
    ops.ensemble_merge_normal(_NormalStub()(x)[None].contiguous(), 0, one)
    assert torch.equal(out, one)
    assert float(spread.max()) <= 1e-3
    # without the sign fix the mirrored member would point elsewhere wherever n_x != 0
    bad = torch.stack([_NormalStub()(x), torch.flip(_NormalStub()(torch.flip(x, dims=(3,))), dims=(3,))])
    wrong = torch.empty_like(out)
    ops.ensemble_merge_normal(bad.contiguous(), 0, wrong)
    assert not torch.equal(wrong, one)


def test_tiled_composition_at_1080p(models):
    from omnidata_b200.ensemble import EnsemblePredictor
    from omnidata_b200.tiled import TiledPredictor
    model = models(1)
    tiled = TiledPredictor(model, tile=(384, 384), overlap=64, max_batch=32)
    sizes = [None, (720, 1280)]
    ens = EnsemblePredictor(tiled, sizes=sizes, flip=True)
    x = _image(1, 1080, 1920, seed=5)
    members = ens.member_predictions(x).clone()
    assert torch.equal(members, _expected_members(tiled, x, sizes, 1))
    out = ens(x)
    st = _solve_on_device(members, ens.flips)
    assert _same(out, E.merge_depth(members.cpu(), ens.flips, st.cpu())[0])
    assert tuple(out.shape) == (1, 1080, 1920)


def test_batch3_equals_three_batch1_calls(models):
    from omnidata_b200.ensemble import EnsemblePredictor
    model = models(1)
    ens = EnsemblePredictor(model, sizes=[None, (320, 320)], flip=True, max_batch=2)
    x = _image(3, 384, 384, seed=6)
    y, s = ens(x, return_spread=True)
    for i in range(3):
        yi, si = ens(x[i:i + 1], return_spread=True)
        assert torch.equal(yi[0], y[i]) and _same(si[0], s[i]), i


def test_graph_replay_and_repeat_calls_equal_eager(models):
    from omnidata_b200.ensemble import EnsemblePredictor
    model = models(1)
    ens = EnsemblePredictor(model, sizes=[None, (448, 448)], flip=True)
    x = _image(2, 384, 384, seed=7)
    e = ens(x)
    assert torch.equal(ens(x), e)
    model.use_cuda_graph = True
    try:
        g1, g2 = ens(x), ens(x)
    finally:
        model.use_cuda_graph = False
        model._graphs.clear()
    assert torch.equal(g1, e) and torch.equal(g2, e)


def test_merge_neither_synchronises_nor_allocates(models):
    from omnidata_b200.ensemble import EnsemblePredictor
    model = models(1)
    ens = EnsemblePredictor(model, sizes=[None, (320, 320)], flip=True)
    x = _image(2, 384, 384, seed=8)
    members = ens.member_predictions(x)
    want, wsp = ens.merge(members, return_spread=True)                          # first call at this shape
    torch.cuda.synchronize()
    n0 = torch.cuda.memory_stats()["allocation.all.allocated"]
    torch.cuda.set_sync_debug_mode("error")
    try:
        out, spread = ens.merge(members, return_spread=True)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.cuda.memory_stats()["allocation.all.allocated"] - n0 == 2       # the two outputs
    assert torch.equal(out, want) and _same(spread, wsp)
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ens.merge(members)
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(graph):
        static = ens.merge(members)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, want)


def test_refusals_before_any_launch(models):
    import evaluate
    from omnidata_b200 import _capi, ops
    from omnidata_b200.ensemble import EnsemblePredictor
    from omnidata_b200.tiled import TiledPredictor
    model = models(1)
    n0 = _capi.launch_count()
    with pytest.raises(ValueError):
        EnsemblePredictor(model, sizes=[None] * 9)                              # 18 members
    for size in [(400, 384), (384, 200), (1056, 1024), (512, 1824)]:
        with pytest.raises(ValueError):
            EnsemblePredictor(model, sizes=[None, size])
    ens = EnsemblePredictor(model, sizes=[(384, 384), None])
    with pytest.raises(ValueError):                                             # the input's own size: hybrid W > 1792
        ens(_image(1, 1024, 1920))
    with pytest.raises(ValueError):
        ens(torch.zeros(1, 3, 384, 384, device=dev, requires_grad=True))
    with pytest.raises(_capi.OdbError):
        ens(torch.zeros(1, 3, 384, 384))
    tiled = TiledPredictor(model)
    with pytest.raises(ValueError):                                             # beyond the 1 024-tile cap
        EnsemblePredictor(tiled, sizes=[None, (20000, 20000)])
    with pytest.raises(SystemExit):
        evaluate.parse_args(["--task", "depth", "--img_path", "x", "--gt_path", "y", "--synthetic_weights",
                             "--ensemble_sizes", "384x"])
    m = torch.zeros(2, 1, 1, 8, 8, device=dev)
    with pytest.raises(_capi.OdbError):                                         # member 0 mirrored
        ops.ensemble_merge_depth(m, 0b01, torch.zeros(1, 2, 2, device=dev, dtype=torch.float64),
                                 torch.zeros(1, 8, 8, device=dev))
    with pytest.raises(_capi.OdbError):                                         # wrong channel count
        ops.ensemble_merge_normal(m, 0b10, torch.zeros(1, 3, 8, 8, device=dev))
    with pytest.raises(_capi.OdbError):
        ops.ensemble_align_solve(torch.zeros(1, 5, device=dev, dtype=torch.float64),
                                 torch.zeros(1, 2, 2, device=dev, dtype=torch.float64))
    assert _capi.launch_count() == n0
    model.train()
    try:
        with pytest.raises(ValueError):
            ens(_image(1, 384, 384))
    finally:
        model.eval()
    assert _capi.launch_count() == n0
