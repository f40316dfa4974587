"""Guided upsampling on the GPU (GuidedPredictor, csrc/guided.cu).

- Kernels on guarded buffers (oracle/guard.py checked_launch: every output written, nothing else touched, a second run
  bit-identical) against the float64 oracle (oracle/guided_oracle.py): the coefficients within 1 fp32 ulp of the
  oracle's rounded ones, the apply within 2e-6 of each output map's range.
- GuidedPredictor: the low-resolution prediction is the model's prediction of the resized input bit for bit, and the
  output is the oracle's filter of it; composition with EnsemblePredictor and around TiledPredictor; batch 3 equals
  three batch-1 calls; CUDA-graph replay gives the eager bits; refine neither synchronises nor allocates beyond its
  output; the refusals raise before any launch."""
import pytest
import torch

from oracle import guided_oracle as G
from oracle.guard import Guarded, checked_launch

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _smooth_scene(B, C, h, w, seed):
    """A guide in [-1, 1] and a prediction that follows it in places, with an edge and noise."""
    g = torch.Generator().manual_seed(seed)
    guide = torch.rand(B, 3, h, w, generator=g) * 2 - 1
    yy, xx = torch.meshgrid(torch.linspace(0, 1, h), torch.linspace(0, 1, w), indexing="ij")
    p = 0.5 * guide[:, :C] + (xx > 0.4).float() + 0.1 * torch.randn(B, C, h, w, generator=g) + yy
    return guide, p


def _ulp(t):
    a = t.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


COEF_CASES = [(2, 1, 384, 384, 4), (1, 3, 768, 1024, 8), (3, 1, 251, 333, 1), (1, 3, 97, 61, 32), (1, 1, 5, 7, 32)]


@pytest.mark.parametrize("B,C,h,w,r", COEF_CASES, ids=[f"{b}x{c}x{h}x{w}-r{r}" for b, c, h, w, r in COEF_CASES])
def test_coefficients_match_oracle(B, C, h, w, r):
    from omnidata_b200 import ops
    eps = 1e-3
    guide, p = _smooth_scene(B, C, h, w, seed=h + w + r)
    gen = _gen(C + r)
    nws = ops.guided_workspace_bytes(B, C, h, w) // 8
    bg, bp, bw, bc = (Guarded(guide.numel(), torch.float32, gen), Guarded(p.numel(), torch.float32, gen),
                      Guarded(nws, torch.float64, gen), Guarded(B * 4 * C * h * w, torch.float32, gen))
    dg, dp, ws, coef = bg.contiguous(B, 3, h, w), bp.contiguous(B, C, h, w), bw.contiguous(nws), \
        bc.contiguous(B, 4 * C, h, w)
    dg.copy_(guide)
    dp.copy_(p)
    got, _ = checked_launch([bg, bp, bw, bc], [coef, ws], lambda: ops.guided_coefficients(dg, dp, r, eps, ws, coef))
    want = G.coefficients(dg, dp, r, eps)                                   # float64 on the device, rounded to fp32
    # 1 ulp of each value; a value within 1e-12 of its plane's largest is held to that floor instead (a coefficient
    # that cancels to almost zero carries the fp64 rounding of the terms it cancelled)
    floor = 1e-12 * want.abs().amax((2, 3), keepdim=True).double()
    err = float(((got.double() - want.double()).abs() / torch.maximum(_ulp(want), floor)).max())
    print(f"coefficients {B}x{C}x{h}x{w} r={r}: max error {err:.2f} fp32 ulp")
    assert err <= 1.0


APPLY_CASES = [((384, 384), (1080, 1920), 1), ((768, 1024), (3024, 4032), 3), ((251, 333), (1000, 751), 3),
               ((251, 333), (1000, 751), 1), ((200, 328), (200, 328), 3), ((120, 160), (61, 77), 1)]


@pytest.mark.parametrize("lo,hi,C", APPLY_CASES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}-c{c}" for a, b, c in APPLY_CASES])
def test_apply_matches_oracle(lo, hi, C):
    from omnidata_b200 import ops
    (h, w), (H, W) = lo, hi
    g = torch.Generator().manual_seed(h + H + C)
    coef = torch.randn(1, 4 * C, h, w, generator=g)
    x = torch.rand(1, 3, H, W, generator=g) * 2 - 1
    gen = _gen(H + C)
    bx, bc, bo = (Guarded(x.numel(), torch.float32, gen), Guarded(coef.numel(), torch.float32, gen),
                  Guarded(C * H * W, torch.float32, gen))
    dx, dc, out = bx.contiguous(1, 3, H, W), bc.contiguous(1, 4 * C, h, w), bo.contiguous(1, C, H, W)
    dx.copy_(x)
    dc.copy_(coef)
    got, = checked_launch([bx, bc, bo], [out], lambda: ops.guided_apply(dx, dc, out))
    want = G.apply(dx, dc)
    for c in range(C):
        rng = float(want[:, c].max() - want[:, c].min())
        err = float((got[:, c].double() - want[:, c]).abs().max()) / rng
        print(f"apply {h}x{w} -> {H}x{W} channel {c}: max error {err:.2e} of its range")
        assert err <= 2e-6


def test_nan_reaches_only_its_windows():
    from omnidata_b200 import ops
    B, C, h, w, r = 1, 1, 40, 50, 2
    guide, p = _smooth_scene(B, C, h, w, seed=1)
    p[0, 0, 20, 25] = float("nan")
    dg, dp = guide.to(dev), p.to(dev)
    coef = torch.empty(B, 4, h, w, device=dev)
    ws = torch.empty(ops.guided_workspace_bytes(B, C, h, w) // 8, device=dev, dtype=torch.float64)
    ops.guided_coefficients(dg, dp, r, 1e-3, ws, coef)
    bad = ~torch.isfinite(coef[0, 3].cpu())
    want = torch.zeros(h, w, dtype=torch.bool)
    want[20 - 2 * r:20 + 2 * r + 1, 25 - 2 * r:25 + 2 * r + 1] = True        # two box passes of radius r
    assert torch.equal(bad, want)


# ------------------------------------------------------------------------------------------ GuidedPredictor
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

    def get(c, backbone="vitb_rn50_384"):
        if (c, backbone) not in cache:
            cache.clear()
            torch.cuda.empty_cache()
            cache[(c, backbone)] = _model(c, backbone)
        return cache[(c, backbone)]
    return get


def _image(b, h, w, seed=0, lo=-1.0):
    g = torch.Generator().manual_seed(seed + h + 7 * w)
    return (torch.rand(b, 3, h, w, generator=g) * (1 - lo) + lo).to(dev)


E2E = [(1, "bf16", "vitb_rn50_384"), (1, "fp32", "vitb_rn50_384"), (1, "fp8", "vitb_rn50_384"),
       (3, "bf16", "vitb_rn50_384"), (3, "fp32", "vitb_rn50_384"), (3, "fp8", "vitb_rn50_384"),
       (1, "bf16", "vitb16_384")]


@pytest.mark.parametrize("c,precision,backbone", E2E, ids=[f"c{c}-{p}-{b}" for c, p, b in E2E])
def test_end_to_end_matches_model_and_oracle(models, c, precision, backbone):
    from omnidata_b200 import ops
    from omnidata_b200.guided import GuidedPredictor
    model = models(c, backbone)
    model.precision = precision
    try:
        x = _image(2, 600, 900, seed=c, lo=-1.0 if c == 1 else 0.0)
        gp = GuidedPredictor(model, size=(384, 576), radius=4, eps=1e-3)
        g, p = gp.low_res_prediction(x)
        g, p = g.clone(), p.clone()
        small = torch.empty(2, 3, 384, 576, device=dev)
        ops.resize_bilinear(x, small)
        with torch.no_grad():
            want_p = model(small).float().reshape(2, c, 384, 576)
        assert torch.equal(g, small) and torch.equal(p, want_p)
        out = gp(x)
        assert tuple(out.shape) == ((2, 600, 900) if c == 1 else (2, 3, 600, 900))
        want = G.guided(x, g, p, 4, 1e-3)
        want = want[:, 0] if c == 1 else want
        rng = float(want.max() - want.min())
        err = float((out.double() - want).abs().max()) / rng
        print(f"{backbone} c={c} {precision}: max |out - oracle| {err:.2e} of the range")
        assert err <= 2e-6
    finally:
        model.precision = "bf16"


def test_ensemble_of_guided_predictors_at_1080p(models):
    from omnidata_b200.ensemble import EnsemblePredictor
    from omnidata_b200.guided import GuidedPredictor
    model = models(1)
    gp = GuidedPredictor(model, size=(576, 1024))
    ens = EnsemblePredictor(gp, flip=True)
    x = _image(1, 1080, 1920, seed=5)
    members = ens.member_predictions(x).clone()
    assert torch.equal(members[0], gp(x)[:, None])
    assert torch.equal(members[1], gp(torch.flip(x, dims=(3,)))[:, None])          # stored as predicted: mirrored
    out = ens(x)
    assert tuple(out.shape) == (1, 1080, 1920) and bool(torch.isfinite(out).all())


def test_guided_around_tiled_at_4032x3024(models):
    from omnidata_b200.guided import GuidedPredictor
    from omnidata_b200.tiled import TiledPredictor
    model = models(1)
    tiled = TiledPredictor(model, tile=(384, 384), overlap=64)
    gp = GuidedPredictor(tiled, size=(1536, 2048))
    x = _image(1, 3024, 4032, seed=6)
    g, p = gp.low_res_prediction(x)
    g, p = g.clone(), p.clone()
    with torch.no_grad():
        assert torch.equal(p[:, 0], tiled(g))
    out = gp(x)
    want = G.guided(x, g, p, 4, 1e-3)[:, 0]
    err = float((out.double() - want).abs().max()) / float(want.max() - want.min())
    print(f"guided around tiled: max |out - oracle| {err:.2e} of the range")
    assert tuple(out.shape) == (1, 3024, 4032) and err <= 2e-6


def test_batch3_equals_three_batch1_calls(models):
    from omnidata_b200.guided import GuidedPredictor
    model = models(1)
    gp = GuidedPredictor(model, size=(384, 512), max_batch=2)
    x = _image(3, 500, 700, seed=7)
    y = gp(x)
    for i in range(3):
        assert torch.equal(gp(x[i:i + 1])[0], y[i]), i


def test_graph_replay_and_repeat_calls_equal_eager(models):
    from omnidata_b200.guided import GuidedPredictor
    model = models(1)
    gp = GuidedPredictor(model, size=(384, 512))
    x = _image(2, 720, 1000, seed=8)
    e = gp(x)
    assert torch.equal(gp(x), e)
    model.use_cuda_graph = True
    try:
        g1, g2 = gp(x), gp(x)
    finally:
        model.use_cuda_graph = False
        model._graphs.clear()
    assert torch.equal(g1, e) and torch.equal(g2, e)


def test_refine_neither_synchronises_nor_allocates(models):
    from omnidata_b200.guided import GuidedPredictor
    model = models(3)
    gp = GuidedPredictor(model, size=(384, 512))
    x = _image(2, 700, 900, seed=9, lo=0.0)
    g, p = gp.low_res_prediction(x)
    want = gp.refine(x, g, p)                                               # first call at this shape
    torch.cuda.synchronize()
    n0 = torch.cuda.memory_stats()["allocation.all.allocated"]
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = gp.refine(x, g, p)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.cuda.memory_stats()["allocation.all.allocated"] - n0 == 1    # the output
    assert torch.equal(out, want)
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        gp.refine(x, g, p)
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(graph):
        static = gp.refine(x, g, p)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, want)


def test_refusals_before_any_launch(models):
    from omnidata_b200 import _capi, ops
    from omnidata_b200.guided import GuidedPredictor
    model = models(1)
    n0 = _capi.launch_count()
    for kw in ({"radius": 0}, {"radius": 33}, {"eps": 0.0}, {"eps": float("nan")}, {"max_batch": 0},
               {"size": (400, 384)}, {"size": (512, 1824)}):
        with pytest.raises(ValueError):
            GuidedPredictor(model, **{"size": (384, 384), **kw})
    gp = GuidedPredictor(model, size=(384, 384))
    with pytest.raises(ValueError):
        gp(torch.zeros(1, 3, 384, 384, device=dev, requires_grad=True))
    with pytest.raises(_capi.OdbError):
        gp(torch.zeros(1, 3, 384, 384))
    with pytest.raises(ValueError):
        gp(torch.zeros(1, 4, 384, 384, device=dev))
    with pytest.raises(ValueError):
        gp(torch.zeros(1, 3, 70000, 1, device=dev))
    g = torch.zeros(1, 3, 16, 16, device=dev)
    coef = torch.zeros(1, 4, 16, 16, device=dev)
    ws = torch.zeros(ops.guided_workspace_bytes(1, 1, 16, 16) // 8, device=dev, dtype=torch.float64)
    with pytest.raises(_capi.OdbError):                                     # two prediction channels
        ops.guided_coefficients(g, torch.zeros(1, 2, 16, 16, device=dev), 2, 1e-3, ws, coef)
    with pytest.raises(_capi.OdbError):                                     # radius beyond the cap
        ops.guided_coefficients(g, torch.zeros(1, 1, 16, 16, device=dev), 33, 1e-3, ws, coef)
    with pytest.raises(_capi.OdbError):                                     # workspace too small
        ops.guided_coefficients(g, torch.zeros(1, 1, 16, 16, device=dev), 2, 1e-3, ws[:10], coef)
    with pytest.raises(_capi.OdbError):                                     # fp64 coefficients
        ops.guided_apply(g, coef.double(), torch.zeros(1, 1, 16, 16, device=dev))
    with pytest.raises(_capi.OdbError):                                     # output with the wrong channel count
        ops.guided_apply(g, coef, torch.zeros(1, 3, 16, 16, device=dev))
    assert _capi.launch_count() == n0
    model.train()
    try:
        with pytest.raises(ValueError):
            gp(_image(1, 384, 384))
    finally:
        model.eval()
    assert _capi.launch_count() == n0
