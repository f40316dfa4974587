"""Anchored tiled inference on the GPU (TiledPredictor(anchor=...), csrc/tiled.cu, csrc/imageproc.cu).

- Kernels on guarded buffers (oracle/guard.py checked_launch: every output written, nothing else touched, a second run
  bit-identical) against the float64 oracle (oracle/tiled_anchor_oracle.py): the antialiased bilinear resize to 2e-6 relative
  L2 of torch's float64 F.interpolate, the anchor moments to fp64 rounding, the anchored solve to 1e-9.
- TiledPredictor with an anchor: the anchor is the model's prediction of the resized image, resized back; the merge of
  the model's own tile and anchor predictions matches the oracle's; batch 3 equals three batch-1 calls; repeat calls
  and CUDA-graph replay give the eager bits; the refusals raise before any launch."""
import pytest
import torch

from oracle import tiled_anchor_oracle as A
from oracle import tiled_oracle as O
from oracle.guard import Guarded, checked_launch

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _grid(H, W, tile, ov):
    oy, ox = O.grid(H, W, tile, ov)
    return len(oy), len(ox)


# ------------------------------------------------------------------------------------------ kernels
RESIZES = [(2, 384, 512, 192, 256), (1, 370, 555, 100, 150), (3, 590, 767, 100, 130), (2, 97, 131, 300, 413),
           (1, 123, 77, 123, 77), (3, 1080, 1920, 250, 333), (3, 3024, 4032, 768, 1024), (1, 768, 1024, 3024, 4032),
           (4, 33, 1, 7, 5)]


@pytest.mark.parametrize("planes,ih,iw,oh,ow", RESIZES, ids=[f"{p}x{a}x{b}-{c}x{d}" for p, a, b, c, d in RESIZES])
def test_resize_matches_torch_antialiased_bilinear(planes, ih, iw, oh, ow):
    """Downscaling by 2x, 3.7x and 5.9x, upscaling, identity, non-square sizes and sizes that are not multiples of 4."""
    from omnidata_b200 import ops
    g = _gen(ih * iw + oh)
    bx, bo = Guarded(planes * ih * iw, torch.float32, g), Guarded(planes * oh * ow, torch.float32, g)
    x, out = bx.contiguous(planes, ih, iw), bo.contiguous(planes, oh, ow)
    x.uniform_(-1.0, 3.0, generator=g)
    got, = checked_launch([bx, bo], [out], lambda: ops.resize_bilinear(x, out))
    want = A.resize(x.cpu(), (oh, ow))
    err = float((got.cpu().double() - want).norm() / want.norm())
    print(f"resize {planes}x{ih}x{iw} -> {oh}x{ow}: relative L2 {err:.2e}")
    assert err <= 2e-6


GEOMS = [(2, 300, 500, (384, 384), 64), (1, 1080, 1920, (384, 384), 64), (1, 3024, 4032, (384, 384), 64),
         (1, 1024, 1024, (512, 512), 64), (2, 97, 1000, (128, 96), 0), (1, 700, 400, (256, 128), 63)]
IDS = [f"{b}x{h}x{w}-t{t[0]}x{t[1]}-o{o}" for b, h, w, t, o in GEOMS]


@pytest.mark.parametrize("b,h,w,tile,ov", GEOMS, ids=IDS)
def test_anchor_moments(b, h, w, tile, ov):
    from omnidata_b200 import ops
    ny, nx = _grid(h, w, tile, ov)
    T = ny * nx
    g = _gen(5 * h + w)
    bp, ba = Guarded(b * T * tile[0] * tile[1], torch.float32, g), Guarded(b * h * w, torch.float32, g)
    bm = Guarded(b * T * 5, torch.float64, g)
    pred, anchor, mom = bp.contiguous(b * T, *tile), ba.contiguous(b, h, w), bm.contiguous(b, T, 5)
    pred.add_(2.0)                                          # non-zero means, as depth has
    anchor.add_(1.5)
    got, = checked_launch([bp, ba, bm], [mom], lambda: ops.tile_anchor_moments(pred, anchor, mom, tile, ov))
    want = A.anchor_moments(pred.cpu(), anchor.cpu(), b, h, w, tile, ov)
    err = float(((got.cpu() - want).abs() / want.abs().clamp_min(1.0)).max())
    print(f"anchor moments {b}x{h}x{w}: max relative error {err:.2e}")
    assert err <= 1e-12
    assert torch.equal(got[..., 0].cpu(), want[..., 0])


def _random_moments(b, ny, nx, seed, flat=False):
    """Overlap moments as tests/test_tiled_gpu.py builds them, and anchor moments of 300 pixels per tile whose anchor
    values are an affine map of the tile's values plus noise (flat: every tile's values equal)."""
    from omnidata_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    P, T = ops.tile_pairs(ny, nx), ny * nx
    a = torch.randn(b, P, 200, generator=gen, dtype=torch.float64) * 0.3 + 1.0
    c = a * (0.5 + torch.rand(b, P, 1, generator=gen, dtype=torch.float64)) + 0.1 * torch.randn(b, P, 1, generator=gen,
                                                                                            dtype=torch.float64)
    c = c + 0.01 * torch.randn(b, P, 200, generator=gen, dtype=torch.float64)
    n = torch.full((b, P), 200.0, dtype=torch.float64)
    m = torch.stack([n, a.sum(-1), c.sum(-1), (a * a).sum(-1), (c * c).sum(-1), (a * c).sum(-1)], -1)
    ta = torch.randn(b, T, 300, generator=gen, dtype=torch.float64) * 0.3 + 1.0
    if flat:
        ta = ta[..., :1].expand(b, T, 300)
    tg = ta * (0.5 + torch.rand(b, T, 1, generator=gen, dtype=torch.float64)) + torch.randn(b, T, 1, generator=gen,
                                                                                          dtype=torch.float64)
    tg = tg + 0.05 * torch.randn(b, T, 300, generator=gen, dtype=torch.float64)
    nt = torch.full((b, T), 300.0, dtype=torch.float64)
    am = torch.stack([nt, ta.sum(-1), (ta * ta).sum(-1), tg.sum(-1), (ta * tg).sum(-1)], -1)
    return m, am


@pytest.mark.parametrize("b,ny,nx,flat", [(1, 1, 1, False), (3, 1, 1, True), (2, 1, 2, False), (2, 4, 6, False),
                                          (1, 10, 13, False), (1, 10, 13, True), (2, 1, 1024, False),
                                          (1, 32, 32, False), (1, 24, 42, False)])
def test_anchored_solve(b, ny, nx, flat):
    """(1, 10, 13): 130 tiles, band in shared memory; (32, 32) and (24, 42): the 1 024-tile cap, band in the global
    workspace; flat: every tile's values equal (the kappa ridge keeps the solve well-posed)."""
    from omnidata_b200 import ops
    T = ny * nx
    g = _gen(T + 7)
    m, am = _random_moments(b, ny, nx, T, flat)
    P = m.shape[1]
    bm, ba = Guarded(max(b * P * 6, 1), torch.float64, g), Guarded(b * T * 5, torch.float64, g)
    bs = Guarded(b * T * 2, torch.float64, g)
    mom = bm.contiguous(b, P, 6) if P else None
    if mom is not None:
        mom.copy_(m)
    amom = ba.contiguous(b, T, 5)
    amom.copy_(am)
    st = bs.contiguous(b, T, 2)
    got, = checked_launch([bm, ba, bs], [st], lambda: ops.tile_align_solve_anchored(mom, amom, st, (ny, nx)))
    want = A.solve(m, am, ny, nx)
    err = float((got.cpu() - want).norm() / want.norm())
    print(f"anchored solve {b}x{ny}x{nx}{' flat' if flat else ''}: rel {err:.2e}")
    assert err <= 1e-9


# ------------------------------------------------------------------------------------------ TiledPredictor
def _model(backbone, c):
    from omnidata_b200 import synthetic
    from omnidata_b200.model import DPTDepthModel, state_dict_spec
    from oracle import weights
    if backbone == "vitb_rn50_384":
        sd = weights.make_state_dict(0, c)
    else:
        sd = synthetic.make_state_dict(0, c, spec=state_dict_spec(c, backbone=backbone))
    m = DPTDepthModel(backbone=backbone, num_channels=c, non_negative=False)   # depth: keep the random-weight map signed
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(backbone, c):
        if (backbone, c) not in cache:
            cache.clear()                                   # one model resident at a time
            torch.cuda.empty_cache()
            cache[(backbone, c)] = _model(backbone, c)
        return cache[(backbone, c)]
    return get


def _image(b, h, w, seed=0):
    g = torch.Generator().manual_seed(seed + h + 7 * w)
    return (torch.rand(b, 3, h, w, generator=g) * 2 - 1).to(dev)


CASES = [("vitb_rn50_384", p, 1, 1080, 1920, (384, 672)) for p in ("bf16", "fp32", "fp8")] + \
        [("vitb_rn50_384", "bf16", 2, 300, 500, (320, 512))] + \
        [("vitb16_384", p, 1, 1080, 1920, (544, 960)) for p in ("bf16", "fp32", "fp8")]


@pytest.mark.parametrize("backbone,precision,b,h,w,anchor", CASES,
                         ids=[f"{bb}-{p}-{b}x{h}x{w}-a{a[0]}x{a[1]}" for bb, p, b, h, w, a in CASES])
def test_anchored_predictor_matches_model_and_oracle(models, backbone, precision, b, h, w, anchor):
    from omnidata_b200 import ops
    from omnidata_b200.tiled import TiledPredictor
    model = models(backbone, 1)
    model.precision = precision
    tile = (384, 384)
    try:
        p = TiledPredictor(model, tile=tile, overlap=64, max_batch=32, anchor=anchor)
        x = _image(b, h, w)
        pred = p.tile_predictions(x)
        g = p.anchor_prediction(x)
        with torch.no_grad():                               # the anchor: model(resize(x)), resized back
            small = torch.empty(b, 3, *anchor, device=dev)
            ops.resize_bilinear(x, small)
            y = model(small).view(b, *anchor).contiguous()
            ref = torch.empty(b, h, w, device=dev)
            ops.resize_bilinear(y, ref)
        assert torch.equal(g, ref)
        out = p.merge(pred, b, h, w, anchor=g)
        assert torch.equal(p(x), out)
        want = A.merge(pred.cpu().double(), g.cpu().double(), b, h, w, tile, 64)
        scale = float(want.abs().max())
        err = float((out.cpu().double() - want).abs().max()) / scale
        # how far the merge sits from the anchor it is fitted to (not a pass criterion: random weights)
        gap = float((out - g).abs().max() / (g.max() - g.min()))
        print(f"{backbone} {precision} {h}x{w} anchor {anchor[0]}x{anchor[1]}: {pred.shape[0]} tiles, max error vs the "
              f"float64 merge {err:.2e} of max |out|; max |out - anchor| {gap:.2e} of the anchor's range")
        assert tuple(out.shape) == (b, h, w)
        assert err <= 2e-6
    finally:
        model.precision = "bf16"


def test_anchored_batch3_equals_three_batch1_calls(models):
    from omnidata_b200.tiled import TiledPredictor
    model = models("vitb_rn50_384", 1)
    p = TiledPredictor(model, max_batch=2, anchor=(448, 576))
    x = _image(3, 700, 900, seed=1)
    y = p(x)
    for i in range(3):
        assert torch.equal(p(x[i:i + 1])[0], y[i]), i
    assert torch.equal(p(x), y)                            # repeat calls: the same bits


def test_anchored_graph_replay_equals_eager(models):
    from omnidata_b200.tiled import TiledPredictor
    model = models("vitb_rn50_384", 1)
    p = TiledPredictor(model, max_batch=8, anchor=(384, 672))
    x = _image(1, 1080, 1920, seed=2)
    e = p(x)
    model.use_cuda_graph = True
    try:
        g1 = p(x)
        g2 = p(x)
    finally:
        model.use_cuda_graph = False
        model._graphs.clear()
    assert torch.equal(g1, e) and torch.equal(g2, e)


def test_anchor_refusals_before_any_launch(models):
    import evaluate
    from omnidata_b200 import _capi, ops
    from omnidata_b200.tiled import TiledPredictor
    normal = models("vitb_rn50_384", 3)
    n0 = _capi.launch_count()
    with pytest.raises(ValueError):                         # an anchor on a normal model
        TiledPredictor(normal, anchor=(384, 384))
    assert _capi.launch_count() == n0
    model = models("vitb_rn50_384", 1)
    n0 = _capi.launch_count()
    for anchor in [(400, 384), (384, 200), (1056, 1024), (512, 1824)]:   # not /32, above 4 096 patches, hybrid W
        with pytest.raises(ValueError):
            TiledPredictor(model, anchor=anchor)
    with pytest.raises(SystemExit):
        evaluate.main(["--task", "depth", "--img_path", "x", "--gt_path", "y", "--synthetic_weights", "--mode",
                       "direct", "--anchor", "384x384"])
    with pytest.raises(_capi.OdbError):                     # the front ends check shapes before launching
        ops.tile_align_solve_anchored(None, torch.zeros(1, 2, 5, device=dev, dtype=torch.float64),
                                      torch.zeros(1, 1, 2, device=dev, dtype=torch.float64), (1, 1))
    with pytest.raises(_capi.OdbError):
        ops.tile_anchor_moments(torch.zeros(4, 384, 384, device=dev), torch.zeros(1, 500, 500, device=dev),
                                torch.zeros(1, 3, 5, device=dev, dtype=torch.float64), (384, 384), 64)
    with pytest.raises(_capi.OdbError):
        ops.resize_bilinear(torch.zeros(2, 10, 10, device=dev), torch.zeros(3, 5, 5, device=dev))
    assert _capi.launch_count() == n0
    vit = models("vitb16_384", 1)
    TiledPredictor(vit, anchor=(512, 1824))                # W > 1 792 is a limit of the hybrid's stem only
