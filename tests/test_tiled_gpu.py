"""Tiled inference on the GPU (omnidata_b200/tiled.py, csrc/tiled.cu).

- Kernels on guarded buffers (oracle/guard.py checked_launch: every output written, nothing else touched, a second run
  bit-identical) against the float64 oracle (oracle/tiled_oracle.py): the gather bit for bit, the overlap moments to
  fp64 rounding, the alignment solve to 1e-9 of the dense float64 solve (shared-memory and workspace band, a flat
  all-zero overlap, the tile-count cap), the blend to a few fp32 ulps.
- TiledPredictor: an image of exactly one tile returns model(x) bit for bit; the tile predictions it merges are
  model(tiles) bit for bit and the merge matches the oracle's merge of them; batch 3 equals three batch-1 calls; repeat
  calls and CUDA-graph replay give the eager bits; the refusals raise before any launch."""
import pytest
import torch

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
GEOMS = [(2, 300, 500, (384, 384), 64), (1, 1080, 1920, (384, 384), 64), (1, 3024, 4032, (384, 384), 64),
         (1, 1024, 1024, (512, 512), 64), (2, 97, 1000, (128, 96), 0), (1, 700, 400, (256, 128), 63)]
IDS = [f"{b}x{h}x{w}-t{t[0]}x{t[1]}-o{o}" for b, h, w, t, o in GEOMS]


@pytest.mark.parametrize("b,h,w,tile,ov", GEOMS, ids=IDS)
def test_gather_bit_exact(b, h, w, tile, ov):
    from omnidata_b200 import ops
    ny, nx = _grid(h, w, tile, ov)
    g = _gen(h + w)
    bx, bt = Guarded(b * 3 * h * w, torch.float32, g), Guarded(b * ny * nx * 3 * tile[0] * tile[1], torch.float32, g)
    x, tiles = bx.contiguous(b, 3, h, w), bt.contiguous(b * ny * nx, 3, *tile)
    got, = checked_launch([bx, bt], [tiles], lambda: ops.tile_gather(x, tiles, tile, ov))
    assert torch.equal(got.cpu(), O.gather(x.cpu(), tile, ov))


@pytest.mark.parametrize("b,h,w,tile,ov", GEOMS, ids=IDS)
def test_overlap_moments(b, h, w, tile, ov):
    from omnidata_b200 import ops
    ny, nx = _grid(h, w, tile, ov)
    P = ops.tile_pairs(ny, nx)
    if P == 0:
        pytest.skip("one tile: no pairs")
    g = _gen(7 * h + w)
    bp, bm = Guarded(b * ny * nx * tile[0] * tile[1], torch.float32, g), Guarded(b * P * 6, torch.float64, g)
    pred, mom = bp.contiguous(b * ny * nx, *tile), bm.contiguous(b, P, 6)
    pred.add_(2.0)                                          # a non-zero mean, as depth has
    got, = checked_launch([bp, bm], [mom], lambda: ops.tile_overlap_moments(pred, mom, (h, w), tile, ov))
    want = O.moments(pred.cpu(), b, h, w, tile, ov)
    err = ((got.cpu() - want).abs() / want.abs().clamp_min(1.0)).max()
    assert float(err) <= 1e-12, float(err)
    # a flat, all-zero overlap: exact zeros beside the pixel counts
    pred.zero_()
    got, = checked_launch([bp, bm], [mom], lambda: ops.tile_overlap_moments(pred, mom, (h, w), tile, ov))
    assert torch.equal(got[..., 1:].cpu(), torch.zeros(b, P, 5, dtype=torch.float64))
    assert torch.equal(got[..., 0].cpu(), want[..., 0])


def _random_moments(b, ny, nx, seed, zero=False):
    """Moments of random overlaps: each pair's b-values an affine map of its a-values plus noise."""
    from omnidata_b200 import ops
    g = torch.Generator().manual_seed(seed)
    P = ops.tile_pairs(ny, nx)
    a = torch.randn(b, P, 200, generator=g, dtype=torch.float64) * 0.3 + 1.0
    c = a * (0.5 + torch.rand(b, P, 1, generator=g, dtype=torch.float64)) + 0.1 * torch.randn(b, P, 1, generator=g,
                                                                                            dtype=torch.float64)
    c = c + 0.01 * torch.randn(b, P, 200, generator=g, dtype=torch.float64)
    if zero:
        a, c = a * 0, c * 0
    n = torch.full((b, P), 200.0, dtype=torch.float64)
    return torch.stack([n, a.sum(-1), c.sum(-1), (a * a).sum(-1), (c * c).sum(-1), (a * c).sum(-1)], -1)


@pytest.mark.parametrize("b,ny,nx,zero", [(1, 1, 1, False), (2, 1, 2, False), (2, 4, 6, False), (1, 10, 13, False),
                                          (1, 10, 13, True), (2, 1, 1024, False), (1, 32, 32, False),
                                          (1, 24, 42, False)])
def test_align_solve(b, ny, nx, zero):
    """(1, 10, 13): 130 tiles, band 260 x 28 in shared memory; (32, 32) and (24, 42): the 1 024-tile cap, band in the
    global workspace."""
    from omnidata_b200 import ops
    T = ny * nx
    g = _gen(T)
    m = _random_moments(b, ny, nx, T, zero)
    P = m.shape[1]
    bm, bs = Guarded(max(b * P * 6, 1), torch.float64, g), Guarded(b * T * 2, torch.float64, g)
    mom = bm.contiguous(b, P, 6) if P else None
    if mom is not None:
        mom.copy_(m)
    st = bs.contiguous(b, T, 2)
    got, = checked_launch([bm, bs], [st], lambda: ops.tile_align_solve(mom, st, (ny, nx)))
    want = O.solve(m, ny, nx)
    err = float((got.cpu() - want).norm() / want.norm())
    print(f"solve {b}x{ny}x{nx}{' zero' if zero else ''}: rel {err:.2e}")
    assert err <= 1e-9
    if T == 1 or zero:
        assert torch.allclose(got.cpu()[..., 0], torch.ones(b, T, dtype=torch.float64), rtol=0, atol=1e-12)


@pytest.mark.parametrize("c,with_st", [(1, True), (3, False)])
@pytest.mark.parametrize("b,h,w,tile,ov", GEOMS, ids=IDS)
def test_blend(b, h, w, tile, ov, c, with_st):
    from omnidata_b200 import ops
    ny, nx = _grid(h, w, tile, ov)
    T = ny * nx
    g = _gen(h * w + c)
    bp, bo = Guarded(b * T * c * tile[0] * tile[1], torch.float32, g), Guarded(b * c * h * w, torch.float32, g)
    bs = Guarded(b * T * 2, torch.float64, g)
    pred, out = bp.contiguous(b * T, c, *tile), bo.contiguous(b, c, h, w)
    st = None
    if with_st:
        st = bs.contiguous(b, T, 2)
        st[..., 0].mul_(0.1).add_(1.0)
    got, = checked_launch([bp, bo, bs], [out], lambda: ops.tile_blend(pred, st, out, tile, ov))
    p64 = pred.cpu().double()
    s32 = None if st is None else st.cpu().float().double()           # the kernel applies (s, t) in fp32
    want = O.blend(p64, s32, b, h, w, tile, ov)
    mag = O.blend(p64.abs(), None if s32 is None else s32.abs(), b, h, w, tile, ov)
    # mag is 0 only where every covering value is an exact 0 (randn yields a few in 10^7 samples); got is 0 there too
    err = float(((got.cpu().double() - want).abs() / mag.clamp_min(1e-300)).max())
    print(f"blend {b}x{h}x{w} c{c}: max error {err * 2 ** 24:.2f} fp32 ulps of the weighted magnitude")
    assert err <= 8 * 2.0 ** -24


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


@pytest.mark.parametrize("backbone,c", [("vitb_rn50_384", 1), ("vitb_rn50_384", 3), ("vitl16_384", 1)])
def test_one_tile_image_equals_model(models, backbone, c):
    from omnidata_b200.tiled import TiledPredictor
    model = models(backbone, c)
    x = _image(2, 384, 384)
    with torch.no_grad():
        y = model(x)
    assert torch.equal(TiledPredictor(model)(x), y)


CASES = [("vitb_rn50_384", 1, "bf16", 1, 300, 500, (384, 384)), ("vitb_rn50_384", 3, "bf16", 1, 300, 500, (384, 384)),
         ("vitb_rn50_384", 1, "fp32", 1, 300, 500, (384, 384)), ("vitb_rn50_384", 1, "bf16", 1, 1080, 1920, (384, 384)),
         ("vitb16_384", 1, "bf16", 1, 1080, 1920, (384, 384)), ("vitl16_384", 1, "bf16", 1, 1080, 1920, (384, 384)),
         ("vitb_rn50_384", 3, "bf16", 1, 1080, 1920, (384, 384)), ("vitb_rn50_384", 1, "fp8", 1, 1080, 1920, (384, 384)),
         ("vitb_rn50_384", 1, "bf16", 1, 3024, 4032, (384, 384)), ("vitb_rn50_384", 1, "bf16", 1, 1024, 1024, (512, 512))]


@pytest.mark.parametrize("backbone,c,precision,b,h,w,tile", CASES,
                         ids=[f"{bb}-c{c}-{p}-{h}x{w}-t{t[0]}" for bb, c, p, b, h, w, t in CASES])
def test_predictor_matches_model_and_oracle(models, backbone, c, precision, b, h, w, tile):
    from omnidata_b200.tiled import TiledPredictor
    model = models(backbone, c)
    model.precision = precision
    try:
        p = TiledPredictor(model, tile=tile, overlap=64, max_batch=32)
        x = _image(b, h, w)
        pred = p.tile_predictions(x)
        tiles = O.gather(x.cpu(), tile, 64).to(dev)
        with torch.no_grad():                               # model(tiles), in chunks of another size than max_batch
            ref = torch.cat([model(tiles[i:i + 13]).view(-1, c, *tile) for i in range(0, tiles.shape[0], 13)])
        assert torch.equal(pred, ref)
        out = p.merge(pred, b, h, w)
        assert torch.equal(p(x), out)
        want = O.merge(pred.cpu().double(), b, h, w, tile, 64)
        scale = float(want.abs().max())
        err = float((out.cpu().double() - want).abs().max()) / scale
        print(f"{backbone} c{c} {precision} {h}x{w}: {pred.shape[0]} tiles, max error vs the float64 merge {err:.2e} "
              f"of max |out|")
        assert tuple(out.shape) == ((b, h, w) if c == 1 else (b, c, h, w))
        assert err <= 2e-6
    finally:
        model.precision = "bf16"


def test_batch3_equals_three_batch1_calls(models):
    from omnidata_b200.tiled import TiledPredictor
    model = models("vitb_rn50_384", 1)
    p = TiledPredictor(model, max_batch=16)
    x = _image(3, 700, 900, seed=1)
    y = p(x)
    for i in range(3):
        assert torch.equal(p(x[i:i + 1])[0], y[i]), i
    assert torch.equal(p(x), y)                            # repeat calls: the same bits


def test_graph_replay_equals_eager(models):
    from omnidata_b200.tiled import TiledPredictor
    model = models("vitb_rn50_384", 1)
    p = TiledPredictor(model, max_batch=8)
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


def test_refusals_before_any_launch(models):
    from omnidata_b200 import _capi, ops
    from omnidata_b200.tiled import TiledPredictor
    model = models("vitb_rn50_384", 1)
    n0 = _capi.launch_count()
    for kw in [dict(tile=(400, 384)), dict(tile=(384, 1824)), dict(tile=(1056, 1024)), dict(overlap=-1),
               dict(overlap=192), dict(tile=(128, 384), overlap=64), dict(max_batch=0)]:
        with pytest.raises(ValueError):
            TiledPredictor(model, **kw)
    p = TiledPredictor(model)
    with pytest.raises(_capi.OdbError):
        p(torch.zeros(1, 3, 500, 500))
    for bad in [torch.zeros(3, 500, 500, device=dev), torch.zeros(1, 4, 500, 500, device=dev),
                torch.zeros(1, 3, 500, 500, device=dev, requires_grad=True)]:
        with pytest.raises(ValueError):
            p(bad)
    with pytest.raises(ValueError):                         # 33 x 32 tiles, above the 1 024-tile cap
        TiledPredictor(model, tile=(64, 64), overlap=0)(torch.zeros(1, 3, 64 * 33, 64 * 32, device=dev))
    model.train()
    try:
        with pytest.raises(ValueError):
            p(torch.zeros(1, 3, 500, 500, device=dev))
    finally:
        model.eval()
    with pytest.raises(_capi.OdbError):                     # the front ends check shapes before launching
        ops.tile_gather(torch.zeros(1, 3, 500, 500, device=dev), torch.zeros(1, 3, 384, 384, device=dev), (384, 384), 64)
    with pytest.raises(_capi.OdbError):
        ops.tile_align_solve(None, torch.zeros(1, 2, 2, device=dev, dtype=torch.float64), (1, 2))
    assert _capi.launch_count() == n0
