"""The backward GEMMs of the train step against float64 at every geometry the engine launches.

Three families of launches carry the backward: weight gradients (bwd.conv_wgrad), the attention backward
(bwd.attention_bwd) and input gradients (ops.conv_gemm with the rotated dgrad operands, stride-2 convolutions as four
parity-plane convolutions that store through strided views of dx).  Each launch here is checked, in bf16 and fp32
storage, on seeded operands against oracle/gemm_oracle.py (float64, the documented definition of each operation) for
  * its error, per element where the kernel's arithmetic bounds it;
  * writing every output element (prefilled with NaN unless it accumulates or aliases an input);
  * writing nothing else: every tensor lives in a buffer with 64 KiB guard bands of random values, and everything
    outside the output elements, inputs included, stays bit-identical (oracle/guard.py);
  * a second run from the same state being bit-identical.
Cases: a table that reaches every branch of the wgrad planner (pixel tile, N tile, split reduction, view kind), the
attention backward over token counts around the 64- and 128-row tiles and the 640-key padding, the two dgrad
compositions, and every distinct geometry a TrainEngine backward of each of the three DPTs (`vitb_rn50_384`, `vitl16_384`,
`vitb16_384`) launches at batch 2 and four input sizes, and of the hybrid and DPT-Large at the train benchmarks' batch 16,
recorded by wrapping the three entry points during one backward and replayed on random data.

Bounds, "measured X, bound Y" with X the largest value over every case of this file, measured on an NVIDIA H100 80GB
HBM3 with a 400 W power limit (the inputs are seeded, so the numbers repeat):
  * wgrad: the operands are exact and the output fp32, so the error is fp32 accumulation only, per element
    |kernel - ref| <= tau * (|dy|^T |x|): bf16 measured tau 1.3e-6 (DPT-Large at batch 16), bound 1.5e-6; fp32 measured
    2.7e-7, bound 1e-6.  rel-L2: bf16 measured 2.6e-5, bound 1e-4 (the engine's large reductions, e.g. the stem's
    73,728 pixels, cancel: rel-L2 grows like tau * sqrt(pixels)), so at batch 16 the bound is 1e-4 x sqrt(16 / 2):
    measured 2.0e-4, bound 2.8e-4; fp32 measured 1.1e-7, bound 4.5e-7.
  * conv_gemm (dgrad): bf16 output, |kernel - ref| <= 0.5 ulp + tau * (|x| |W| + |bias| + |residual|), the one rounding
    of the fp32 result plus fp32 accumulation: measured tau 4.3e-7, bound 1e-6; fp32 output (no rounding term):
    measured 2.4e-7, bound 1e-6.  The compositions against float64 autograd, rel-L2: bf16 measured 2.1e-3, bound 4e-3
    (the bf16 stores); fp32 measured 1.1e-7, bound 4e-7.
  * attention bf16: against the rounded oracle (the kernel's rounding points), an element passes within one bf16 ulp
    plus ATT_ABS = 1e-3 x the rms of its image's q / k / v block (fp32 against float64 accumulation).  A rounding flip
    of P or dS upstream moves a few elements further: measured fraction 1.2e-4, bound 2.5e-4, and no element beyond
    10.2 such units, bound 16.  Against the exact gradient: measured rel-L2 3.3e-3, bound 1e-2.  The forward's lse,
    which the rounded oracle starts from, against float64: measured max abs error 3.2e-6, bound 1e-5.
    fp32 against the exact gradient: measured rel-L2 1.4e-7, bound 5e-7.
"""
import pytest
import torch
import torch.nn.functional as F

from oracle import gemm_oracle as G
from oracle.guard import Guarded, checked_launch, geometry, materialize, same_storage, ulp_bf16

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float32]
TAU_WGRAD = {torch.bfloat16: 1.5e-6, torch.float32: 1e-6}
REL_WGRAD = {torch.bfloat16: 1e-4, torch.float32: 4.5e-7}
TAU_CONV = {torch.bfloat16: 1e-6, torch.float32: 1e-6}
REL_DGRAD = {torch.bfloat16: 4e-3, torch.float32: 4e-7}
ATT_ABS, ATT_FLIPS, ATT_MAX = 1e-3, 2.5e-4, 16.0
LSE_ABS = 1e-5


def dev():
    return torch.device("cuda:0")


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-300))


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


# ------------------------------------------------------------------------------------------ checks on identical operands
def check_wgrad(bufs, views, taps, dy, out, accumulate, rel_scale=1.0):
    """conv_wgrad into `out` against wgrad_ref (plus the prior content when accumulating) -> max tau, rel-L2.
    rel_scale widens the rel-L2 bound for batches above 2: the cancellation grows like sqrt(pixels)."""
    from omnidata_b200 import bwd
    prior = out.double().clone() if accumulate else 0.0
    ref = G.wgrad_ref(views, taps, dy) + prior
    scale = G.wgrad_abs_ref(views, taps, dy) + (prior.abs() if accumulate else 0.0)
    k, = checked_launch(bufs, [out], lambda: bwd.conv_wgrad(views, taps, dy, out, accumulate=accumulate),
                        prefill_nan=not accumulate)
    tau = float(((k.double() - ref).abs() / scale.clamp_min(1e-30)).max())
    r = rel(k, ref)
    assert tau <= TAU_WGRAD[dy.dtype] and r <= rel_scale * REL_WGRAD[dy.dtype], (tau, r)
    return {"tau": tau, "rel": r}


def check_conv(bufs, views, taps, weight, out, bias=None, residual=None, prefill_nan=True):
    """ops.conv_gemm into `out` against conv_gemm_ref (with the residual's content before the launch) -> max tau."""
    from omnidata_b200 import ops
    o4 = G.as4(out)
    grid = tuple(o4.shape[:3])
    ref = G.conv_gemm_ref(views, taps, weight, grid, bias=bias, residual=residual)
    scale = G.conv_acc_ref(views, taps, weight, grid, absolute=True)
    if bias is not None:
        scale = scale + bias.double().abs()
    if residual is not None:
        scale = scale + G.as4(residual).double().abs()
    k, = checked_launch(bufs, [out], lambda: ops.conv_gemm(views, taps, weight, out, bias=bias, residual=residual),
                        prefill_nan=prefill_nan)
    k = G.as4(k).double()
    err = (k - ref).abs()
    if out.dtype == torch.bfloat16:
        err = (err - 0.5 * torch.maximum(ulp_bf16(k), ulp_bf16(ref))).clamp_min(0)
    tau = float((err / scale.clamp_min(1e-30)).max())
    assert tau <= TAU_CONV[out.dtype], tau
    return {"tau": tau}


def check_attention(bufs, qkv, o, d_o, lse, dqkv, heads=12, scale=0.125):
    """o, lse from ops.attention of qkv, then attention_bwd into dqkv against the exact and the rounded oracle."""
    from omnidata_b200 import bwd, ops
    ops.attention(qkv, o, heads=heads, scale=scale, lse=lse)
    torch.cuda.synchronize()
    k, = checked_launch(bufs, [dqkv], lambda: bwd.attention_bwd(qkv, o, d_o, lse, dqkv, heads=heads, scale=scale))
    exact = G.attention_bwd_ref(qkv, o, d_o, scale=scale)
    e_exact = rel(k, exact)
    if qkv.dtype == torch.float32:
        assert e_exact <= 5e-7, e_exact
        return {"exact": e_exact}
    e_lse = float((lse.double() - G.lse_ref(qkv, heads, scale)).abs().max())   # the rounded oracle starts from it
    assert e_lse <= LSE_ABS, e_lse
    rnd = G.attention_bwd_ref(qkv, o, d_o, lse, rounded=True, scale=scale)
    kd = k.double()
    b, t, c3 = qkv.shape
    err = (kd - rnd).abs().view(b, t, 3, -1)
    rms = rnd.view(b, t, 3, -1).pow(2).mean(dim=(1, 3), keepdim=True).sqrt()           # per image and q / k / v block
    units = err / (ulp_bf16(rnd).view(b, t, 3, -1) + ATT_ABS * rms)
    flips, worst = float((units > 1).double().mean()), float(units.max())
    assert e_exact <= 1e-2 and flips <= ATT_FLIPS and worst <= ATT_MAX, (e_exact, flips, worst)
    return {"exact": e_exact, "flips": flips, "worst": worst, "lse": e_lse}


# ------------------------------------------------------------------------------------------ a. conv_wgrad, planner branches
# (id, view kind, B, H, W of the dy grid, C, n, taps, accumulate).  Kinds: "4d" contiguous [B,H,W,C]; "rows" 2-D
# [W, C] (a ViT linear layer, B = H = 1); "s2" the strided view t[:, ::2, ::2, :] (downsample); "tok" the token window
# t[:, 1:, :].unsqueeze(1) (readout); "same" / "sym1" the four parity planes of a [B, 2H, 2W, C] tensor with
# ops._parity_taps(kind).  The comment is the plan on a 132-SM H100: pixel tile, N tile, splits -> reduction.
WGRAD_CASES = [
    ("w96-3x3", "4d", 2, 3, 96, 64, 128, "3x3", False),          # 64x1 full + ragged, bn 64, 1 split -> direct
    ("w40-3x3", "4d", 2, 24, 40, 128, 64, "3x3", False),         # 32x2 ragged, bn 128, 6 splits -> plain
    ("stem", "4d", 2, 128, 20, 160, 64, "1", False),              # 16x4 ragged, C = 160: bn 192, 16 splits -> lanes
    ("same-w15", "same", 2, 10, 15, 256, 256, "same", False),     # 8x8 ragged, bn 256, MT 2 -> direct
    ("sym1-w12", "sym1", 2, 12, 12, 768, 768, "sym1", False),     # act_postprocess4.4: NT 3, MT 6 -> direct
    ("rows-1250", "rows", 1, 1, 1250, 1024, 768, "1", False),     # patch projection: 64x1 ragged, NT 4, 2 splits -> plain
    ("tok-601-acc", "tok", 2, 1, 601, 768, 768, "1", True),       # readout token window, accumulate, 2 splits -> plain
    ("cls", "4d", 1, 1, 2, 768, 768, "1", False),                 # the readout's [1,1,B,D] cls rows -> direct
    ("w2-n32-acc", "4d", 2, 2, 2, 64, 32, "3x3", True),           # 8x8 ragged, n 32, accumulate: 1 split -> plain
    ("w20-n104", "4d", 2, 10, 20, 64, 104, "3x3", False),         # n 104 (ragged M tile) -> direct
    ("rows-qkv", "rows", 1, 1, 1154, 768, 2304, "1", False),      # attn.qkv at T = 577: MT 18, 2 splits -> plain
    ("w96-lanes-acc", "4d", 2, 64, 96, 64, 64, "1", True),        # 32 splits -> lanes, accumulate
    ("s2-w20", "s2", 2, 48, 20, 256, 512, "1", False),            # downsample view, 6 splits -> plain
    ("w40-lanes", "4d", 2, 96, 40, 256, 64, "1", False),          # 24 splits -> lanes
]


def _wgrad_plan(B, H, W, C, n, ntaps, accumulate, sms):
    """(pixel tile width, N tile, N tiles, reduction) as csrc/bgemm_tc.cu wgrad_plan chooses them."""
    tw = 64 if W >= 64 else 32 if W >= 32 else 16 if W >= 16 else 8
    ksteps = -(-W // tw) * -(-H // (64 // tw)) * B
    bn = min(-(-C // 64) * 64, 256)
    tiles = -(-n // 128) * -(-C // bn) * ntaps
    splits = max(1, min(1 if tiles >= sms else sms // tiles, ksteps // 8, 256))
    kps = -(-ksteps // splits)
    splits = -(-ksteps // kps)
    red = "direct" if splits == 1 and not accumulate else "lanes" if splits >= 16 and n * ntaps * C <= 131072 else "plain"
    return tw, bn, -(-C // bn), red


def _taps(name):
    from omnidata_b200 import ops
    return {"3x3": ops.TAPS_3X3, "1": ops.TAPS_1}.get(name) or ops._parity_taps(name)


def test_wgrad_cases_reach_every_planner_branch():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    plans = [_wgrad_plan(B, H, W, C, n, len(_taps(t)), acc, sms) for _, _, B, H, W, C, n, t, acc in WGRAD_CASES]
    assert {p[0] for p in plans} == {64, 32, 16, 8} and {p[1] for p in plans} == {64, 128, 192, 256}
    assert any(p[2] > 1 for p in plans) and {p[3] for p in plans} == {"direct", "plain", "lanes"}, plans
    assert {c[1] for c in WGRAD_CASES} == {"4d", "rows", "s2", "tok", "same", "sym1"}


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("case", WGRAD_CASES, ids=[c[0] for c in WGRAD_CASES])
def test_conv_wgrad(case, dtype):
    _, kind, B, H, W, C, n, tname, acc = case
    g = gen(WGRAD_CASES.index(case))
    taps = _taps(tname)
    if kind in ("s2", "same", "sym1"):
        xb = Guarded(B * 4 * H * W * C, dtype, g)
        parent = xb.contiguous(B, 2 * H, 2 * W, C)
        views = [parent[:, ::2, ::2, :]] if kind == "s2" else [parent[:, py::2, px::2, :] for py in (0, 1) for px in (0, 1)]
    elif kind == "tok":
        xb = Guarded(B * (W + 1) * C, dtype, g)
        views = [xb.contiguous(B, W + 1, C)[:, 1:, :].unsqueeze(1)]
    elif kind == "rows":
        xb = Guarded(W * C, dtype, g)
        views = [xb.contiguous(W, C)]
    else:
        xb = Guarded(B * H * W * C, dtype, g)
        views = [xb.contiguous(B, H, W, C)]
    dyb = Guarded(B * H * W * n, dtype, g)
    dy = dyb.contiguous(W, n) if kind == "rows" else dyb.contiguous(B, H, W, n)
    ob = Guarded(n * len(taps) * C, torch.float32, g)
    out = ob.contiguous(n, len(taps) * C)
    res = check_wgrad([xb, dyb, ob], views, taps, dy, out, acc)
    print(f"wgrad {case[0]} {dtype}: tau {res['tau']:.2e}, rel-L2 {res['rel']:.2e}")


# ------------------------------------------------------------------------------------------ b. attention_bwd
ATT_TOKENS = [5, 25, 65, 127, 128, 129, 301, 577, 601, 625, 637, 640]


def _attention_buffers(b, t, dtype, seed, heads=12):
    g = gen(seed)
    bufs = [Guarded(b * t * 3 * heads * 64, dtype, g), Guarded(b * t * heads * 64, dtype, g),
            Guarded(b * t * heads * 64, dtype, g), Guarded(b * t * 3 * heads * 64, dtype, g)]
    qkv, o, d_o, dqkv = (bufs[0].contiguous(b, t, 3 * heads * 64), bufs[1].contiguous(b, t, heads * 64),
                         bufs[2].contiguous(b, t, heads * 64), bufs[3].contiguous(b, t, 3 * heads * 64))
    lse = None
    if dtype == torch.bfloat16:
        bufs.append(Guarded(b * heads * t, torch.float32, g))
        lse = bufs[-1].contiguous(b, heads, t)
    return bufs, qkv, o, d_o, lse, dqkv


# (tokens, heads): the ViT-B width at every token count above, DPT-Large's 16 heads (qkv 3072 wide) at a few
ATT_CASES = [(t, 12) for t in ATT_TOKENS] + [(t, 16) for t in (65, 577, 601, 640)]


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("b", [1, 3])
@pytest.mark.parametrize("t,heads", ATT_CASES, ids=[str(t) if h == 12 else f"{t}-{h}heads" for t, h in ATT_CASES])
def test_attention_bwd(t, heads, b, dtype):
    bufs, qkv, o, d_o, lse, dqkv = _attention_buffers(b, t, dtype, 1000 * b + t + heads, heads)
    qkv.view(b, t, 3, -1)[:, :, :2] *= 1.5                    # wider logits: a peaked softmax
    res = check_attention(bufs, qkv, o, d_o, lse, dqkv, heads)
    print(f"attention_bwd b={b} T={t} heads={heads} {dtype}: " + ", ".join(f"{k} {v:.2e}" for k, v in res.items()))


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
def test_attention_bwd_rejects_more_than_640_tokens(dtype):
    from omnidata_b200 import _capi, bwd
    bufs, qkv, o, d_o, _, dqkv = _attention_buffers(1, 641, dtype, 7)
    lse = torch.zeros(1, 12, 641, device=dev()) if dtype == torch.bfloat16 else None
    n0 = _capi.launch_count()
    with pytest.raises(_capi.OdbError):
        bwd.attention_bwd(qkv, o, d_o, lse, dqkv)
    assert _capi.launch_count() == n0


def test_attention_bwd_rejects_bad_arguments():
    """The kernels address o, d_o, dqkv and lse from qkv's (b, T) alone: a mismatch is refused before any launch."""
    from omnidata_b200 import _capi, bwd
    bf, f32 = torch.bfloat16, torch.float32
    b, t = 2, 65
    mk = lambda *s, dt=bf: torch.zeros(*s, device=dev(), dtype=dt)
    qkv, o, d_o, lse, dqkv = mk(b, t, 2304), mk(b, t, 768), mk(b, t, 768), mk(b, 12, t, dt=f32), mk(b, t, 2304)
    bad = [
        dict(qkv=mk(b, t, 2304 + 64)),                 # not 3 * heads * 64 wide
        dict(qkv=mk(b * t, 2304)),                     # not [b, T, 3 * heads * 64]
        dict(qkv=mk(b, t, 4608)[..., :2304]),          # not contiguous
        dict(o=mk(b, t - 1, 768)), dict(o=mk(b, t, 768, dt=f32)), dict(o=mk(b, t, 1536)[..., :768]),
        dict(d_o=mk(b + 1, t, 768)), dict(d_o=mk(b, t, 768, dt=f32)),
        dict(dqkv=mk(b, t, 768)), dict(dqkv=mk(b, t + 1, 2304)), dict(dqkv=mk(b, t, 2304, dt=f32)),
        dict(lse=None), dict(lse=mk(b, 12, t - 1, dt=f32)), dict(lse=mk(b, 12, t)), dict(lse=mk(b, t, 12, dt=f32)),
    ]
    n0 = _capi.launch_count()
    for over in bad:
        a = dict(qkv=qkv, o=o, d_o=d_o, lse=lse, dqkv=dqkv)
        a.update(over)
        with pytest.raises(_capi.OdbError):
            bwd.attention_bwd(a["qkv"], a["o"], a["d_o"], a["lse"], a["dqkv"])
    assert _capi.launch_count() == n0
    q32 = mk(b, t, 2304, dt=f32)
    with pytest.raises(_capi.OdbError):                       # fp32: o / d_o / dqkv must be fp32 as well
        bwd.attention_bwd(q32, o, d_o, None, dqkv)
    assert _capi.launch_count() == n0


# ------------------------------------------------------------------------------------------ c. dgrad compositions
GRIDS = [(24, 24), (10, 15), (2, 3)]          # output grids of the stride-2 layer: inputs 48x48, 20x30, 4x6


def _zero_bias(n, dtype):
    """The engine's dgrad launches carry a zero fp32 bias in bf16 (it selects the straight-line epilogues), none in fp32."""
    return torch.zeros(n, device=dev()) if dtype == torch.bfloat16 else None


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("mode", ["same", "sym1"])
@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_stride2_input_grad(grid, mode, dtype):
    """train.parity_dgrad_operands + four conv_gemm launches into the parity planes of dx, as TrainEngine._dgrad_s2:
    each launch checked on its own operands, each writes exactly its plane, together all of dx == float64 autograd."""
    from omnidata_b200.train import parity_dgrad_operands
    h, w = grid
    B, c, n = 2, 64, 128
    g = gen(h * 100 + w + (mode == "sym1"))
    w4 = (torch.randn(n, c, 3, 3, generator=g, device=dev()) * 0.05).to(dtype)
    wb = w4.reshape(n, c, 9).permute(1, 2, 0).flip(1).reshape(c, 9 * n).contiguous()      # odb_pack_weight's dgrad layout
    dyb, dxb = Guarded(B * h * w * n, dtype, g), Guarded(B * 4 * h * w * c, dtype, g)
    dy, dx = dyb.contiguous(B, h, w, n), dxb.contiguous(B, 2 * h, 2 * w, c)
    dx.fill_(float("nan"))
    taus = []
    for (py, px), (wp, taps) in parity_dgrad_operands(wb, n, mode).items():
        bias = _zero_bias(c, dtype)
        taus.append(check_conv([dyb, dxb], [dy], taps, wp, dx[:, py::2, px::2, :], bias=bias, prefill_nan=False)["tau"])
    assert bool(torch.isfinite(dx).all())                     # every element written, by exactly one plane's launch
    xd = torch.zeros(B, c, 2 * h, 2 * w, dtype=torch.float64, device=dev(), requires_grad=True)
    y = F.conv2d(F.pad(xd, (0, 1, 0, 1)), w4.double(), stride=2) if mode == "same" else \
        F.conv2d(xd, w4.double(), stride=2, padding=1)
    gx, = torch.autograd.grad(y, (xd,), dy.double().permute(0, 3, 1, 2))
    gx = gx.permute(0, 2, 3, 1)
    r = rel(dx, gx)
    assert r <= REL_DGRAD[dtype], r
    print(f"stride-2 dgrad {mode} {grid} {dtype}: tau {max(taus):.2e}, rel-L2 vs autograd {r:.2e}")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_downsample_input_grad(grid, dtype):
    """The first bottleneck of a stride-2 stage: dt_in = 0; dt_in[:, ::2, ::2] = downsample dgrad; dt_in += conv1 dgrad
    (residual = out = dt_in) == float64 autograd of both 1x1 convolutions summed."""
    from omnidata_b200 import ops
    h, w = grid
    B, cin, cout, mid = 2, 256, 512, 128
    g = gen(h * 100 + w)
    wd = (torch.randn(cout, cin, generator=g, device=dev()) * 0.05).to(dtype)
    w1 = (torch.randn(mid, cin, generator=g, device=dev()) * 0.05).to(dtype)
    ddb, dy1b, db = Guarded(B * h * w * cout, dtype, g), Guarded(B * 4 * h * w * mid, dtype, g), Guarded(B * 4 * h * w * cin, dtype, g)
    dd, dy1, dt_in = ddb.contiguous(B, h, w, cout), dy1b.contiguous(B, 2 * h, 2 * w, mid), db.contiguous(B, 2 * h, 2 * w, cin)
    bufs = [ddb, dy1b, db]
    dt_in.zero_()
    wdT, w1T = wd.t().contiguous(), w1.t().contiguous()
    t1 = check_conv(bufs, [dd], ops.TAPS_1, wdT, dt_in[:, ::2, ::2, :], bias=_zero_bias(cin, dtype))["tau"]
    t2 = check_conv(bufs, [dy1], ops.TAPS_1, w1T, dt_in, bias=_zero_bias(cin, dtype), residual=dt_in, prefill_nan=False)["tau"]
    xd = torch.zeros(B, cin, 2 * h, 2 * w, dtype=torch.float64, device=dev(), requires_grad=True)
    yd = F.conv2d(xd, wd.double()[:, :, None, None], stride=2)
    y1 = F.conv2d(xd, w1.double()[:, :, None, None])
    gx, = torch.autograd.grad((yd * dd.double().permute(0, 3, 1, 2)).sum() + (y1 * dy1.double().permute(0, 3, 1, 2)).sum(), (xd,))
    r = rel(dt_in, gx.permute(0, 2, 3, 1))
    assert r <= REL_DGRAD[dtype], r
    print(f"downsample dgrad {grid} {dtype}: tau {max(t1, t2):.2e}, rel-L2 vs autograd {r:.2e}")


# ------------------------------------------------------------------------------------------ d. every engine geometry
SIZES = [(384, 384), (320, 480), (64, 96), (96, 1664)]


BACKBONES = ["vitb_rn50_384", "vitl16_384", "vitb16_384"]


def _model(backbone):
    from omnidata_b200 import synthetic
    from omnidata_b200.model import DPTDepthModel, state_dict_spec
    model = DPTDepthModel(backbone=backbone)
    model.load_state_dict(synthetic.make_state_dict(0, 1, spec=state_dict_spec(1, backbone=backbone)), strict=True)
    return model.to(dev())


def _record(backbone, size, precision, batch=2):
    """One TrainEngine forward + backward; the backward's conv_gemm / conv_wgrad / attention_bwd launches
    -> {geometry: count}, and the wgrad destinations the engine should have produced but did not."""
    from omnidata_b200 import bwd, ops
    from omnidata_b200.train import TrainEngine
    H, W = size
    model = _model(backbone)
    eng = TrainEngine(model.train(), precision)
    g = torch.Generator(device="cpu").manual_seed(H * 7 + W)
    eng.forward((torch.rand(batch, 3, H, W, generator=g) * 2 - 1).to(dev()))
    dout = torch.randn(batch, eng.C, H, W, generator=g).to(dev())
    geoms, wgrad_outs = {}, []
    conv0, wgrad0, attn0 = ops.conv_gemm, bwd.conv_wgrad, bwd.attention_bwd
    defaults = {"bias": None, "residual": None, "act": 0}

    def conv(views, taps, weight, out, **kw):
        extra = {k: v for k, v in kw.items() if k not in defaults}
        assert not extra, f"conv_gemm flags the replay does not model: {sorted(extra)}"
        ts = {f"v{i}": v for i, v in enumerate(views)}
        ts.update(weight=weight, out=out, bias=kw.get("bias"), residual=kw.get("residual"))
        key = ("conv", geometry(ts), tuple(map(tuple, taps)), kw.get("act", 0))
        geoms[key] = geoms.get(key, 0) + 1
        return conv0(views, taps, weight, out, **kw)

    def wgrad(views, taps, dy, out, accumulate=False):
        ts = {f"v{i}": v for i, v in enumerate(views)}
        ts.update(dy=dy, out=out)
        key = ("wgrad", geometry(ts), tuple(map(tuple, taps)), bool(accumulate))
        geoms[key] = geoms.get(key, 0) + 1
        wgrad_outs.append(out.data_ptr())
        return wgrad0(views, taps, dy, out, accumulate=accumulate)

    def attention(qkv, o, d_o, lse, dqkv, heads=12, scale=0.125):
        key = ("attn", geometry(dict(qkv=qkv, o=o, d_o=d_o, lse=lse, dqkv=dqkv)), (), (heads, scale))
        geoms[key] = geoms.get(key, 0) + 1
        return attn0(qkv, o, d_o, lse, dqkv, heads=heads, scale=scale)

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "conv_gemm", conv)
        mp.setattr(bwd, "conv_wgrad", wgrad)
        mp.setattr(bwd, "attention_bwd", attention)
        eng.backward(dout)
    torch.cuda.synchronize()
    # every layer's weight gradient, each readout's token and cls halves and (hybrid) the stem go through conv_wgrad
    dest = {(eng.gp_layer[L.key] if L.key in eng.gp_layer else eng.G[L.weight]).data_ptr(): L.key for L in eng.layers}
    missing = sorted(k for p, k in dest.items() if p not in wgrad_outs)
    expected_calls = len(eng.layers) + 2 * len(eng.readouts) + int(eng.hybrid)
    del eng, model
    torch.cuda.empty_cache()
    return geoms, missing, len(wgrad_outs), expected_calls


def _replay(key, seed, batch):
    kind, geom, taps, extra = key
    bufs, ts = materialize(geom, gen(seed))
    views = [ts[f"v{i}"] for i in range(4) if f"v{i}" in ts]
    if kind == "wgrad":
        return "wgrad", check_wgrad(bufs, views, list(taps), ts["dy"], ts["out"], extra, rel_scale=(batch / 2) ** 0.5)
    if kind == "conv":
        out, res = ts["out"], ts["residual"]
        return "dgrad", check_conv(bufs, views, list(taps), ts["weight"], out, bias=ts["bias"], residual=res,
                                   prefill_nan=not same_storage(res, out))
    heads, scale = extra
    return "attention", check_attention(bufs, ts["qkv"], ts["o"], ts["d_o"], ts["lse"], ts["dqkv"], heads, scale)


def _replay_recording(backbone, size, precision, batch=2):
    geoms, missing, n_wgrad, expected = _record(backbone, size, precision, batch)
    assert not missing and n_wgrad == expected, (missing, n_wgrad, expected)
    assert {k[0] for k in geoms} == {"conv", "wgrad", "attn"}
    worst = {}
    for i, key in enumerate(geoms):
        cls, res = _replay(key, i, batch)
        for m, v in res.items():
            worst[f"{cls} {m}"] = max(worst.get(f"{cls} {m}", 0.0), v)
    print(f"{backbone} batch {batch} {size} {precision}: {len(geoms)} distinct geometries of {sum(geoms.values())} "
          "launches; worst " + ", ".join(f"{k} {v:.2e}" for k, v in sorted(worst.items())))


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("size", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
@pytest.mark.parametrize("backbone", BACKBONES)
def test_every_engine_backward_geometry(backbone, size, precision):
    _replay_recording(backbone, size, precision)


@pytest.mark.parametrize("backbone", ["vitb_rn50_384", "vitl16_384"])
def test_train_benchmark_backward_geometry(backbone):
    """The backward the train benchmarks time (bench.py --config 4 for the hybrid, profiles/plain_vit_train.py for
    DPT-Large): batch 16, 384 x 384, bf16, where the planners pick their widest tiles and fewest splits."""
    _replay_recording(backbone, (384, 384), "bf16", batch=16)
