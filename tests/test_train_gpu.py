"""Backward of the network (train_depth.py:183-190: loss.backward() over DPTDepthModel) on the GPU box.

Checker: torch.autograd over the oracle's restatement of the reference forward (oracle/dpt_oracle.py::forward_fp32,
bit-identical to the unmodified reference module in the build container) with the same seeded weights, evaluated on
the GPU in FLOAT64 — the exact gradient of the reference arithmetic.  The reference's own fp32 autograd (torch library
kernels, TF32 off) is measured against the same truth as the yardstick: on this network it is 2.3e-3 away globally
(the ResNetV2 GroupNorm chain is ill-conditioned in fp32).  Gradients of ALL 368 parameter tensors are compared:
  * precision='fp32' (FP32-pipe twins of every backward kernel, partial sums combined in fp64): global rel-L2 <= 5e-4
    (measured 1.6e-4), every tensor <= 5e-3 (measured max 2.2e-3), and closer to the truth than torch's fp32 autograd;
  * precision='bf16' (wgmma dgrad / wgrad / attention backward): the orchestration is the SAME code as the fp32 mode
    (verified above) and every bf16 kernel is verified on its own against float64 on identical inputs at every geometry
    the engine launches (tests/test_bwd_gemm_gpu.py).  End to end, a bf16 forward moves ~3 % of the activations that sit
    next to a ReLU threshold to the other side (the final ReLU alone: forward drift 3.8e-2), so ANY bf16 pipeline's
    gradient differs from the exact one by O(sqrt(fraction flipped)): measured against the float64 truth, stock
    torch.autocast(bfloat16) training of the same network is 0.141 away globally (0.44 on the ResNetV2 tensors, ~0.11
    on the ViT / decoder tensors), this pipeline 0.202 (0.44 / ~0.18; it stores bf16 where autocast keeps fp32 GroupNorm
    outputs).  Committed bounds: global <= 0.26, cosine >= 0.975, every tensor <= 0.6, and <= 1.6 x the stock-autocast
    error measured live in the same test.
Per-kernel backward tests compare each backward kernel with torch.autograd of the same op in float64."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev())


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


# ------------------------------------------------------------------------------------------ kernels (fp32 storage)
def test_layernorm_bwd_kernel():
    for c in (256, 512, 768, 1024):                          # the kernel's four instances (VPL = c / 256)
        _check_layernorm_bwd(c)


def _check_layernorm_bwd(c):
    from omnidata_b200 import bwd
    rows = 4 * 577
    x, dy, g, ds_in = rnd(rows, c) * 2 + 0.3, rnd(rows, c, seed=1), rnd(c) * 0.1 + 1, rnd(rows, c, seed=2)
    xd = x.double().requires_grad_(True); gd = g.double().requires_grad_(True); bd = torch.zeros(c, device=dev(), dtype=torch.float64, requires_grad=True)
    y = F.layer_norm(xd, (c,), gd, bd, 1e-6)
    gx, gg, gb = torch.autograd.grad(y, (xd, gd, bd), dy.double())
    ds_out, dgam, dbet = torch.empty_like(x), torch.empty(c, device=dev()), torch.empty(c, device=dev())
    bwd.layernorm_bwd(dy, x, g, ds_in, ds_out, None, dgam, dbet)
    torch.cuda.synchronize()
    assert rel(ds_out, gx + ds_in.double()) < 1e-5 and rel(dgam, gg) < 1e-5 and rel(dbet, gb) < 1e-5
    # with the fused column sums of ds_out (bias gradient of the linear layer in front): same results + the sums
    ds2, dgam2, dbet2, dcol = torch.empty_like(x), torch.empty(c, device=dev()), torch.empty(c, device=dev()), torch.empty(c, device=dev())
    bwd.layernorm_bwd(dy, x, g, ds_in, ds2, None, dgam2, dbet2, dcolsum=dcol)
    torch.cuda.synchronize()
    assert torch.equal(ds2, ds_out) and torch.equal(dgam2, dgam) and torch.equal(dbet2, dbet)
    assert rel(dcol, ds_out.double().sum(0)) < 1e-5
    # accumulate: every parameter output adds to what is there
    bwd.layernorm_bwd(dy, x, g, ds_in, ds2, None, dgam2, dbet2, accumulate=True, dcolsum=dcol)
    torch.cuda.synchronize()
    assert rel(dgam2, 2 * gg) < 1e-5 and rel(dbet2, 2 * gb) < 1e-5 and rel(dcol, 2 * ds_out.double().sum(0)) < 1e-5
    # a row count that does not fill the grid (fewer rows than warps)
    bwd.layernorm_bwd(dy[:5], x[:5], g, None, ds2[:5], None, dgam2, dbet2, dcolsum=dcol)
    torch.cuda.synchronize()
    y5 = F.layer_norm(xd[:5], (c,), gd, bd, 1e-6)
    gx5, gg5 = torch.autograd.grad(y5, (xd, gd), dy[:5].double())
    assert rel(ds2[:5], gx5[:5]) < 1e-5 and rel(dgam2, gg5) < 1e-5 and rel(dcol, gx5[:5].sum(0)) < 1e-5
    # bf16 incoming gradient + bf16 copy of the result
    dyb = dy.to(torch.bfloat16)
    cp = torch.empty(rows, c, device=dev(), dtype=torch.bfloat16)
    bwd.layernorm_bwd(dyb, x, g, None, ds_out, cp, dgam, dbet)
    torch.cuda.synchronize()
    gx2, = torch.autograd.grad(F.layer_norm(xd, (c,), gd, bd, 1e-6), (xd,), dyb.double())
    assert rel(ds_out, gx2) < 1e-5 and torch.equal(cp, ds_out.to(torch.bfloat16))


@pytest.mark.parametrize("c,hw", [(64, 48 * 48), (256, 24 * 24), (1024, 144)])
def test_groupnorm_bwd_kernel(c, hw):
    from omnidata_b200 import bwd, ops
    b = 3
    x, dy = rnd(b, hw, c) * 2 + 0.3, rnd(b, hw, c, seed=1)
    g, bt = rnd(c) * 0.1 + 1, rnd(c) * 0.1
    st = torch.empty(b, 32, 2, device=dev()); ops.groupnorm_stats(x, st)
    xd = x.double().transpose(1, 2).requires_grad_(True); gd = g.double().requires_grad_(True); bd = bt.double().requires_grad_(True)
    y = F.relu(F.group_norm(xd, 32, gd, bd, 1e-5))
    gx, gg, gb = torch.autograd.grad(y, (xd, gd, bd), dy.double().transpose(1, 2))
    out = torch.empty_like(x); ops.groupnorm_apply(x, st, g, bt, out, relu=True)
    dx, dgam, dbet = torch.empty_like(x), torch.empty(c, device=dev()), torch.empty(c, device=dev())
    bwd.groupnorm_bwd(dy, x, st, g, dx, dgam, dbet, mask=out)
    torch.cuda.synchronize()
    assert rel(dx, gx.transpose(1, 2)) < 2e-5 and rel(dgam, gg) < 2e-5 and rel(dbet, gb) < 2e-5


def test_elementwise_bwd_kernels():
    from omnidata_b200 import bwd
    # GELU
    u, dy = rnd(1000, 768) * 2, rnd(1000, 768, seed=1)
    ud = u.double().requires_grad_(True)
    gu, = torch.autograd.grad(F.gelu(ud), (ud,), dy.double())
    y, du = torch.empty_like(u), torch.empty_like(u)
    bwd.gelu_fwd(u, y); bwd.gelu_bwd(dy, u, du)
    torch.cuda.synchronize()
    assert rel(y, F.gelu(u.double())) < 1e-6 and rel(du, gu) < 1e-6
    # mask_add
    a, b_, m = rnd(64, 256), rnd(64, 256, seed=1), rnd(64, 256, seed=2)
    out = torch.empty_like(a)
    bwd.mask_add(out, b_, a=a, mask=m)
    torch.cuda.synchronize()
    assert torch.equal(out, a + b_ * (m > 0))
    # bilinear x2 adjoint
    z, dout = rnd(2, 12, 20, 64), rnd(2, 24, 40, 64, seed=3)
    zd = z.double().permute(0, 3, 1, 2).requires_grad_(True)
    up = F.interpolate(zd, scale_factor=2, mode="bilinear", align_corners=True)
    gz, = torch.autograd.grad(up, (zd,), dout.double().permute(0, 3, 1, 2))
    dz = torch.empty_like(z)
    bwd.upsample2x_bwd(dout, dz)
    torch.cuda.synchronize()
    assert rel(dz, gz.permute(0, 2, 3, 1)) < 1e-6
    # column sums
    x = rnd(3, 577, 768)
    o1, o2 = torch.empty(1, 768, device=dev()), torch.empty(3, 768, device=dev())
    bwd.colsum(x.view(-1, 768), o1); bwd.colsum(x[:, 1:, :], o2, batches=3)
    torch.cuda.synchronize()
    assert rel(o1[0], x.double().sum((0, 1))) < 1e-6 and rel(o2, x[:, 1:].double().sum(1)) < 1e-6
    # many rows x few columns (a decoder convolution's output gradient, bf16: many slabs, ragged unroll tail), accumulate,
    # and a handful of rows x many columns (pos_embed: one slab)
    xb = rnd(40013, 64, seed=3).to(torch.bfloat16)
    o3 = torch.full((1, 64), 2.0, device=dev())
    bwd.colsum(xb, o3, accumulate=True)
    xw = rnd(3, 577 * 768, seed=4)
    o4 = torch.empty(1, 577 * 768, device=dev())
    bwd.colsum(xw, o4)
    torch.cuda.synchronize()
    assert rel(o3[0], xb.double().sum(0) + 2.0) < 1e-6 and rel(o4[0], xw.double().sum(0)) < 1e-6


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_pack_table_multi(dtype):
    """One-launch packing of several layers == the layer-by-layer definition (forward operand, rotated / transposed
    dgrad operand, weight standardisation, zero padding); covers the vector paths and the odd-extent fallback."""
    from omnidata_b200 import bwd
    specs = [  # n, c, taps, n_pad, c_pad, standardize
        (100, 768, 1, 128, 768, False),      # linear layer: float4 path, padded rows
        (64, 64, 9, 64, 64, True),           # 3x3 with weight standardisation
        (256, 64, 1, 256, 64, True),         # 1x1 with weight standardisation (vector path + statistics)
        (24, 40, 9, 64, 64, False),          # padded channels both ways
        (33, 35, 1, 33, 35, False),          # odd extents: scalar paths
    ]
    layers, refs = [], []
    for i, (n, c, taps, n_pad, c_pad, std) in enumerate(specs):
        w = rnd(n, c, taps, scale=0.05, seed=10 + i) + 0.01
        fwd = torch.full((n_pad, taps * c_pad), 7.0, device=dev()).to(dtype)
        bk = torch.full((c_pad, taps * n_pad), 7.0, device=dev()).to(dtype)
        layers.append((w, fwd, bk, n, c, taps, n_pad, c_pad, std))
        wh = w.double()
        if std:
            m = wh.mean(dim=(1, 2), keepdim=True)
            sd = (wh.var(dim=(1, 2), unbiased=False, keepdim=True)).sqrt()
            wh = (wh - m) / (sd + 1e-8)
        rf = torch.zeros(n_pad, taps, c_pad, dtype=torch.float64, device=dev())
        rf[:n, :, :c] = wh.permute(0, 2, 1)
        rb = torch.zeros(c_pad, taps, n_pad, dtype=torch.float64, device=dev())
        rb[:c, :, :n] = wh.permute(1, 2, 0).flip(1)
        refs.append((rf.reshape(n_pad, -1), rb.reshape(c_pad, -1)))
    bwd.PackTable(layers, dtype).run()
    torch.cuda.synchronize()
    tol = 1e-6 if dtype == torch.float32 else 4e-3
    for (w, fwd, bk, *_), (rf, rb) in zip(layers, refs):
        assert rel(fwd, rf) < tol and rel(bk, rb) < tol
        assert torch.equal(fwd == 0, rf == 0) and torch.equal(bk == 0, rb == 0)          # padding is exactly zero
        # the transposed operand holds exactly the forward operand's rounded values
        n_pad, c_pad = fwd.shape[0], bk.shape[0]
        taps = fwd.shape[1] // c_pad
        assert torch.equal(bk.view(c_pad, taps, n_pad), fwd.view(n_pad, taps, c_pad).permute(2, 1, 0).flip(1))


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("backbone", ["vitb_rn50_384", "vitl16_384", "vitb16_384"])
def test_engine_and_inference_operand_tables_agree(backbone, precision):
    """The train engine and inference hand dpt_forward operand tables with the same keys, shapes and dtypes, but for the
    documented differences: head conv2 (operand and bias) padded to 64 rows in training, the ConvTransposes' table
    operands (engine only; inference reads their per-phase operands), the dead refinenet4.resConfUnit1 (inference
    only)."""
    from omnidata_b200.model import DPTDepthModel
    from omnidata_b200.train import TrainEngine
    model = DPTDepthModel(backbone=backbone).to(dev())
    model.precision = precision
    inf = model._prepack(dev())
    eng = TrainEngine(model, precision).pk
    spec = lambda table: {k: (tuple(t.shape), t.dtype) for k, t in table.items()}
    adt = torch.float32 if precision == "fp32" else torch.bfloat16
    g_eng, g_inf = spec(eng["gemm"]), spec(inf["gemm"])
    assert g_eng.pop("head2") == ((64, 9 * 128), adt) and g_inf.pop("head2") == ((32, 9 * 128), adt)
    for cv in (1, 2):
        assert g_inf.pop(f"ff4.rcu1.c{cv}") == ((256, 9 * 256), adt)
    if not model.arch["hybrid"]:
        for n in (1, 2):
            assert g_eng.pop(f"pp{n}t")[1] == adt
    assert g_eng == g_inf and all(dt == adt for _, dt in g_eng.values())
    v_eng, v_inf = spec(eng["vec"]), spec(inf["vec"])
    b2 = "scratch.output_conv.2.bias"
    assert v_eng.pop(b2) == ((64,), torch.float32) and v_inf.pop(b2) == ((32,), torch.float32)
    for cv in (1, 2):
        assert v_inf.pop(f"scratch.refinenet4.resConfUnit1.conv{cv}.bias") == ((256,), torch.float32)
    assert v_eng == v_inf and all(dt == torch.float32 for _, dt in v_eng.values())


def test_stem_and_head_bwd_kernels():
    from omnidata_b200 import bwd, ops
    b, h, w, c = 2, 32, 48, 64
    s0, dt = rnd(b, h, w, c) * 2, rnd(b, h // 2, w // 2, c, seed=1)
    g, bt = rnd(c) * 0.1 + 1, rnd(c) * 0.1
    st = torch.empty(b, 32, 2, device=dev()); ops.groupnorm_stats(s0, st)
    xd = s0.double().permute(0, 3, 1, 2).requires_grad_(True)
    gn = F.group_norm(xd, 32, g.double(), bt.double(), 1e-5)
    gn.retain_grad()
    t = F.max_pool2d(F.pad(F.relu(gn), (0, 1, 0, 1), value=float("-inf")), 3, 2)
    t.backward(dt.double().permute(0, 3, 1, 2))
    g_s0 = torch.empty_like(s0)
    bwd.stem_pool_bwd(dt, s0, st, g, bt, g_s0)
    torch.cuda.synchronize()
    assert rel(g_s0, gn.grad.permute(0, 2, 3, 1)) < 1e-5
    # head tail
    a = rnd(2, 16, 24, 64).abs(); a[..., 32:] = 0
    w4, b4, dout = rnd(1, 32, scale=0.2), rnd(1) + 0.5, rnd(2, 1, 16, 24, seed=5)
    out = torch.empty(2, 1, 16, 24, device=dev())
    bwd.head_tail_fwd(a, w4, b4, out, True)
    ad = a[..., :32].double().requires_grad_(True); wd = w4.double().requires_grad_(True); bd = b4.double().requires_grad_(True)
    ref = F.relu(torch.einsum("bhwj,kj->bkhw", F.relu(ad), wd) + bd[None, :, None, None])
    ga, gw, gb = torch.autograd.grad(ref, (ad, wd, bd), dout.double())
    da, dw, db = torch.empty_like(a), torch.empty(1, 32, device=dev()), torch.empty(1, device=dev())
    bwd.head_tail_bwd(dout, out, a, w4, da, dw, db, True)
    torch.cuda.synchronize()
    assert rel(out, ref) < 1e-5 and rel(da[..., :32], ga) < 1e-5 and rel(dw, gw) < 1e-5 and rel(db, gb) < 1e-5
    assert float(da[..., 32:].abs().max()) == 0.0


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-5), (torch.bfloat16, 3e-3)])
def test_conv_wgrad_and_pack(dtype, tol):
    from omnidata_b200 import bwd, ops
    b, h, w_, c, n = 2, 24, 32, 64, 128
    x, dy = rnd(b, h, w_, c).to(dtype), rnd(b, h, w_, n, seed=1).to(dtype)
    wt = rnd(n, c, 3, 3, scale=0.05)
    # 3x3 stride 1
    xd = x.double().permute(0, 3, 1, 2); wd = wt.double().requires_grad_(True)
    gw, = torch.autograd.grad(F.conv2d(xd, wd, padding=1), (wd,), dy.double().permute(0, 3, 1, 2))
    gp = torch.empty(n, 9 * c, device=dev())
    bwd.conv_wgrad([x], bwd.TAPS_3X3, dy, gp)
    dw = torch.empty_like(wt)
    bwd.unpack_wgrad(gp, wt, dw, n, c, 9, c, False)
    torch.cuda.synchronize()
    assert rel(dw, gw) < tol
    # stride 2 (TF-SAME) through parity planes, with weight standardisation in the chain
    def std(w):
        s, m = torch.std_mean(w, dim=[1, 2, 3], keepdim=True, unbiased=False)
        return (w - m) / (s + 1e-8)
    dy2 = rnd(b, h // 2, w_ // 2, n, seed=2).to(dtype)
    wd2 = wt.double().requires_grad_(True)
    y2 = F.conv2d(F.pad(xd, (0, 1, 0, 1)), std(wd2), stride=2)
    gw2, = torch.autograd.grad(y2, (wd2,), dy2.double().permute(0, 3, 1, 2))
    planes = [x[:, py::2, px::2, :] for py in range(2) for px in range(2)]
    bwd.conv_wgrad(planes, ops._parity_taps("same"), dy2, gp)
    bwd.unpack_wgrad(gp, wt, dw, n, c, 9, c, True)
    torch.cuda.synchronize()
    assert rel(dw, gw2) < tol
    # pack: forward operand == pack_conv_weight(std(w)), dgrad operand reproduces conv_transpose
    fwd = torch.empty(n, 9 * c, device=dev(), dtype=dtype); bk = torch.empty(c, 9 * n, device=dev(), dtype=dtype)
    bwd.pack_weight(wt, fwd, bk, n, c, 9, n, c, True)
    torch.cuda.synchronize()
    assert rel(fwd.float(), ops.pack_conv_weight(std(wt), torch.float32)) < (1e-6 if dtype == torch.float32 else 4e-3)
    dx = torch.empty_like(x)
    ops.conv3x3(dy, bk, dx)
    xg = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    gx, = torch.autograd.grad(F.conv2d(xg, std(wt).double(), padding=1), (xg,), dy.double().permute(0, 3, 1, 2))
    torch.cuda.synchronize()
    assert rel(dx.float(), gx.permute(0, 2, 3, 1)) < (1e-5 if dtype == torch.float32 else 6e-3)


# ------------------------------------------------------------------------------------------ whole network
def _reference_grads(sd, x, R, dtype=torch.float64):
    """torch.autograd over the reference arithmetic (oracle restatement) on the GPU; float64 = the exact gradient."""
    from oracle import dpt_oracle
    leaves = {k: v.to(dev()).to(dtype).requires_grad_(True) for k, v in sd.items()}
    y = dpt_oracle.forward_fp32(leaves, x.to(dev()), dtype=dtype)
    loss = (y * R.to(dtype)).sum()
    grads = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
    return y.detach(), {k: (g if g is not None else torch.zeros_like(leaves[k])) for k, g in zip(leaves, grads)}


def _engine_grads(sd, x, R, precision):
    from omnidata_b200.model import DPTDepthModel
    model = DPTDepthModel(backbone="vitb_rn50_384")
    model.load_state_dict(sd, strict=True)
    model = model.to(dev()).train()
    model.precision = precision
    for p in model.parameters():
        p.grad = None
    y = model(x.to(dev()))                     # train() mode under autograd -> differentiable forward
    assert y.requires_grad
    loss = (y * R).sum()
    loss.backward()
    return y.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}


@pytest.fixture(scope="module")
def grads_case():
    from oracle import make_golden, weights
    sd = weights.make_state_dict(0, 1)
    x = make_golden.golden_input(1, seed=0)
    g = torch.Generator(device="cpu").manual_seed(123)
    R = torch.randn(1, 384, 384, generator=g).to(dev())
    y_ref, g_ref = _reference_grads(sd, x, R)
    _, g_ref32 = _reference_grads(sd, x, R, torch.float32)
    return sd, x, R, y_ref, g_ref, g_ref32


def _compare(g_ref, g_mine, per_tensor_tol, global_tol, min_cos):
    worst, num, den, dot, n1, n2 = [], 0.0, 0.0, 0.0, 0.0, 0.0
    assert set(g_ref) == set(g_mine) and len(g_ref) == 368
    for k, gr in g_ref.items():
        gm = g_mine[k].double()
        gr = gr.double()
        if float(gr.norm()) == 0.0:            # dead parameters (timm classifier head / final norm, refinenet4.resConfUnit1)
            assert float(gm.norm()) == 0.0, k
            continue
        e = float((gm - gr).norm() / gr.norm())
        worst.append((e, k))
        num += float((gm - gr).pow(2).sum()); den += float(gr.pow(2).sum())
        dot += float((gm * gr).sum()); n1 += float(gm.pow(2).sum()); n2 += float(gr.pow(2).sum())
    worst.sort(reverse=True)
    glob, cos = (num / den) ** 0.5, dot / (n1 * n2) ** 0.5
    print(f"global rel-L2 {glob:.3e}, cosine {cos:.6f}; worst tensors: " + ", ".join(f"{k} {e:.2e}" for e, k in worst[:6]))
    assert glob <= global_tol and cos >= min_cos, (glob, cos)
    assert worst[0][0] <= per_tensor_tol, worst[:6]
    return glob


def test_network_backward_fp32_mode_matches_autograd_of_the_reference(grads_case):
    sd, x, R, y_ref, g_ref, g_ref32 = grads_case
    y, g = _engine_grads(sd, x, R, "fp32")
    assert rel(y, y_ref) <= 1e-5
    _compare(g_ref, g, per_tensor_tol=5e-3, global_tol=5e-4, min_cos=0.999999)
    # for the record: torch's own fp32 autograd against the same truth (cuDNN algorithm choice makes it vary between
    # 1e-6 and 2.3e-3 from run to run on this network; not asserted)
    _compare(g_ref, g_ref32, per_tensor_tol=1.0, global_tol=1.0, min_cos=0.0)


def test_network_backward_bf16_mode(grads_case):
    from oracle import dpt_oracle
    sd, x, R, y_ref, g_ref, g_ref32 = grads_case
    y, g = _engine_grads(sd, x, R, "bf16")
    mine = _compare(g_ref, g, per_tensor_tol=0.6, global_tol=0.26, min_cos=0.975)
    # the bf16 yardstick: stock torch.autocast training of the reference arithmetic on the same GPU / weights / input
    leaves = {k: v.to(dev()).float().requires_grad_(True) for k, v in sd.items()}
    with torch.autocast("cuda", dtype=torch.bfloat16):
        yac = dpt_oracle.forward_fp32(leaves, x.to(dev()))
    gac = torch.autograd.grad((yac.float() * R).sum(), list(leaves.values()), allow_unused=True)
    g_ac = {k: (gg if gg is not None else torch.zeros_like(leaves[k])) for k, gg in zip(leaves, gac)}
    stock = _compare(g_ref, g_ac, per_tensor_tol=10.0, global_tol=10.0, min_cos=0.0)
    assert mine <= 1.6 * stock, (mine, stock)
    y2, g2 = _engine_grads(sd, x, R, "bf16")
    assert all(torch.equal(g[k], g2[k]) for k in g)            # deterministic: fixed-order reductions everywhere


# ------------------------------------------------------------------------------------------ loss mix + train step
def test_depth_step_loss_matches_the_autograd_path():
    """DepthStepLoss (sync-free launch sequence of the train step) == depth_step_losses under torch.autograd (which is
    pinned to the reference modules in tests/test_losses_gpu.py): values and d loss / d pred."""
    import numpy as np
    from omnidata_b200 import losses
    from oracle import loss_oracle
    pred, gt, mf = (t.to(dev()) for t in loss_oracle.loss_inputs(0))
    pred = (pred * 1.3 - 0.1).contiguous()                      # some values outside [0, 1]: the clamp matters
    midas, vnl = losses.MidasLoss(0.1, 4), losses.VNL_Loss(1.0, 1.0, (384, 384))
    np.random.seed(3)
    pts = vnl.select_index()
    p = pred.clone().requires_grad_(True)
    pc = torch.clamp(p, 0, 1)
    mask = losses.make_valid_mask(mf)
    _, ssi, reg = midas(pc, gt, mask)
    vn = vnl(pc, gt, points=pts)
    loss = ssi + 0.1 * reg + 10 * vn
    loss.backward()
    fn = losses.DepthStepLoss((384, 384))
    out, dpred = fn(pred, gt, mf, full_mix=True, points=pts)
    torch.cuda.synchronize()
    assert rel(out[0], loss.detach()) < 1e-6 and rel(out[1], ssi.detach()) < 1e-6 and rel(out[3], vn.detach()) < 1e-6
    assert rel(dpred, p.grad) < 1e-6
    out1, dpred1 = fn(pred, gt, mf, full_mix=False)
    p2 = pred.clone().requires_grad_(True)
    _, ssi2, _ = midas(torch.clamp(p2, 0, 1), gt, mask)
    ssi2.backward()
    torch.cuda.synchronize()
    assert rel(out1[0], ssi2.detach()) < 1e-6 and rel(dpred1, p2.grad) < 1e-6


def test_train_step_runs_learns_and_is_deterministic():
    """configs[4] on one GPU at a small batch: three optimizer steps on a fixed batch lower the loss, the flat master
    weights move, every number is finite, and two identical runs are bit-identical."""
    import numpy as np
    from omnidata_b200 import synthetic
    from omnidata_b200.model import DPTDepthModel
    from omnidata_b200.train import DepthTrainStep
    # Adam's first step moves every weight by lr: at lr 1e-4 that sign step drives this seeded synthetic network's
    # output to zero in the fp32 mode as well (measured on an H100), after which the virtual-normal loss is undefined;
    # at 1e-6 three steps lower the loss in both precisions
    LR = 1e-6
    g = torch.Generator(device="cpu").manual_seed(9)
    rgb = (torch.rand(2, 3, 384, 384, generator=g) * 2 - 1).to(dev())
    gt = torch.rand(2, 1, 384, 384, generator=g).to(dev())
    mask = (torch.rand(2, 1, 384, 384, generator=g) > 0.1).float().to(dev())
    runs = []
    for _ in range(2):
        model = DPTDepthModel()
        model.load_state_dict(synthetic.make_state_dict(0, 1), strict=True)
        model = model.to(dev()).train()
        step = DepthTrainStep(model, lr=LR, clip=10.0, precision="bf16")
        w0 = step.engine.flat.clone()
        np.random.seed(11)
        hist = [step.step(rgb, gt, mask, full_mix=True).cpu() for _ in range(3)]
        torch.cuda.synchronize()
        runs.append((hist, step.engine.flat.clone()))
        assert all(torch.isfinite(h).all() for h in hist)
        assert float(hist[-1][0]) < float(hist[0][0])               # the loss goes down on the fixed batch
        assert float((step.engine.flat - w0).abs().max()) > 0
        assert float(hist[0][4]) > 0                                # gradient norm
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0])) and torch.equal(runs[0][1], runs[1][1])
    # the same three steps replayed as ONE CUDA graph (the eager step is host-bound): bit-identical losses, gradient
    # norms, weights and optimizer state — including the capture's warm-up step being undone; then a change of the loss
    # mix (a second graph over the same buffers) and new inputs through the static copies
    model = DPTDepthModel()
    model.load_state_dict(synthetic.make_state_dict(0, 1), strict=True)
    model = model.to(dev()).train()
    step = DepthTrainStep(model, lr=LR, clip=10.0, precision="bf16")
    step.use_cuda_graph = True
    np.random.seed(11)
    hist = [step.step(rgb, gt, mask, full_mix=True).cpu() for _ in range(3)]
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(hist, runs[0][0])) and torch.equal(step.engine.flat, runs[0][1])
    assert step.opt.step_count == 3 and step.global_step == 3 and len(step._graphs) == 1
    ref = DepthTrainStep(DPTDepthModel().to(dev()).train(), lr=LR, clip=10.0, precision="bf16")
    ref.engine.flat.copy_(step.engine.flat); ref.opt.exp_avg.copy_(step.opt.exp_avg); ref.opt.exp_avg_sq.copy_(step.opt.exp_avg_sq)
    ref.opt.step_count = 3
    rgb2, gt2 = rgb.flip(0).contiguous(), gt.flip(0).contiguous()
    a = [step.step(rgb2, gt2, mask, full_mix=False).cpu(), step.step(rgb, gt, mask, full_mix=False).cpu()]
    b = [ref.step(rgb2, gt2, mask, full_mix=False).cpu(), ref.step(rgb, gt, mask, full_mix=False).cpu()]
    torch.cuda.synchronize()
    assert len(step._graphs) == 2
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and torch.equal(step.engine.flat, ref.engine.flat)
