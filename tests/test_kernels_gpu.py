"""Per-kernel numerics: each CUDA kernel (called through the C ABI) against a plain PyTorch fp32
evaluation of the same op on the same bf16 inputs.  Tolerance: rel-L2 <= 1e-3 against the fp32
result rounded to bf16 (the kernels compute bf16 x bf16 -> fp32 accumulate -> one bf16 rounding)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 1e-3


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def dev():
    return torch.device("cuda:0")


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dev())


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def check(out, ref_fp32, name, tol=TOL):
    ref = ref_fp32.to(torch.bfloat16).float()
    err = rel_l2(out.float(), ref)
    maxabs = float((out.float() - ref).abs().max())
    assert math.isfinite(err) and err <= tol, f"{name}: rel-L2 {err:.3e} (max abs {maxabs:.3e}) > {tol}"


def ops():
    from omnidata_b200 import ops as o
    return o


@pytest.mark.parametrize("m,k,n,block_n", [
    (300, 64, 64, 64), (128, 128, 64, 64), (1000, 768, 768, 0), (1000, 768, 768, 256), (1000, 768, 768, 128),
    (577 * 4, 768, 2304, 0), (2000, 3072, 768, 0), (333, 160, 64, 64), (40000, 768, 768, 256), (20000, 256, 512, 0),
])
def test_linear_plain(m, k, n, block_n):
    o = ops()
    x = rnd(m, k).to(torch.bfloat16)
    w = rnd(n, k, scale=k ** -0.5).to(torch.bfloat16)
    out = torch.full((m, n), float("nan"), device=dev(), dtype=torch.bfloat16)
    o.linear(x, w, out, block_n=block_n)
    torch.cuda.synchronize()
    check(out, x.float() @ w.float().t(), f"linear {m}x{k}x{n} bn{block_n}")


@pytest.mark.parametrize("m,k,n", [(300, 64, 256), (1000, 768, 768), (577 * 32, 768, 2304), (5000, 3072, 768),
                                   (128 * 3, 256, 512)])
def test_linear_cta_pair(m, k, n):
    """CTA pairs: a 2-CTA cluster shares the weight tile by TMA multicast (odd tile counts included)."""
    o = ops()
    x = rnd(m, k).to(torch.bfloat16)
    w = rnd(n, k, scale=k ** -0.5).to(torch.bfloat16)
    bias = rnd(n)
    res = rnd(m, n, seed=11).to(torch.bfloat16)
    out = torch.full((m, n), float("nan"), device=dev(), dtype=torch.bfloat16)
    o.linear(x, w, out, bias=bias, residual=res, act=o.ACT_GELU, block_n=256, cta_pair=1)
    torch.cuda.synchronize()
    check(out, F.gelu(x.float() @ w.float().t() + bias) + res.float(), f"pair linear {m}x{k}x{n}")
    single = torch.empty_like(out)
    o.linear(x, w, single, bias=bias, residual=res, act=o.ACT_GELU, block_n=256, cta_pair=-1)
    torch.cuda.synchronize()
    assert torch.equal(out, single)          # same accumulation order => bit-identical to the 1-CTA kernel


@pytest.mark.parametrize("b,h,w_", [(2, 48, 48), (3, 24, 24), (1, 96, 96)])
def test_conv3x3_cta_pair(b, h, w_):
    o = ops()
    c = 256
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    skip = rnd(b, h, w_, c, seed=5).to(torch.bfloat16)
    w = rnd(c, c, 3, 3, scale=(9 * c) ** -0.5).to(torch.bfloat16)
    bias = rnd(c)
    out = torch.full((b, h, w_, c), float("nan"), device=dev(), dtype=torch.bfloat16)
    out2 = torch.empty_like(out)
    o.conv3x3(x, o.pack_conv_weight(w), out, bias=bias, residual=skip, out2=out2, block_n=256, cta_pair=1)
    torch.cuda.synchronize()
    ref = conv_ref(x, w) + bias + skip.float()
    check(out, ref, "pair conv3x3 residual")
    check(out2, F.relu(ref), "pair conv3x3 relu copy")


@pytest.mark.parametrize("act", [0, 1, 2])
def test_linear_epilogue(act):
    o = ops()
    m, k, n = 1500, 768, 1024
    x = rnd(m, k).to(torch.bfloat16)
    w = rnd(n, k, scale=k ** -0.5).to(torch.bfloat16)
    bias = rnd(n)
    res = rnd(m, n).to(torch.bfloat16)
    out = torch.empty((m, n), device=dev(), dtype=torch.bfloat16)
    out2 = torch.empty_like(out)
    o.linear(x, w, out, bias=bias, residual=res, act=act, out2=out2)
    torch.cuda.synchronize()
    v = x.float() @ w.float().t() + bias
    v = [v, F.relu(v), F.gelu(v)][act] + res.float()
    check(out, v, f"linear epilogue act{act}")
    check(out2, F.relu(v), f"linear epilogue act{act} relu copy")


def conv_ref(x, w, stride=1, padding=1):
    """x [B,H,W,C] bf16, w [N,C,kh,kw] bf16 -> [B,Ho,Wo,N] fp32."""
    y = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), stride=stride, padding=padding)
    return y.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("b,h,w_,c,n,tile", [
    (2, 24, 24, 64, 128, None), (2, 48, 48, 256, 256, None), (1, 96, 96, 64, 64, None), (3, 12, 12, 128, 256, None),
    (1, 24, 24, 768, 256, (8, 16)), (1, 192, 192, 64, 128, (32, 4)),
])
def test_conv3x3(b, h, w_, c, n, tile):
    o = ops()
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    w = rnd(n, c, 3, 3, scale=(9 * c) ** -0.5).to(torch.bfloat16)
    bias = rnd(n)
    out = torch.full((b, h, w_, n), float("nan"), device=dev(), dtype=torch.bfloat16)
    o.conv3x3(x, o.pack_conv_weight(w), out, bias=bias, act=o.ACT_RELU, tile=tile)
    torch.cuda.synchronize()
    check(out, F.relu(conv_ref(x, w) + bias), f"conv3x3 {b}x{h}x{w_}x{c}->{n}")


@pytest.mark.parametrize("b,h,w_,c,n,bn,pair", [
    (2, 96, 96, 64, 64, 0, 0), (2, 48, 48, 256, 256, 0, 0), (3, 24, 24, 768, 256, 0, 0), (2, 12, 12, 256, 256, 0, 0),
    (1, 192, 192, 128, 128, 0, 0), (1, 384, 384, 64, 64, 0, 0), (2, 96, 96, 256, 256, 256, 1), (3, 48, 48, 256, 256, 256, 1),
    (2, 40, 56, 128, 128, 0, 0),
])
def test_conv3x3_halo_mode(b, h, w_, c, n, bn, pair, hmode=1):
    """Halo tiles (one input box per K block, nine shifted wgmma descriptors) == per-tap boxes."""
    o = ops()
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    skip = rnd(b, h, w_, n, seed=5).to(torch.bfloat16)
    w = rnd(n, c, 3, 3, scale=(9 * c) ** -0.5).to(torch.bfloat16)
    bias = rnd(n)
    wp = o.pack_conv_weight(w)
    out = torch.full((b, h, w_, n), float("nan"), device=dev(), dtype=torch.bfloat16)
    out2 = torch.full((b, h, w_, n), float("nan"), device=dev(), dtype=torch.bfloat16)
    partial = torch.empty((b * 1280 * 4 * 32 * 2,), device=dev())
    stats = torch.empty((b, 32, 2), device=dev())
    o.conv3x3(x, wp, out, bias=bias, residual=skip, out2=out2, halo=hmode, block_n=bn, cta_pair=pair,
              gn_stats=(partial, stats))
    torch.cuda.synchronize()
    ref = conv_ref(x, w) + bias + skip.float()
    check(out, ref, f"halo conv3x3 {b}x{h}x{w_}x{c}->{n}")
    check(out2, F.relu(ref), "halo conv3x3 relu copy")
    base = torch.empty_like(out)
    stats_b = torch.empty_like(stats)
    o.conv3x3(x, wp, base, bias=bias, residual=skip, halo=-1, block_n=bn, cta_pair=pair, gn_stats=(partial, stats_b))
    torch.cuda.synchronize()
    assert rel_l2(out.float(), base.float()) < 3e-4        # same math, different K order (kb-major vs tap-major)
    assert rel_l2(stats, stats_b) < 1e-4


@pytest.mark.parametrize("b,h,w_,c", [(2, 64, 384, 128), (1, 66, 200, 128), (2, 40, 100, 64), (1, 384, 384, 128)])
def test_head_tail_halo(b, h, w_, c):
    """Head tail with the resident-weights halo kernel (the default for this layer) and with per-tap boxes."""
    o = ops()
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    w = rnd(32, c, 3, 3, scale=(9 * c) ** -0.5).to(torch.bfloat16)
    bias, hw, hb = rnd(32), rnd(3, 32, scale=0.3), rnd(3, scale=0.1)
    outs = []
    for halo in (1, -1):
        hout = torch.full((b, 3, h, w_), float("nan"), device=dev(), dtype=torch.float32)
        o.conv3x3(x, o.pack_conv_weight(w), None, bias=bias, head=(hw, hb, hout, True), halo=halo)
        torch.cuda.synchronize()
        outs.append(hout)
    v = F.relu(conv_ref(x, w) + bias)
    ref = F.relu(torch.einsum("bhwj,kj->bkhw", v, hw) + hb[None, :, None, None])
    assert rel_l2(outs[0], ref) < 1e-4 and rel_l2(outs[1], ref) < 1e-4


def test_conv3x3_residual_dual():
    o = ops()
    b, h, w_, c = 2, 48, 48, 256
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    skip = rnd(b, h, w_, c, seed=5).to(torch.bfloat16)
    w = rnd(c, c, 3, 3, scale=(9 * c) ** -0.5).to(torch.bfloat16)
    bias = rnd(c)
    for bn in (128, 256):
        out = torch.empty((b, h, w_, c), device=dev(), dtype=torch.bfloat16)
        out2 = torch.empty_like(out)
        o.conv3x3(x, o.pack_conv_weight(w), out, bias=bias, residual=skip, out2=out2, block_n=bn)
        torch.cuda.synchronize()
        ref = conv_ref(x, w) + bias + skip.float()
        check(out, ref, f"conv3x3 residual bn{bn}")
        check(out2, F.relu(ref), f"conv3x3 residual relu copy bn{bn}")


@pytest.mark.parametrize("mode", ["same", "sym1"])
def test_conv3x3_stride2(mode):
    o = ops()
    b, h, w_, c, n = 2, 48, 48, 128, 128
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    w = rnd(n, c, 3, 3, scale=(9 * c) ** -0.5).to(torch.bfloat16)
    out = torch.empty((b, h // 2, w_ // 2, n), device=dev(), dtype=torch.bfloat16)
    o.conv3x3_s2(x, o.pack_conv_weight(w), out, mode)
    torch.cuda.synchronize()
    xn = x.float().permute(0, 3, 1, 2)
    if mode == "same":
        xn = F.pad(xn, (0, 1, 0, 1))
        ref = F.conv2d(xn, w.float(), stride=2)
    else:
        ref = F.conv2d(xn, w.float(), stride=2, padding=1)
    check(out, ref.permute(0, 2, 3, 1), f"conv3x3 s2 {mode}")


def test_conv1x1_stride2_view():
    o = ops()
    b, h, w_, c, n = 2, 48, 48, 256, 512
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    w = rnd(n, c, 1, 1, scale=c ** -0.5).to(torch.bfloat16)
    out = torch.empty((b, h // 2, w_ // 2, n), device=dev(), dtype=torch.bfloat16)
    o.conv1x1(x[:, ::2, ::2, :], o.pack_conv_weight(w), out)
    torch.cuda.synchronize()
    check(out, conv_ref(x, w, stride=2, padding=0), "conv1x1 s2")


@pytest.mark.parametrize("hc", [1, 3])
def test_head_tail(hc):
    o = ops()
    b, h, w_, c = 2, 64, 96, 128
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    w = rnd(32, c, 3, 3, scale=(9 * c) ** -0.5).to(torch.bfloat16)
    bias = rnd(32)
    hw = rnd(hc, 32, scale=0.3)
    hb = rnd(hc, scale=0.1)
    hout = torch.full((b, hc, h, w_), float("nan"), device=dev(), dtype=torch.float32)
    o.conv3x3(x, o.pack_conv_weight(w), None, bias=bias, head=(hw, hb, hout, True))
    torch.cuda.synchronize()
    v = F.relu(conv_ref(x, w) + bias)                      # [b,h,w,32]
    ref = F.relu(torch.einsum("bhwj,kj->bkhw", v, hw) + hb[None, :, None, None])
    err = rel_l2(hout, ref)
    assert err < 1e-4, f"head tail rel-L2 {err:.3e}"


def test_readout_style_token_window():
    """A = tokens[:, 1:, :] (strided window), per-image bias, GELU, output [B,24,24,C]."""
    o = ops()
    b, n, c = 3, 577, 768
    tok = rnd(b, n, c).to(torch.bfloat16)
    w = rnd(c, c, scale=c ** -0.5).to(torch.bfloat16)
    bias = rnd(b, c)
    out = torch.full((b, 1, 576, c), float("nan"), device=dev(), dtype=torch.bfloat16)
    o.linear(tok[:, 1:, :].unsqueeze(1), w, out, bias=bias, bias_per_image=True, act=o.ACT_GELU)
    torch.cuda.synchronize()
    ref = F.gelu(tok[:, 1:, :].float() @ w.float().t() + bias[:, None, :])
    check(out.view(b, 576, c), ref, "token window linear")


def test_patch_proj_style_pos_residual():
    """Output written into tokens[:, 1:, :] with a batch-broadcast residual (pos_embed)."""
    o = ops()
    b, c, k = 3, 768, 1024
    x = rnd(b, 1, 576, k).to(torch.bfloat16)
    w = rnd(c, k, scale=k ** -0.5).to(torch.bfloat16)
    bias = rnd(c)
    pos = rnd(1, 1, 577, c).to(torch.bfloat16)
    tokens = torch.zeros(b, 577, c, device=dev(), dtype=torch.bfloat16)
    o.linear(x, w, tokens[:, 1:, :].unsqueeze(1), bias=bias, residual=pos[:, :, 1:, :])
    torch.cuda.synchronize()
    ref = x.float().view(b, 576, k) @ w.float().t() + bias + pos[0, 0, 1:].float()
    check(tokens[:, 1:, :], ref, "patch proj + pos")
    assert float(tokens[:, 0, :].abs().max()) == 0.0


# the four widths the LayerNorm kernels are instantiated for (VPL = cols / 256); DPT-Large runs 1024
LN_COLS = [256, 512, 768, 1024]


def test_layernorm():
    o = ops()
    for cols in LN_COLS:
        x = (rnd(4 * 577, cols) * 3 + 0.5).to(torch.bfloat16)
        g, bta = rnd(cols) * 0.1 + 1, rnd(cols) * 0.1
        out = torch.empty_like(x)
        o.layernorm(x, g, bta, out, 1e-6)
        torch.cuda.synchronize()
        check(out, F.layer_norm(x.float(), (cols,), g, bta, 1e-6), f"layernorm {cols}")


@pytest.mark.parametrize("b,tokens", [(2, 577), (1, 64), (1, 100), (13, 257), (33, 577)])
def test_attention(b, tokens):
    o = ops()
    qkv = rnd(b, tokens, 2304)
    qkv[..., :1536] *= 2.0            # peaky softmax, as in a trained ViT
    qkv = qkv.to(torch.bfloat16)
    out = torch.full((b, tokens, 768), float("nan"), device=dev(), dtype=torch.bfloat16)
    o.attention(qkv, out)
    torch.cuda.synchronize()
    q, k, v = qkv.float().view(b, tokens, 3, 12, 64).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) * 0.125
    # the kernel's own definition of where P is rounded to bf16 (see oracle/gemm_oracle.py)
    from oracle.gemm_oracle import attention_bf16
    ref = attention_bf16(q, k, v)    # plain torch ops, on the GPU
    check(out, ref.transpose(1, 2).reshape(b, tokens, 768), f"attention b{b} n{tokens}", tol=1e-3)
    exact = (torch.softmax(s, dim=-1) @ v).transpose(1, 2).reshape(b, tokens, 768)
    assert rel_l2(out.float(), exact) < 4e-3


@pytest.mark.parametrize("c,hw", [(64, 96 * 96), (256, 96 * 96), (128, 48 * 48), (1024, 24 * 24), (512, 100)])
def test_groupnorm(c, hw):
    o = ops()
    b = 3
    x = (rnd(b, hw, c) * 2 + 0.3).to(torch.bfloat16)
    g, bta = rnd(c) * 0.1 + 1, rnd(c) * 0.1
    stats = torch.empty(b, 32, 2, device=dev())
    o.groupnorm_stats(x, stats)
    out = torch.empty_like(x)
    o.groupnorm_apply(x, stats, g, bta, out, relu=True)
    torch.cuda.synchronize()
    xn = x.float().transpose(1, 2)  # [b,c,hw]
    ref = F.relu(F.group_norm(xn, 32, g, bta, 1e-5)).transpose(1, 2)
    check(out, ref, f"groupnorm c{c}")
    # with a normalised shortcut
    s = (rnd(b, hw, c, seed=9) * 1.5).to(torch.bfloat16)
    sstats = torch.empty(b, 32, 2, device=dev())
    o.groupnorm_stats(s, sstats)
    g2, b2 = rnd(c, seed=3) * 0.1 + 1, rnd(c, seed=4) * 0.1
    o.groupnorm_apply(x, stats, g, bta, out, relu=True, res=s, res_stats=sstats, res_gamma=g2, res_beta=b2)
    torch.cuda.synchronize()
    ref = F.relu(F.group_norm(xn, 32, g, bta, 1e-5) + F.group_norm(s.float().transpose(1, 2), 32, g2, b2, 1e-5))
    check(out, ref.transpose(1, 2), f"groupnorm+gn shortcut c{c}")
    o.groupnorm_apply(x, stats, g, bta, out, relu=True, res=s)
    torch.cuda.synchronize()
    ref = F.relu(F.group_norm(xn, 32, g, bta, 1e-5) + s.float().transpose(1, 2))
    check(out, ref.transpose(1, 2), f"groupnorm+identity shortcut c{c}")


@pytest.mark.parametrize("b,h,w_,c,n,pair", [(2, 96, 96, 64, 64, 0), (3, 48, 48, 128, 512, 0), (2, 24, 24, 256, 1024, 0),
                                              (2, 48, 48, 256, 256, 1), (3, 24, 24, 1024, 256, 0), (2, 20, 36, 64, 128, 0),
                                              (3, 48, 48, 128, 128, 1)])
def test_conv_fused_groupnorm_stats(b, h, w_, c, n, pair):
    """GroupNorm statistics produced by the conv epilogue (+ finalize) == statistics of the stored output."""
    o = ops()
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    w = rnd(n, c, 3, 3, scale=(9 * c) ** -0.5).to(torch.bfloat16)
    out = torch.empty((b, h, w_, n), device=dev(), dtype=torch.bfloat16)
    partial = torch.full((b * 128 * 4 * 32 * 2,), float("nan"), device=dev())
    stats = torch.full((b, 32, 2), float("nan"), device=dev())
    bn = (256 if n % 256 == 0 else 128) if pair else 0
    o.conv3x3(x, o.pack_conv_weight(w), out, gn_stats=(partial, stats), cta_pair=pair, block_n=bn)
    torch.cuda.synchronize()
    check(out, conv_ref(x, w, padding=1), "conv with fused stats")
    # the statistics are those of the UNROUNDED fp32 accumulators (what timm GroupNormAct normalises in the
    # reference), i.e. of the fp32 convolution of the same bf16 operands — not of the stored bf16 tensor
    y = conv_ref(x, w, padding=1).double().reshape(b, h * w_, 32, n // 32)
    mean = y.mean(dim=(1, 3))
    var = y.var(dim=(1, 3), unbiased=False)
    assert rel_l2(stats[..., 0], mean) < 1e-5 or float((stats[..., 0].double() - mean).abs().max()) < 2e-6
    assert rel_l2(stats[..., 1], 1.0 / torch.sqrt(var + 1e-5)) < 1e-5
    stats2 = torch.empty_like(stats)
    o.conv3x3(x, o.pack_conv_weight(w), out, gn_stats=(partial, stats2), cta_pair=pair, block_n=bn)
    torch.cuda.synchronize()
    assert torch.equal(stats, stats2)                      # deterministic
    # the standalone statistics kernel sees the stored (bf16-rounded) output: equal up to the rounding noise
    stats3 = torch.empty_like(stats)
    o.groupnorm_stats(out, stats3)
    torch.cuda.synchronize()
    assert rel_l2(stats3[..., 1], stats[..., 1]) < 1e-4
    assert float((stats3[..., 0] - stats[..., 0]).abs().max()) < 1e-3
    # the specialised (default) and the generic epilogue: same output, same partial sums, bit for bit
    out_g, stats_g = torch.empty_like(out), torch.empty_like(stats)
    o.conv3x3(x, o.pack_conv_weight(w), out_g, gn_stats=(partial, stats_g), cta_pair=pair, block_n=bn, epilogue=-1)
    torch.cuda.synchronize()
    assert torch.equal(out, out_g) and torch.equal(stats, stats_g)


def test_conv_out2_gelu_copy():
    """out keeps the pre-activation, out2 = exact-erf GELU of the same fp32 value (train-mode mlp.fc1)."""
    o = ops()
    rows, c, n = 2 * 577, 256, 1024
    x = rnd(rows, c).to(torch.bfloat16)
    w = rnd(n, c, scale=c ** -0.5).to(torch.bfloat16)
    bias = rnd(n)
    out = torch.empty((rows, n), device=dev(), dtype=torch.bfloat16)
    out2 = torch.empty_like(out)
    o.linear(x, w, out, bias=bias, out2=out2, out2_act=o.ACT_GELU)
    act = torch.empty_like(out)
    o.linear(x, w, act, bias=bias, act=o.ACT_GELU)            # the inference epilogue
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t() + bias
    check(out, ref, "pre-activation")
    check(out2, F.gelu(ref), "gelu copy")
    assert torch.equal(out2, act)


def test_stem_path():
    o = ops()
    b, h, w_ = 2, 64, 96
    x = rnd(b, 3, h, w_)
    cols = torch.full((b * (h // 2) * (w_ // 2), 160), float("nan"), device=dev(), dtype=torch.bfloat16)
    o.stem_im2col(x, cols)
    torch.cuda.synchronize()
    xp = F.pad(x, (2, 3, 2, 3))
    ref = F.unfold(xp, 7, stride=2)  # [b, 3*49, L] with channel-major (c, ky, kx)
    ref = ref.view(b, 3, 49, -1).permute(0, 3, 2, 1).reshape(b * (h // 2) * (w_ // 2), 147)
    assert torch.equal(cols[:, :147].float(), ref.to(torch.bfloat16).float())
    assert float(cols[:, 147:].abs().max()) == 0.0
    # GN + ReLU + maxpool (TF-SAME (0,1))
    c = 64
    y = (rnd(b, h, w_, c) * 2).to(torch.bfloat16)
    g, bta = rnd(c) * 0.1 + 1, rnd(c) * 0.1
    stats = torch.empty(b, 32, 2, device=dev())
    o.groupnorm_stats(y, stats)
    out = torch.empty(b, h // 2, w_ // 2, c, device=dev(), dtype=torch.bfloat16)
    o.stem_gn_relu_maxpool(y, stats, g, bta, out)
    torch.cuda.synchronize()
    yn = F.relu(F.group_norm(y.float().permute(0, 3, 1, 2), 32, g, bta, 1e-5))
    ref = F.max_pool2d(F.pad(yn, (0, 1, 0, 1), value=float("-inf")), 3, 2).permute(0, 2, 3, 1)
    check(out, ref, "stem gn relu maxpool")


@pytest.mark.parametrize("h,w_,c", [(12, 12, 256), (96, 96, 256), (48, 40, 128)])
def test_upsample2x_add(h, w_, c):
    o = ops()
    b = 2
    z = rnd(b, h, w_, c).to(torch.bfloat16)
    res = rnd(b, 2 * h, 2 * w_, c, seed=2).to(torch.bfloat16)
    out = torch.empty_like(res)
    outr = torch.empty_like(res)
    o.upsample2x_add(z, out, res=res, out_relu=outr)
    torch.cuda.synchronize()
    up = F.interpolate(z.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
    ref = up.permute(0, 2, 3, 1) + res.float()
    check(out, ref, "upsample2x+add")
    check(outr, F.relu(ref), "upsample2x+add relu")
    o.upsample2x_add(z, out)
    torch.cuda.synchronize()
    check(out, up.permute(0, 2, 3, 1), "upsample2x")


def test_cls_and_readout_bias():
    o = ops()
    b, c = 4, 768
    tokens = rnd(b, 577, c).to(torch.bfloat16)
    cls, pos0 = rnd(c), rnd(c, seed=1)
    t2 = tokens.clone()
    o.write_cls_row(t2, cls, pos0)
    w = rnd(c, 2 * c, scale=(2 * c) ** -0.5).to(torch.bfloat16)
    bias = rnd(c)
    out = torch.empty(b, c, device=dev())
    o.readout_cls_bias(w, bias, tokens, out)
    torch.cuda.synchronize()
    assert torch.equal(t2[:, 0].float(), (cls + pos0).to(torch.bfloat16).float().expand(b, c))
    assert torch.equal(t2[:, 1:], tokens[:, 1:])
    ref = tokens[:, 0].float() @ w[:, c:].float().t() + bias
    assert rel_l2(out, ref) < 1e-5


# ---- specialised epilogues (odb_conv_gemm_desc.epilogue): the straight-line bias / bias+relu /
# bias+gelu / bias+residual(TMA) bodies against the PyTorch reference AND bit-for-bit against the
# generic epilogue, on every tile geometry the network uses (CTA pair, N tiles 64/128/256, ragged M)
@pytest.mark.parametrize("m,k,n,block_n,pair", [
    (577 * 8, 768, 2304, 0, 0), (577 * 8, 768, 768, 256, 1), (577 * 8, 768, 768, 256, -1), (1000, 256, 128, 0, 0),
    (333, 160, 64, 64, 0), (130, 64, 256, 0, 0), (4000, 3072, 768, 0, 0), (128 * 296 + 5, 128, 256, 256, 1),
    (128 * 300 + 77, 1152, 128, 128, 1), (128 * 300 + 77, 1152, 128, 128, -1),
])
@pytest.mark.parametrize("mode", ["bias", "relu", "gelu", "res", "res_inplace"])
def test_linear_fast_epilogues(m, k, n, block_n, pair, mode):
    o = ops()
    x = rnd(m, k).to(torch.bfloat16)
    w = rnd(n, k, scale=k ** -0.5).to(torch.bfloat16)
    bias = rnd(n)
    res = rnd(m, n, seed=3).to(torch.bfloat16)
    act = {"bias": 0, "relu": 1, "gelu": 2, "res": 0, "res_inplace": 0}[mode]
    outs = []
    for epi in (0, -1):
        out = torch.full((m, n), float("nan"), device=dev(), dtype=torch.bfloat16)
        kw = dict(bias=bias, act=act, block_n=block_n, cta_pair=pair, epilogue=epi)
        if mode == "res":
            kw["residual"] = res
        elif mode == "res_inplace":
            out.copy_(res)
            kw["residual"] = out                       # x += f(x): the ViT residual stream
        o.linear(x, w, out, **kw)
        torch.cuda.synchronize()
        outs.append(out)
    v = x.float() @ w.float().t() + bias
    v = [v, F.relu(v), F.gelu(v)][act]
    if mode.startswith("res"):
        v = v + res.float()
    check(outs[0], v, f"fast epilogue {mode} {m}x{k}x{n}")
    assert torch.equal(outs[0], outs[1]), f"fast vs generic epilogue differ ({mode})"


@pytest.mark.parametrize("b,h,w_,c,n", [(2, 48, 48, 256, 256), (1, 24, 24, 256, 256), (2, 20, 36, 64, 128), (3, 12, 12, 256, 64)])
@pytest.mark.parametrize("mode", ["relu", "res"])
def test_conv3x3_fast_epilogues(b, h, w_, c, n, mode):
    o = ops()
    x = rnd(b, h, w_, c).to(torch.bfloat16)
    w = rnd(n, c, 3, 3, scale=(9 * c) ** -0.5).to(torch.bfloat16)
    bias = rnd(n)
    skip = rnd(b, h, w_, n, seed=5).to(torch.bfloat16)
    outs = []
    for epi in (0, -1):
        out = torch.full((b, h, w_, n), float("nan"), device=dev(), dtype=torch.bfloat16)
        if mode == "relu":
            o.conv3x3(x, o.pack_conv_weight(w), out, bias=bias, act=o.ACT_RELU, epilogue=epi)
        else:
            o.conv3x3(x, o.pack_conv_weight(w), out, bias=bias, residual=skip, epilogue=epi)
        torch.cuda.synchronize()
        outs.append(out)
    ref = conv_ref(x, w) + bias
    ref = F.relu(ref) if mode == "relu" else ref + skip.float()
    check(outs[0], ref, f"conv3x3 fast epilogue {mode}")
    assert torch.equal(outs[0], outs[1])


def test_gelu_epilogue_accuracy():
    """The polynomial exact-erf GELU of the epilogue: bf16 result = correctly rounded x*Phi(x) except for
    rounding flips on near-ties (identity weight, so the GEMM adds nothing)."""
    o = ops()
    m, k = 4096, 64
    g = torch.Generator().manual_seed(0)
    # (for x < -8 the kernel clamps the exponent polynomial: |error| < 1e-14 absolute, not tested here)
    x = torch.cat([torch.linspace(-8, 8, m * k // 2), torch.randn(m * k // 2, generator=g) * 2]).view(m, k)
    x = x.to(dev()).to(torch.bfloat16)
    eye = torch.eye(k, device=dev()).to(torch.bfloat16)
    out = torch.empty(m, k, device=dev(), dtype=torch.bfloat16)
    o.linear(x, eye, out, bias=torch.zeros(k, device=dev()), act=o.ACT_GELU)
    torch.cuda.synchronize()
    xd = x.double()
    exact = xd * 0.5 * torch.special.erfc(-xd / math.sqrt(2.0))    # (1 + erf) cancels for x < -5
    ref = exact.float().to(torch.bfloat16)
    flips = (out != ref)
    assert float(flips.float().mean()) < 2e-3
    # a flipped element is still within one bf16 ulp of the exact value
    err = (out.double() - exact).abs()
    ulp = torch.maximum(exact.abs(), torch.tensor(1e-30, device=dev(), dtype=torch.float64)) * 2.0 ** -7
    assert bool((err <= ulp + 1e-12).all())


# ---- fp32 residual stream: tensor-core GEMM (bf16 operands) with an fp32 residual and an fp32 result
# (EPI_BIAS_RES_F32: ViT attn.proj / mlp.fc2 / patch projection)
@pytest.mark.parametrize("m,k,n,block_n,pair", [
    (577 * 8, 768, 768, 0, 0), (577 * 8, 3072, 768, 256, 1), (1000, 768, 768, 256, -1), (900, 256, 128, 128, -1),
    (5000, 512, 128, 128, 1), (300, 64, 64, 64, -1), (577 * 32, 768, 768, 0, 0), (128 * 3, 256, 512, 256, 1),
])
@pytest.mark.parametrize("inplace", [False, True])
def test_linear_fp32_residual_stream(m, k, n, block_n, pair, inplace):
    o = ops()
    x = rnd(m, k).to(torch.bfloat16)
    w = rnd(n, k, scale=k ** -0.5).to(torch.bfloat16)
    bias = rnd(n)
    res = rnd(m, n, seed=11) * 3
    ref = (x.double() @ w.double().t() + bias.double() + res.double())
    out = res.clone() if inplace else torch.full((m, n), float("nan"), device=dev())
    o.linear(x, w, out, bias=bias, residual=(out if inplace else res), block_n=block_n, cta_pair=pair)
    torch.cuda.synchronize()
    err = rel_l2(out, ref)
    assert err < 2e-6, f"fp32-out linear {m}x{k}x{n}: {err:.3e}"      # fp32 accumulate + fp32 epilogue, no bf16 rounding


def test_patch_proj_fp32_tokens():
    """Output written into the fp32 token stream tokens[:, 1:, :] with the per-image replicated pos_embed as residual."""
    o = ops()
    b, c, k = 3, 768, 1024
    x = rnd(b, 1, 576, k).to(torch.bfloat16)
    w = rnd(c, k, scale=k ** -0.5).to(torch.bfloat16)
    bias = rnd(c)
    pos = rnd(576, c).unsqueeze(0).expand(b, -1, -1).contiguous()
    tokens = torch.zeros(b, 577, c, device=dev())
    o.linear(x, w, tokens[:, 1:, :].unsqueeze(1), bias=bias, residual=pos.unsqueeze(1))
    torch.cuda.synchronize()
    ref = x.double().view(b, 576, k) @ w.double().t() + bias.double() + pos.double()
    assert rel_l2(tokens[:, 1:, :], ref) < 2e-6
    assert float(tokens[:, 0, :].abs().max()) == 0.0


def test_layernorm_fp32_stream_and_cast():
    o = ops()
    for cols in LN_COLS:
        x = rnd(4 * 577, cols) * 3 + 0.5
        g, bta = rnd(cols) * 0.1 + 1, rnd(cols) * 0.1
        out = torch.empty_like(x, dtype=torch.bfloat16)
        o.layernorm(x, g, bta, out, 1e-6)
        xb = torch.empty_like(out)
        o.cast_f32_bf16(x, xb)
        torch.cuda.synchronize()
        check(out, F.layer_norm(x, (cols,), g, bta, 1e-6), f"layernorm fp32 in {cols}")
        assert torch.equal(xb, x.to(torch.bfloat16)), cols
