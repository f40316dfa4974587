"""oracle/gemm_oracle.py against torch's own convolution and autograd, in float64 on the CPU: the float64 references
the backward GEMM tests hold the kernels to (tests/test_bwd_gemm_gpu.py) are themselves right.  The stride-2 input
gradient is the engine's own plan (train.parity_dgrad_operands) on a dgrad operand in odb_pack_weight's layout."""
import pytest
import torch
import torch.nn.functional as F

from oracle import gemm_oracle as G

TOL = 1e-12
GRIDS = [(24, 24), (10, 15), (2, 3)]          # parity-plane (= output) grids of the stride-2 layers


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed + sum(shape)), dtype=torch.float64)


def rel(a, b):
    return float((a.detach() - b.detach()).norm() / b.detach().norm())


def nchw(t):
    return t.permute(0, 3, 1, 2)


def _conv(x, w, mode):
    """x [B,C,H,W]: the reference convolution of each tap set (3x3 stride 1 pad 1; stride 2 TF-SAME; stride 2 pad 1)."""
    if mode == "3x3":
        return F.conv2d(x, w, padding=1)
    if mode == "same":
        return F.conv2d(F.pad(x, (0, 1, 0, 1)), w, stride=2)
    return F.conv2d(x, w, stride=2, padding=1)


def _views_taps(x, mode):
    from omnidata_b200 import ops
    if mode == "3x3":
        return [x], ops.TAPS_3X3
    return [x[:, py::2, px::2, :] for py in (0, 1) for px in (0, 1)], ops._parity_taps(mode)


CASES = [("3x3", (5, 7))] + [(m, g) for m in ("same", "sym1") for g in GRIDS]


@pytest.mark.parametrize("mode,grid", CASES, ids=[f"{m}-{h}x{w}" for m, (h, w) in CASES])
def test_conv_gemm_ref_and_wgrad_ref_match_torch(mode, grid):
    from omnidata_b200 import ops
    h, w = grid
    s = 1 if mode == "3x3" else 2
    B, c, n = 2, 8, 16
    x = rnd(B, s * h, s * w, c)
    wt = rnd(n, c, 3, 3, seed=1)
    bias, res = rnd(n, seed=2), rnd(B, h, w, n, seed=3)
    views, taps = _views_taps(x, mode)
    y = G.conv_gemm_ref(views, taps, ops.pack_conv_weight(wt, torch.float64), (B, h, w), bias=bias, residual=res)
    ref = nchw(x).requires_grad_(True)
    wr = wt.clone().requires_grad_(True)
    yt = _conv(ref, wr, mode) + bias[:, None, None]
    assert rel(y, yt.permute(0, 2, 3, 1) + res) < TOL
    act = G.conv_gemm_ref(views, taps, ops.pack_conv_weight(wt, torch.float64), (B, h, w), bias=bias, act=1)
    assert rel(act, torch.relu(yt).permute(0, 2, 3, 1)) < TOL
    dy = rnd(B, h, w, n, seed=4)
    gw, = torch.autograd.grad(yt, (wr,), nchw(dy))
    assert rel(G.wgrad_ref(views, taps, dy), ops.pack_conv_weight(gw, torch.float64)) < TOL


def test_two_dimensional_views_are_rows():
    """[rows, C] means B = H = 1 for both oracles (a linear layer), and a token window is a plain strided view."""
    x, w, dy = rnd(37, 24), rnd(16, 24, seed=1), rnd(37, 16, seed=2)
    from omnidata_b200 import ops
    assert rel(G.conv_gemm_ref([x], ops.TAPS_1, w, (1, 1, 37))[0, 0], x @ w.t()) < TOL
    assert rel(G.wgrad_ref([x], ops.TAPS_1, dy), dy.t() @ x) < TOL
    tok = rnd(2, 38, 24, seed=3)
    dyt = rnd(2, 1, 37, 16, seed=4)
    ref = torch.einsum("btn,btc->nc", dyt[:, 0], tok[:, 1:])
    assert rel(G.wgrad_ref([tok[:, 1:, :].unsqueeze(1)], ops.TAPS_1, dyt), ref) < TOL


@pytest.mark.parametrize("mode", ["same", "sym1"])
@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_stride2_dgrad_plan_matches_autograd(mode, grid):
    """parity_dgrad_operands on the dgrad operand [c][9 * n] (tap slot 8 - t holds W_t^T, as test_pack_table_multi
    builds it) + one conv_gemm_ref per parity plane == the autograd input gradient of the stride-2 convolution."""
    from omnidata_b200.train import parity_dgrad_operands
    h, w = grid
    B, c, n = 2, 8, 16
    wt = rnd(n, c, 3, 3, seed=5)
    wb = wt.reshape(n, c, 9).permute(1, 2, 0).flip(1).reshape(c, 9 * n)
    dy = rnd(B, h, w, n, seed=6)
    dx = torch.full((B, 2 * h, 2 * w, c), float("nan"), dtype=torch.float64)
    for (py, px), (wp, taps) in parity_dgrad_operands(wb, n, mode).items():
        dx[:, py::2, px::2, :] = G.conv_gemm_ref([dy], taps, wp, (B, h, w))
    xr = torch.zeros(B, c, 2 * h, 2 * w, dtype=torch.float64, requires_grad=True)
    gx, = torch.autograd.grad(_conv(xr, wt, mode), (xr,), nchw(dy))
    assert rel(dx, gx.permute(0, 2, 3, 1)) < TOL


@pytest.mark.parametrize("t", [5, 65, 130])
def test_attention_bwd_ref(t):
    """Exact mode == the closed-form softmax-attention backward; rounded mode is bf16-valued and within bf16 error."""
    b, heads = 2, 2
    qkv = rnd(b, t, 3 * heads * 64) * 1.5
    d_o = rnd(b, t, heads * 64, seed=1)
    q, k, v = qkv.view(b, t, 3, heads, 64).permute(2, 0, 3, 1, 4)
    do = d_o.view(b, t, heads, 64).transpose(1, 2)
    p = torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1)
    o = p @ v
    ds = p * (do @ v.transpose(-1, -2) - (o * do).sum(-1, keepdim=True)) * 0.125
    closed = torch.stack([ds @ k, ds.transpose(-1, -2) @ q, p.transpose(-1, -2) @ do]).permute(1, 3, 0, 2, 4)
    o_rows = o.transpose(1, 2).reshape(b, t, heads * 64)
    g = G.attention_bwd_ref(qkv, o_rows, d_o)
    assert rel(g, closed.reshape(b, t, -1)) < TOL
    qkv16, o16, do16 = (z.to(torch.bfloat16) for z in (qkv, o_rows, d_o))
    r = G.attention_bwd_ref(qkv16, o16, do16, rounded=True)
    assert torch.equal(r, r.to(torch.bfloat16).double())
    assert rel(r, G.attention_bwd_ref(qkv16, o16, do16)) < 2e-2


# ------------------------------------------------------------------------------------------ the forward's definitions
@pytest.mark.parametrize("max_elems", [G.CHUNK_ELEMS, 1], ids=["whole", "per-image"])
def test_conv_gemm_ref_forward_epilogues(max_elems):
    """bias per image, a residual broadcast over the batch, the relu / gelu out2 copies, evaluated whole and one image
    at a time (the chunked path) == torch's convolution, relu and exact-erf gelu."""
    from omnidata_b200 import ops
    B, h, w, c, n = 3, 5, 7, 8, 16
    x, wt = rnd(B, h, w, c), rnd(n, c, 3, 3, seed=1)
    bias_b, res1 = rnd(B, n, seed=2), rnd(1, h, w, n, seed=3)
    yt = (F.conv2d(nchw(x), wt, padding=1) + bias_b[:, :, None, None]).permute(0, 2, 3, 1)
    wp = ops.pack_conv_weight(wt, torch.float64)
    kw = dict(bias=bias_b, bias_per_image=True, max_elems=max_elems)
    y, y2 = G.conv_gemm_ref([x], ops.TAPS_3X3, wp, (B, h, w), residual=res1, out2_act=1, **kw)
    assert rel(y, yt + res1) < TOL and rel(y2, torch.relu(yt + res1)) < TOL
    assert rel(G.conv_gemm_ref([x], ops.TAPS_3X3, wp, (B, h, w), residual=res1[0], **kw), yt + res1) < TOL   # [H, W, n]
    pre, act = G.conv_gemm_ref([x], ops.TAPS_3X3, wp, (B, h, w), out2_act=2, **kw)
    assert rel(pre, yt) < TOL and rel(act, F.gelu(yt)) < TOL
    assert rel(G.conv_gemm_ref([x], ops.TAPS_3X3, wp, (B, h, w), act=2, **kw), F.gelu(yt)) < TOL
    absolute = G.conv_acc_ref([x], ops.TAPS_3X3, wp, (B, h, w), absolute=True, max_elems=max_elems)
    assert rel(absolute, F.conv2d(nchw(x).abs(), wt.abs(), padding=1).permute(0, 2, 3, 1)) < TOL


@pytest.mark.parametrize("mode,grid", CASES, ids=[f"{m}-{h}x{w}" for m, (h, w) in CASES])
def test_chunked_references_are_the_same_definitions(mode, grid):
    """conv_gemm_ref / wgrad_ref over chunks of images == the whole batch at once (to float64 rounding)."""
    from omnidata_b200 import ops
    h, w = grid
    s = 1 if mode == "3x3" else 2
    B, c, n = 5, 8, 16
    x = rnd(B, s * h, s * w, c)
    wp = ops.pack_conv_weight(rnd(n, c, 3, 3, seed=1), torch.float64)
    views, taps = _views_taps(x, mode)
    dy = rnd(B, h, w, n, seed=4)
    per_image = h * w * len(taps) * c
    for m in (1, 2 * per_image):                        # one image, then two images per chunk (a ragged last chunk)
        assert rel(G.conv_gemm_ref(views, taps, wp, (B, h, w), max_elems=m),
                   G.conv_gemm_ref(views, taps, wp, (B, h, w))) < TOL
        assert rel(G.wgrad_ref(views, taps, dy, max_elems=m), G.wgrad_ref(views, taps, dy)) < TOL


def test_gn_stats_ref():
    """mean and rstd == what F.group_norm normalises with (biased variance, eps 1e-5), for 2 to 32 channels a group."""
    for n in (64, 256, 1024):
        y = rnd(2, 6, 5, n) * 3 + 1.5
        st = G.gn_stats_ref(y)
        b = y.shape[0]
        mean = st[..., 0].repeat_interleave(n // 32, dim=1)[:, None, None, :]
        rstd = st[..., 1].repeat_interleave(n // 32, dim=1)[:, None, None, :]
        gn = F.group_norm(nchw(y), 32, eps=1e-5).permute(0, 2, 3, 1)
        assert rel((y - mean) * rstd, gn) < TOL
        assert rel(st[..., 0], y.reshape(b, 30, 32, n // 32).mean(dim=(1, 3))) < TOL


@pytest.mark.parametrize("relu", [False, True])
def test_head_tail_ref(relu):
    """relu(conv + bias) -> 1x1 conv to head_c channels + bias -> relu? == torch, NCHW."""
    y, hw, hb = rnd(2, 6, 5, 32), rnd(3, 32, seed=1), rnd(3, seed=2)
    o = F.conv2d(torch.relu(nchw(y)), hw[:, :, None, None], hb)
    assert rel(G.head_tail_ref(y, hw, hb, relu), torch.relu(o) if relu else o) < TOL


@pytest.mark.parametrize("heads", [2, 16])
@pytest.mark.parametrize("t", [5, 65, 130])
def test_attention_ref_and_lse(t, heads):
    """Exact mode == softmax attention; rounded mode (the kernel's P rounding) within bf16 error of it; lse == the
    log-sum-exp of the logits in the kernel's log2 units."""
    b = 2
    qkv = rnd(b, t, 3 * heads * 64) * 1.5
    q, k, v = qkv.view(b, t, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2)
    closed = (torch.softmax(s * 0.125, -1) @ v).transpose(1, 2).reshape(b, t, -1)
    assert rel(G.attention_ref(qkv, heads), closed) < TOL
    assert rel(G.attention_ref(qkv, heads, rounded=True), closed) < 1e-2
    c = 0.125 * G._LOG2E_F32
    ln2 = torch.log(torch.tensor(2.0, dtype=torch.float64))
    assert rel(G.lse_ref(qkv, heads), torch.logsumexp(s * c * ln2, -1) / ln2) < TOL
    # the backward's P from it sums to one per row
    p = torch.exp2(s * c - G.lse_ref(qkv, heads)[..., None])
    assert float((p.sum(-1) - 1).abs().max()) < TOL
