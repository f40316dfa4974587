"""The fp32 residual-stream GEMM (EPI_BIAS_RES_F32: attn.proj, mlp.fc2, the patch projection) gives the same bits
whatever N tile, CTA pairing or aliasing the launch uses.

Each output element is res + (acc + bias) with acc the fp32 wgmma sum over K in a fixed order that does not depend on
the N tile, so the 64-, 128- and 256-wide instances and the CTA pairs must agree bit for bit, and updating the stream
in place (out aliasing residual, as inference does) must give the bits of a separate output.  Covered at the ViT
shapes with ragged M (B * 577 token rows, not a multiple of the 128-row tile) and at the patch projection's geometry:
output rows 1.. of each image's token block, residual the per-image replicated position rows.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

# (block_n, cta_pair): every fp32 instance the launcher has
INSTANCES = [(64, -1), (128, -1), (256, -1), (128, 1), (256, 1)]


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def dev():
    return torch.device("cuda:0")


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dev())


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def ops():
    from omnidata_b200 import ops as o
    return o


@pytest.mark.parametrize("m,k,n", [(577 * 8, 768, 768), (577 * 8, 3072, 768), (577 * 3, 1024, 768), (300, 64, 256)])
def test_fp32_residual_bits_across_tiles_and_aliasing(m, k, n):
    o = ops()
    x = rnd(m, k, seed=1).to(torch.bfloat16)
    w = rnd(n, k, scale=k ** -0.5, seed=2).to(torch.bfloat16)
    bias = rnd(n, seed=3)
    res = rnd(m, n, seed=4) * 3
    ref = x.double() @ w.double().t() + bias.double() + res.double()
    outs = {}
    for block_n, pair in INSTANCES:
        out = torch.full((m, n), float("nan"), device=dev())
        o.linear(x, w, out, bias=bias, residual=res, block_n=block_n, cta_pair=pair)
        stream = res.clone()
        o.linear(x, w, stream, bias=bias, residual=stream, block_n=block_n, cta_pair=pair)
        outs[(block_n, pair)] = (out, stream)
    torch.cuda.synchronize()
    first, _ = outs[INSTANCES[0]]
    assert rel_l2(first, ref) < 2e-6
    for key, (out, stream) in outs.items():
        assert torch.equal(out, first), f"{m}x{k}x{n} block_n {key[0]} pair {key[1]} differs from block_n 64"
        assert torch.equal(stream, out), f"{m}x{k}x{n} block_n {key[0]} pair {key[1]}: in place differs"


def test_patch_proj_fp32_bits_across_tiles():
    o = ops()
    b, c, k = 3, 768, 1024
    x = rnd(b, 1, 576, k, seed=5).to(torch.bfloat16)
    w = rnd(c, k, scale=k ** -0.5, seed=6).to(torch.bfloat16)
    bias = rnd(c, seed=7)
    pos = rnd(576, c, seed=8).unsqueeze(0).expand(b, -1, -1).contiguous()
    cls = rnd(b, 1, c, seed=9)
    ref = x.double().view(b, 576, k) @ w.double().t() + bias.double() + pos.double()
    first = None
    for block_n, pair in INSTANCES:
        tokens = torch.cat([cls, torch.full((b, 576, c), float("nan"), device=dev())], dim=1)
        o.linear(x, w, tokens[:, 1:, :].unsqueeze(1), bias=bias, residual=pos.unsqueeze(1), block_n=block_n,
                 cta_pair=pair)
        torch.cuda.synchronize()
        assert torch.equal(tokens[:, :1, :], cls), f"block_n {block_n} pair {pair} wrote the cls rows"
        if first is None:
            first = tokens
            assert rel_l2(tokens[:, 1:, :], ref) < 2e-6
        assert torch.equal(tokens, first), f"block_n {block_n} pair {pair} differs from block_n 64"
