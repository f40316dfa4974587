"""The fp8 inference mode on the GPU: the e4m3 quantisers bit for bit, the scaled e4m3 GEMM against float64 on the same
operands at the ViT layer shapes, and the whole models (error next to bf16's, batch invariance, CUDA graph, repeat bits,
refusals, switching back to bf16)."""
import pytest
import torch

from omnidata_b200 import _capi, ops
from omnidata_b200.model import DPTDepthModel, quantize_rows_e4m3

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
GUARD = 4096


def guarded(shape, dtype, fill):
    """A tensor of `shape` inside a buffer with GUARD elements of `fill` bits either side."""
    n = 1
    for s in shape:
        n *= s
    raw = torch.empty(n + 2 * GUARD, dtype=torch.uint8 if dtype == ops.E4M3 else dtype, device=dev)
    raw.fill_(fill)
    t = raw[GUARD:GUARD + n]
    t = t.view(ops.E4M3) if dtype == ops.E4M3 else t
    return raw, t.view(shape)


def guards_intact(raw, fill):
    g = torch.cat([raw[:GUARD], raw[-GUARD:]])
    return bool((g == fill).all())


def assert_same_bits(q, rq, src):
    a, b = q.view(torch.uint8), rq.view(torch.uint8)
    bad = (a != b).nonzero()
    if len(bad):
        r, c = bad[0].tolist()
        raise AssertionError(f"{len(bad)} e4m3 bytes differ; first at ({r}, {c}): source {src[r, c].item()!r}, "
                             f"kernel {a[r, c].item():#04x}, rule {b[r, c].item():#04x}; row amax "
                             f"{src[r].abs().max().item()!r}")


def quant_ref(x32):
    """Per-row e4m3 quantisation of an fp32 tensor [rows, C] (the packer's rule, on the same device)."""
    return quantize_rows_e4m3(x32)


@pytest.mark.parametrize("cols", [768, 1024, 3072, 4096])
def test_rowquant_bit_exact(cols):
    g = torch.Generator(device=dev).manual_seed(cols)
    rows = 1155
    x = (torch.randn(rows, cols, device=dev, generator=g) * torch.logspace(-3, 2, rows, device=dev)[:, None])
    x = x.to(torch.bfloat16)
    x[7] = 0
    x[8, 5] = 1e4                                         # one dominant element
    raw_q, q = guarded((rows, cols), ops.E4M3, 0x5A)
    raw_s, s = guarded((rows,), torch.float32, 0.0)
    raw_s.fill_(-7.0)
    ops.rowquant_e4m3(x, q, s)
    torch.cuda.synchronize()
    rq, rs = quant_ref(x.float())
    assert_same_bits(q, rq, x.float())
    assert torch.equal(s, rs) and s[7] == 1.0
    assert guards_intact(raw_q, 0x5A) and guards_intact(raw_s, -7.0)
    q2, s2 = torch.empty_like(q), torch.empty_like(s)
    ops.rowquant_e4m3(x, q2, s2)
    assert torch.equal(q2.view(torch.uint8), q.view(torch.uint8)) and torch.equal(s2, s)


@pytest.mark.parametrize("cols", [768, 1024])
@pytest.mark.parametrize("xdt", [torch.float32, torch.bfloat16])
def test_layernorm_e4m3_bit_exact(cols, xdt):
    g = torch.Generator(device=dev).manual_seed(cols + 1)
    rows = 1155
    x = (torch.randn(rows, cols, device=dev, generator=g) * 3 + 0.5).to(xdt)
    gamma = torch.randn(cols, device=dev, generator=g)
    beta = torch.randn(cols, device=dev, generator=g)
    gamma[:] = torch.where(torch.arange(cols, device=dev) == 3, 0.0, gamma)
    zero_row = torch.zeros(cols, device=dev)
    raw_q, q = guarded((rows, cols), ops.E4M3, 0xA5)
    raw_s, s = guarded((rows,), torch.float32, 0.0)
    raw_s.fill_(-7.0)
    ops.layernorm_e4m3(x, gamma, beta, q, s)
    # the fp32 LayerNorm of the same kernel arithmetic, quantised by the rule (x fp32: the (f32, f32) instance)
    if xdt == torch.float32:
        z = torch.empty(rows, cols, device=dev)
        ops.layernorm(x, gamma, beta, z)
    else:
        z = torch.nn.functional.layer_norm(x.float(), (cols,), gamma, beta, 1e-6)
    torch.cuda.synchronize()
    rq, rs = quant_ref(z)
    if xdt == torch.float32:
        assert_same_bits(q, rq, z)
        assert torch.equal(s, rs)
    else:       # no fp32-output instance for a bf16 input: the dequantised values are within one e4m3 step of z
        assert ((q.float() * s[:, None] - z).abs() <= z.abs() / 8 + s[:, None] * 2 ** -8).all()
    assert guards_intact(raw_q, 0xA5) and guards_intact(raw_s, -7.0)
    # an all-zero LayerNorm output row (gamma = beta = 0) gets scale 1 and q 0
    z0 = torch.empty(2, cols, dtype=ops.E4M3, device=dev)
    s0 = torch.empty(2, device=dev)
    ops.layernorm_e4m3(x[:2].contiguous(), zero_row, zero_row, z0, s0)
    torch.cuda.synchronize()
    assert (s0 == 1.0).all() and (z0.float() == 0).all()
    q2, s2 = torch.empty_like(q), torch.empty_like(s)
    ops.layernorm_e4m3(x, gamma, beta, q2, s2)
    assert torch.equal(q2.view(torch.uint8), q.view(torch.uint8)) and torch.equal(s2, s)


def _gemm_case(rows, n, k, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(rows, k, device=dev, generator=g) * torch.logspace(-1, 1, rows, device=dev)[:, None]
    w = torch.randn(n, k, device=dev, generator=g) / k ** 0.5
    qa, sa = quant_ref(a)
    qw, sw = quant_ref(w)
    bias = torch.randn(n, device=dev, generator=g) * 0.1
    acc = qa.double() @ qw.double().t()
    absacc = qa.double().abs() @ qw.double().abs().t()
    scale = sa.double()[:, None] * sw.double()[None, :]
    return qa, sa, qw, sw, bias, acc * scale + bias.double(), absacc * scale


# Hopper's e4m3 wgmma does not accumulate in full fp32 inside the tensor core: measured on an H100 (700 W), its error
# against the float64 sum reaches 5.1e-4 (about 2^-11) of the sum of the terms' magnitudes at K = 768..4096, where fp32
# accumulation would stay near 2.4e-6.  The bound is that measurement with a margin of 4.
ACC_E4M3 = 2.0 ** -9

# the ViT layer shapes (N, K) of D = 768 and 1024, at the token counts of batch 2 / 384x384 and a ragged count
SHAPES = [(3 * D, D) for D in (768, 1024)] + [(D, D) for D in (768, 1024)] + [(4 * D, D) for D in (768, 1024)] + \
         [(D, 4 * D) for D in (768, 1024)]


@pytest.mark.parametrize("rows", [1154, 301])
@pytest.mark.parametrize("n,k", SHAPES)
@pytest.mark.parametrize("epi", ["bias", "gelu", "res"])
def test_linear_fp8_against_float64(rows, n, k, epi):
    qa, sa, qw, sw, bias, ref, absref = _gemm_case(rows, n, k, rows + n + k)
    if epi == "res":
        res = torch.randn(rows, n, device=dev)
        raw, out = guarded((rows, n), torch.float32, 0.0)
        raw.fill_(-3.0)
        out.copy_(torch.full_like(out, 5.0))
        ops.linear_fp8(qa, sa, qw, sw, out, bias=bias, residual=res)
        want = ref + res.double()
        tol = ACC_E4M3 * absref + 1e-6 * want.abs()
    else:
        raw, out = guarded((rows, n), torch.bfloat16, 0.0)
        raw.fill_(-3.0)
        act = ops.ACT_GELU if epi == "gelu" else ops.ACT_NONE
        ops.linear_fp8(qa, sa, qw, sw, out, bias=bias, act=act)
        want = torch.nn.functional.gelu(ref) if epi == "gelu" else ref
        tol = ACC_E4M3 * absref + 2.0 ** -8 * want.abs() + 1e-6
    torch.cuda.synchronize()
    err = (out.double() - want).abs()
    assert (err <= tol).all(), (err / tol).max().item()
    assert guards_intact(raw, -3.0)


def _run(model, x):
    with torch.no_grad():
        return model(x).clone()


# rel-L2 error of the fp8 output against the fp32 mode at 384x384, batch 2, seed 0 (randomly initialised weights, whose
# outputs amplify rounding: bf16 measured 0.52 / 0.019 / 0.006), measured on an H100 at 0.546 / 0.144 / 0.058; the
# ceilings add about 20 % to those measurements
CEILING = {"vitb_rn50_384": 0.66, "vitb16_384": 0.18, "vitl16_384": 0.07}


@pytest.mark.parametrize("backbone", ["vitb_rn50_384", "vitb16_384", "vitl16_384"])
def test_fp8_model(backbone):
    torch.manual_seed(0)
    m = DPTDepthModel(backbone=backbone).to(dev).eval()
    x = torch.rand(2, 3, 384, 384, device=dev) * 2 - 1
    m.precision = "fp32"
    ref = _run(m, x)
    m.precision = "bf16"
    bf = _run(m, x)
    m.precision = "fp8"
    f8 = _run(m, x)
    rel = lambda y: ((y.double() - ref.double()).norm() / ref.double().norm()).item()
    print(f"{backbone}: rel-L2 error against fp32 mode: bf16 {rel(bf):.2e}  fp8 {rel(f8):.2e}")
    assert rel(f8) <= CEILING[backbone]
    assert torch.equal(_run(m, x), f8)                              # repeat: same bits
    assert torch.equal(_run(m, x[1:2]), f8[1:2])                     # independent of the batch
    m.use_cuda_graph = True
    assert torch.equal(_run(m, x), f8)                              # CUDA-graph replay = eager
    m.use_cuda_graph = False
    m.precision = "bf16"
    assert torch.equal(_run(m, x), bf)                              # bf16 bits come back


def test_fp8_batch17_and_highres():
    torch.manual_seed(0)
    m = DPTDepthModel(backbone="vitb_rn50_384").to(dev).eval()
    m.precision = "fp8"
    x = torch.rand(17, 3, 384, 384, device=dev)
    y = _run(m, x)
    assert torch.equal(_run(m, x[5:6]), y[5:6])
    xh = torch.rand(1, 3, 480, 640, device=dev)
    yh = _run(m, xh)
    m.precision = "fp32"
    rh = _run(m, xh)
    rel = ((yh.double() - rh.double()).norm() / rh.double().norm()).item()
    print(f"vitb_rn50_384 480x640: fp8 rel-L2 error against fp32 mode {rel:.2e}")
    assert rel < 0.61        # measured 0.505 on an H100


def test_fp8_refusals():
    from omnidata_b200.train import DepthTrainStep, NormalTrainStep, TrainEngine
    m = DPTDepthModel(backbone="vitb16_384").to(dev)
    m.precision = "fp8"
    n0 = _capi.launch_count()
    x = torch.rand(1, 3, 384, 384, device=dev)
    m.train()
    with pytest.raises(ValueError):
        m(x)
    m.eval()
    with pytest.raises(ValueError):
        m(x.requires_grad_())
    with pytest.raises(ValueError):
        TrainEngine(m, "fp8")
    with pytest.raises(ValueError):
        DepthTrainStep(m, precision="fp8", input_size=(384, 384))
    mn = DPTDepthModel(backbone="vitb16_384", num_channels=3).to(dev)
    with pytest.raises(ValueError):
        NormalTrainStep(mn, precision="fp8", input_size=(384, 384))
    assert _capi.launch_count() == n0
