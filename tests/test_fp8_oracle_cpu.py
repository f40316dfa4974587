"""The fp8 mode's arithmetic, without a GPU: the per-row e4m3 quantiser the weight packer uses against a direct
restatement of the rule (all-zero rows, saturation at +-448, round-to-nearest-even ties), and the fp8 oracle's
quantiser and per-GEMM definition (oracle/fp8_oracle.py) against the packer and a float64 einsum."""
import torch

from omnidata_b200.model import quantize_rows_e4m3

E4M3 = torch.float8_e4m3fn


def e4m3_value_table():
    """Every finite e4m3fn value, as float64, from its bit pattern: sign, 4-bit exponent (bias 7), 3-bit mantissa."""
    vals = {}
    for b in range(256):
        s, e, m = b >> 7, (b >> 3) & 15, b & 7
        if e == 15 and m == 7:
            continue                                     # NaN
        v = (m / 8.0) * 2.0 ** -6 if e == 0 else (1 + m / 8.0) * 2.0 ** (e - 7)
        vals[b] = -v if s else v
    return vals


def quantize_restated(w: torch.Tensor):
    """The rule written out element by element: scale = amax / 448 (fp32), y = w * fp32(448 / amax), the nearest e4m3
    value to y with ties to the even mantissa, |y| > 448 saturating to +-448; an all-zero row: scale 1, q 0."""
    import math
    table = e4m3_value_table()
    q = torch.empty(w.shape, dtype=torch.uint8)
    s = torch.empty(w.shape[0], dtype=torch.float32)
    for r in range(w.shape[0]):
        amax = w[r].abs().max().float()
        s[r] = amax / 448.0 if amax > 0 else 1.0
        inv = (torch.tensor(448.0) / amax) if amax > 0 else torch.tensor(0.0)
        for c in range(w.shape[1]):
            y = float(w[r, c].float() * inv)
            y = max(-448.0, min(448.0, y))
            neg = math.copysign(1.0, y) < 0
            # candidates of y's sign (a value that rounds to zero keeps its sign); nearest, then the even mantissa
            cands = [(v, b) for b, v in table.items() if (b >> 7) == neg]
            q[r, c] = min(cands, key=lambda vb: (abs(vb[0] - y), vb[1] & 1))[1]
    return q, s


def test_weight_quantiser_matches_the_rule():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(6, 40, generator=g) * torch.tensor([1e-3, 1.0, 30.0, 1.0, 1.0, 1.0])[:, None]
    w[3] = 0.0                                          # all-zero row
    w[4, :] = torch.linspace(-1.0, 1.0, 40)
    w[4, 0] = -2.0                                      # amax row: exactly -448 after scaling
    # ties: with amax = 448 the scale is 1, so these values sit exactly halfway between two e4m3 neighbours
    w[5, :] = 0.0
    w[5, 0] = 448.0
    w[5, 1:9] = torch.tensor([1.0625, 1.1875, 17.0, 19.0, -1.0625, 0.013671875, 240.0, 432.0])
    q, s = quantize_rows_e4m3(w)
    rq, rs = quantize_restated(w)
    assert q.dtype == E4M3
    assert torch.equal(q.view(torch.uint8), rq), (q.view(torch.uint8) ^ rq).nonzero()
    assert torch.equal(s, rs)
    assert s[3] == 1.0 and (q[3].float() == 0).all()
    assert q[4, 0].float() == -448.0
    # the ties went to the even mantissa
    assert q[5, 1:9].float().tolist() == [1.0, 1.25, 16.0, 20.0, -1.0, 0.013671875, 240.0, 448.0]


def test_oracle_gemm_is_the_dequantised_product():
    """oracle/fp8_oracle.py: its quantiser gives the packer's bits, and its scaled GEMM equals a float64 einsum of the
    dequantised operands (the definition tests/test_fp8_gpu.py and tests/test_fp8_model_gpu.py hold the kernels to)."""
    from oracle.fp8_oracle import linear_fp8_ref, quantize_rows_e4m3 as oracle_quantize
    g = torch.Generator().manual_seed(1)
    a, w, b = torch.randn(33, 256, generator=g), torch.randn(64, 256, generator=g), torch.randn(64, generator=g)
    a[4] = 0
    qa, sa = oracle_quantize(a)
    qw, sw = oracle_quantize(w)
    pa, ps = quantize_rows_e4m3(a)
    assert torch.equal(qa.view(torch.uint8), pa.view(torch.uint8)) and torch.equal(sa, ps)
    ref = torch.einsum("rk,ck->rc", qa.double() * sa.double()[:, None], qw.double() * sw.double()[:, None]) + b.double()
    assert torch.allclose(linear_fp8_ref(qa, sa, qw, sw, b), ref, rtol=1e-12, atol=1e-12)
    assert ((qa.double() * sa.double()[:, None]) - a.double()).abs().max() <= a.abs().max() / 16
