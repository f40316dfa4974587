"""The fp8 inference mode's arithmetic (DESIGN.md §3 "Rounding points"), restated in plain PyTorch: e4m3 quantisation
emulated with torch.float8_e4m3fn, products and sums of the dequantised operands in float64.

- `quantize_rows_e4m3`: the per-row rule (ops.cu e4m3_inv_scale / e4m3_row_scale / quant8_e4m3, and the weight packer
  model.quantize_rows_e4m3).
- `linear_fp8_ref`: one scaled GEMM, v = (qa qw^T) * (sa[r] * sw[c]) + bias[c] (conv_gemm.cu fp8_read_row_scaled /
  fp8_add_frag_res_f32: one fma after the e4m3 wgmma sum), then the layer's epilogue.
- `vit_block_fp8`: one ViT block of the fp8 launch sequence (model.dpt_forward): LayerNorm -> quantise -> qkv (bf16
  store) -> attention (gemm_oracle.attention_bf16, bf16 store) -> quantise -> proj + fp32 residual -> LayerNorm ->
  quantise -> fc1 + GELU (bf16 store) -> quantise -> fc2 + fp32 residual.  The rest of the network is the bf16 path.
"""
import torch
import torch.nn.functional as F

from .gemm_oracle import attention_bf16

E4M3 = torch.float8_e4m3fn


def quantize_rows_e4m3(x: torch.Tensor):
    """(q e4m3, s fp32 [rows]) of fp32 rows x [rows, C]: amax = max |x|, s = amax / 448, q = e4m3_rn_satfinite(x * fp32(448 /
    amax)), IEEE divisions (tensor by tensor); an all-zero row: s = 1, q = x * 0."""
    x = x.float()
    amax = x.abs().amax(dim=-1)
    nz = amax > 0
    c = torch.full_like(amax, 448.0)
    safe = torch.where(nz, amax, torch.ones_like(amax))
    s = torch.where(nz, safe / c, torch.ones_like(amax))
    inv = torch.where(nz, c / safe, torch.zeros_like(amax))
    return (x * inv[..., None]).clamp(-448.0, 448.0).to(E4M3), s


def linear_fp8_ref(qa, sa, qw, sw, bias, act: str = "none", residual=None) -> torch.Tensor:
    """float64 value of the scaled GEMM: (qa qw^T) * (sa[r] sw[c]) + bias[c], then GELU (act "gelu") or + residual."""
    acc = qa.double() @ qw.double().t()
    v = acc * (sa.double()[:, None] * sw.double()[None, :]) + bias.double()[None, :]
    if act == "gelu":
        v = F.gelu(v)
    if residual is not None:
        v = v + residual.double()
    return v


def linear_fp8_abs(qa, sa, qw, sw) -> torch.Tensor:
    """sum_k |qa qw| * sa sw: the magnitude the e4m3 wgmma sum's error is measured against."""
    return (qa.double().abs() @ qw.double().abs().t()) * (sa.double()[:, None] * sw.double()[None, :])


def _bf16(t):
    return t.to(torch.bfloat16).double()


def vit_block_fp8(x: torch.Tensor, sd: dict, prefix: str, heads: int) -> torch.Tensor:
    """Block `prefix` (e.g. "pretrained.model.blocks.3.") of the fp8 mode on its fp32 input stream x [B, T, D]; returns
    the block's output stream in float64.  Weights are quantised from the fp32 parameters by the same rule."""
    B, T, D = x.shape
    g = lambda k: sd[prefix + k].to(x.device)
    wq = {n: quantize_rows_e4m3(g(n + ".weight").float()) for n in ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2")}

    def lin(h, n, **kw):
        qa, sa = quantize_rows_e4m3(h.reshape(B * T, -1))
        return linear_fp8_ref(qa, sa, *wq[n], g(n + ".bias").float(), **kw).view(B, T, -1)

    x = x.double()
    h = F.layer_norm(x.float(), (D,), g("norm1.weight").float(), g("norm1.bias").float(), 1e-6)
    qkv = _bf16(lin(h, "attn.qkv"))
    q, k, v = qkv.view(B, T, 3, heads, 64).permute(2, 0, 3, 1, 4)
    a = _bf16(attention_bf16(q, k, v).permute(0, 2, 1, 3).reshape(B, T, D))
    x = lin(a.float(), "attn.proj", residual=x.reshape(B * T, D)).float().double()       # the stream is stored fp32
    h = F.layer_norm(x.float(), (D,), g("norm2.weight").float(), g("norm2.bias").float(), 1e-6)
    m = _bf16(lin(h, "mlp.fc1", act="gelu"))
    return lin(m.float(), "mlp.fc2", residual=x.reshape(B * T, D)).float().double()
