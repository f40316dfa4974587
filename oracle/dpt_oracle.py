"""TEST INFRASTRUCTURE — functional CPU restatement of the reference DPT-Hybrid-384 forward.

`forward_fp32(sd, x)` follows the reference dataflow operation by operation in plain PyTorch fp32
over a reference-layout state_dict (citations are into the reference's omnidata_tools/torch/;
"timm" = timm 0.4.12, third-party, restated in oracle/timm_shim).  It is validated in the build
container against the UNMODIFIED reference module (oracle/make_golden.py, tests/test_oracle_cpu.py)
and is what the GPU tests compare taps against (the reference is not part of this repository).

`forward_bf16(sd, x)` is the same arithmetic with the product's rounding points: operands are
bf16, accumulation and elementwise math are fp32, and a value is rounded to bf16 exactly where
the CUDA pipeline stores it to HBM (DESIGN.md "rounding points"); the ViT residual stream stays fp32
and GroupNorm statistics are taken from the unrounded conv output, as in the product.  It also applies the two
algebraic re-orderings the product uses (1x1 out_conv before the bilinear upsample; ProjectReadout
weight split), which are exact in real arithmetic.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .gemm_oracle import attention_bf16

# the wgmma attention kernel's rounding points, defined once in gemm_oracle (kept under this name for its callers)
_attention_bf16 = attention_bf16

P = "pretrained.model."
BB = P + "patch_embed.backbone."


# ----------------------------------------------------------------------------- shared pieces
def std_weight(w: torch.Tensor, eps: float = 1e-8) -> torch.Tensor:
    """timm StdConv2dSame: per-output-channel standardisation, biased std, (w - mean) / (std + eps)."""
    std, mean = torch.std_mean(w, dim=[1, 2, 3], keepdim=True, unbiased=False)
    return (w - mean) / (std + eps)


def same_pad(x: torch.Tensor, k: int, s: int, value: float = 0.0) -> torch.Tensor:
    """TF-SAME padding (timm pad_same): total = max((ceil(n/s)-1)*s + k - n, 0), before = total // 2."""
    def tot(n):
        return max((math.ceil(n / s) - 1) * s + k - n, 0)
    ph, pw = tot(x.shape[-2]), tot(x.shape[-1])
    if ph or pw:
        x = F.pad(x, [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2], value=value)
    return x


def _ident(t):
    return t


def _bf16(t):
    return t.to(torch.bfloat16).float()


# ----------------------------------------------------------------------------- fp32, reference order
def forward_fp32(sd: Dict[str, torch.Tensor], x: torch.Tensor, taps: Optional[dict] = None,
                 non_negative: bool = True, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """DPTDepthModel.forward (modules/midas/dpt_depth.py:106-107) == DPT.forward(x).squeeze(1).
    dtype=torch.float64 evaluates the same arithmetic in double precision: the 'exact' reference against which the
    fp32 noise of both the reference and this repo is measured (gradient tests)."""
    taps = {} if taps is None else taps
    g = lambda k: sd[k].to(dtype)
    x = x.to(dtype)

    # ---- timm ResNetV2 stem + stages (hooks "1","2": modules/midas/vit.py:363-368)
    def sconv(t, key, stride=1):
        w = std_weight(g(key))
        return F.conv2d(same_pad(t, w.shape[-1], stride), w, None, stride)

    def gn(t, prefix, act):
        t = F.group_norm(t, 32, g(prefix + ".weight"), g(prefix + ".bias"), 1e-5)
        return F.relu(t) if act else t

    t = gn(sconv(x, BB + "stem.conv.weight", 2), BB + "stem.norm", True)
    t = F.max_pool2d(same_pad(t, 3, 2, float("-inf")), 3, 2)
    feats = []
    for s, depth in enumerate((3, 4, 9)):
        for b in range(depth):
            p = f"{BB}stages.{s}.blocks.{b}."
            stride = 2 if (b == 0 and s > 0) else 1
            sc = t
            if b == 0:
                sc = gn(sconv(t, p + "downsample.conv.weight", stride), p + "downsample.norm", False)
            y = gn(sconv(t, p + "conv1.weight"), p + "norm1", True)
            y = gn(sconv(y, p + "conv2.weight", stride), p + "norm2", True)
            y = gn(sconv(y, p + "conv3.weight"), p + "norm3", False)
            t = F.relu(y + sc)
        feats.append(t)
    taps["layer_1_pre"], taps["layer_2_pre"] = feats[0], feats[1]

    # ---- forward_flex (modules/midas/vit.py:119-155): proj, cls, pos, 12 blocks (final norm is dead)
    B = x.shape[0]
    tok = F.conv2d(feats[2], g(P + "patch_embed.proj.weight"), g(P + "patch_embed.proj.bias"))
    gh, gw = tok.shape[-2:]
    tok = tok.flatten(2).transpose(1, 2)
    tok = torch.cat((g(P + "cls_token").expand(B, -1, -1), tok), dim=1)
    pos = g(P + "pos_embed")
    if (gh, gw) != (24, 24):  # _resize_pos_embed (modules/midas/vit.py:102-116)
        grid = pos[0, 1:].reshape(1, 24, 24, -1).permute(0, 3, 1, 2)
        grid = F.interpolate(grid, size=(gh, gw), mode="bilinear")
        pos = torch.cat([pos[:, :1], grid.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)], dim=1)
    tok = tok + pos
    hooked = {}
    for i in range(12):
        p = f"{P}blocks.{i}."
        h = F.layer_norm(tok, (768,), g(p + "norm1.weight"), g(p + "norm1.bias"), 1e-6)
        qkv = F.linear(h, g(p + "attn.qkv.weight"), g(p + "attn.qkv.bias"))
        N = qkv.shape[1]
        q, k, v = qkv.reshape(B, N, 3, 12, 64).permute(2, 0, 3, 1, 4)
        a = ((q @ k.transpose(-2, -1)) * 0.125).softmax(dim=-1) @ v
        a = a.transpose(1, 2).reshape(B, N, 768)
        tok = tok + F.linear(a, g(p + "attn.proj.weight"), g(p + "attn.proj.bias"))
        h = F.layer_norm(tok, (768,), g(p + "norm2.weight"), g(p + "norm2.bias"), 1e-6)
        h = F.gelu(F.linear(h, g(p + "mlp.fc1.weight"), g(p + "mlp.fc1.bias")))
        tok = tok + F.linear(h, g(p + "mlp.fc2.weight"), g(p + "mlp.fc2.bias"))
        if i in (8, 11):
            hooked[i] = tok
    taps["tokens_8"], taps["tokens_11"] = hooked[8], hooked[11]

    # ---- forward_vit reassemble (modules/midas/vit.py:61-99, 431-462)
    def readout(tk, n):
        pp = f"pretrained.act_postprocess{n}."
        cls = tk[:, :1].expand(-1, tk.shape[1] - 1, -1)                      # ProjectReadout :43-47
        f = F.gelu(F.linear(torch.cat((tk[:, 1:], cls), -1), g(pp + "0.project.0.weight"),
                            g(pp + "0.project.0.bias")))
        f = f.transpose(1, 2).reshape(B, 768, gh, gw)                        # Transpose + Unflatten
        return F.conv2d(f, g(pp + "3.weight"), g(pp + "3.bias"))
    layer_1, layer_2 = feats[0], feats[1]
    layer_3 = readout(hooked[8], 3)
    layer_4 = readout(hooked[11], 4)
    layer_4 = F.conv2d(layer_4, g("pretrained.act_postprocess4.4.weight"),
                       g("pretrained.act_postprocess4.4.bias"), stride=2, padding=1)
    taps.update(layer_1=layer_1, layer_2=layer_2, layer_3=layer_3, layer_4=layer_4)

    # ---- DPT.forward decoder (modules/midas/dpt_depth.py:73-83)
    rn = [F.conv2d(l, g(f"scratch.layer{i}_rn.weight"), None, padding=1)
          for i, l in zip((1, 2, 3, 4), (layer_1, layer_2, layer_3, layer_4))]
    for i in range(4):
        taps[f"layer_{i + 1}_rn"] = rn[i]

    def rcu(t, prefix):                                                      # modules/midas/blocks.py:263-286
        o = F.conv2d(F.relu(t), g(prefix + "conv1.weight"), g(prefix + "conv1.bias"), padding=1)
        o = F.conv2d(F.relu(o), g(prefix + "conv2.weight"), g(prefix + "conv2.bias"), padding=1)
        return o + t

    def fusion(n, *xs):                                                      # modules/midas/blocks.py:320-341
        p = f"scratch.refinenet{n}."
        o = xs[0]
        if len(xs) == 2:
            o = o + rcu(xs[1], p + "resConfUnit1.")
        o = rcu(o, p + "resConfUnit2.")
        o = F.interpolate(o, scale_factor=2, mode="bilinear", align_corners=True)
        return F.conv2d(o, g(p + "out_conv.weight"), g(p + "out_conv.bias"))

    path_4 = fusion(4, rn[3])
    path_3 = fusion(3, path_4, rn[2])
    path_2 = fusion(2, path_3, rn[1])
    path_1 = fusion(1, path_2, rn[0])
    taps.update(path_4=path_4, path_3=path_3, path_2=path_2, path_1=path_1)

    # ---- head (modules/midas/dpt_depth.py:91-99)
    o = F.conv2d(path_1, g("scratch.output_conv.0.weight"), g("scratch.output_conv.0.bias"), padding=1)
    o = F.interpolate(o, scale_factor=2, mode="bilinear", align_corners=True)
    o = F.relu(F.conv2d(o, g("scratch.output_conv.2.weight"), g("scratch.output_conv.2.bias"), padding=1))
    o = F.conv2d(o, g("scratch.output_conv.4.weight"), g("scratch.output_conv.4.bias"))
    taps["head_pre_relu"] = o
    if non_negative:
        o = F.relu(o)
    return o.squeeze(1)


# ----------------------------------------------------------------------------- product rounding points
def _attention_online_bf16(q, k, v, chunk: int = 64):
    """Arithmetic of the legacy mma.sync kernel (attention.cu): flash-style online softmax over
    64-key chunks, P of a chunk rounded to bf16, fp32 running row sum of the unrounded values."""
    scale_log2e = float(torch.tensor(0.125, dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32))
    n = q.shape[-2]
    o = torch.zeros_like(q)
    m = torch.full(q.shape[:-1], float("-inf"), dtype=q.dtype, device=q.device)
    l = torch.zeros(q.shape[:-1], dtype=q.dtype, device=q.device)
    for c0 in range(0, n, chunk):
        s_ = (q @ k[..., c0:c0 + chunk, :].transpose(-2, -1)) * scale_log2e
        m_new = torch.maximum(m, s_.amax(dim=-1))
        alpha = torch.exp2(m - m_new)
        p = torch.exp2(s_ - m_new[..., None])
        l = l * alpha + p.sum(dim=-1)
        o = o * alpha[..., None] + _bf16(p) @ v[..., c0:c0 + chunk, :]
        m = m_new
    return o / l[..., None]


def forward_bf16(sd: Dict[str, torch.Tensor], x: torch.Tensor, taps: Optional[dict] = None,
                 non_negative: bool = True) -> torch.Tensor:
    """Same network with bf16 operands / fp32 accumulation and a bf16 rounding wherever the CUDA
    pipeline (omnidata_b200/model.py) stores an activation.  NCHW fp32 tensors holding bf16 values."""
    taps = {} if taps is None else taps
    g = lambda k: sd[k].float()
    r = _bf16
    wq = lambda t: t.to(torch.bfloat16).float()          # weights are stored in bf16
    B = x.shape[0]

    def sconv(t, key, stride=1):
        """-> (conv output rounded to bf16 as stored, GroupNorm statistics of the UNROUNDED fp32 output: the conv
        epilogue sums its fp32 accumulators, like timm GroupNormAct which normalises the fp32 conv output)."""
        w = wq(std_weight(g(key)))
        y = F.conv2d(same_pad(t, w.shape[-1], stride), w, None, stride)
        yg = y.double().reshape(y.shape[0], 32, -1)
        mean = yg.mean(dim=2)
        var = (yg * yg).mean(dim=2) - mean * mean
        rstd = 1.0 / torch.sqrt(var.clamp_min(0) + 1e-5)
        return r(y), (mean.float(), rstd.float())

    def gn_raw(ys, prefix):
        y, (mean, rstd) = ys
        Bn, Cn = y.shape[:2]
        cpg = Cn // 32
        a = rstd.repeat_interleave(cpg, dim=1) * g(prefix + ".weight")[None]                 # [B, C]
        sh = g(prefix + ".bias")[None] - mean.repeat_interleave(cpg, dim=1) * a
        return y * a[:, :, None, None] + sh[:, :, None, None]

    xin = r(x.float())                                    # im2col stores the image as bf16
    s0 = sconv(xin, BB + "stem.conv.weight", 2)
    taps["stem_conv"] = s0[0]
    t = F.relu(gn_raw(s0, BB + "stem.norm"))
    t = r(F.max_pool2d(same_pad(t, 3, 2, float("-inf")), 3, 2))
    taps["stem_pool"] = t
    feats = []
    for s, depth in enumerate((3, 4, 9)):
        for b in range(depth):
            p = f"{BB}stages.{s}.blocks.{b}."
            stride = 2 if (b == 0 and s > 0) else 1
            sc = t
            if b == 0:
                sc = gn_raw(sconv(t, p + "downsample.conv.weight", stride), p + "downsample.norm")
            y = r(F.relu(gn_raw(sconv(t, p + "conv1.weight"), p + "norm1")))
            y = r(F.relu(gn_raw(sconv(y, p + "conv2.weight", stride), p + "norm2")))
            y = gn_raw(sconv(y, p + "conv3.weight"), p + "norm3")
            t = r(F.relu(y + sc))
            taps[f"s{s}b{b}_out"] = t
        feats.append(t)

    gh, gw = feats[2].shape[-2:]
    pos = g(P + "pos_embed")
    if (gh, gw) != (24, 24):  # _resize_pos_embed (modules/midas/vit.py:102-116), done once at pre-pack time
        grid = pos[0, 1:].reshape(1, 24, 24, -1).permute(0, 3, 1, 2)
        grid = F.interpolate(grid, size=(gh, gw), mode="bilinear")
        pos = torch.cat([pos[:, :1], grid.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)], dim=1)
    # the residual stream is fp32 (proj / fc2 epilogues add into fp32 storage; LayerNorm reads fp32): no rounding
    tok = F.conv2d(feats[2], wq(g(P + "patch_embed.proj.weight")), g(P + "patch_embed.proj.bias"))
    tok = tok.flatten(2).transpose(1, 2) + pos[:, 1:]
    cls = (g(P + "cls_token") + pos[:, :1]).expand(B, -1, -1)
    tok = torch.cat((cls, tok), dim=1)
    taps["tokens_in"] = tok
    hooked = {}
    for i in range(12):
        p = f"{P}blocks.{i}."
        h = r(F.layer_norm(tok, (768,), g(p + "norm1.weight"), g(p + "norm1.bias"), 1e-6))
        qkv = r(F.linear(h, wq(g(p + "attn.qkv.weight")), g(p + "attn.qkv.bias")))
        N = qkv.shape[1]
        q, k, v = qkv.reshape(B, N, 3, 12, 64).permute(2, 0, 3, 1, 4)
        a = attention_bf16(q, k, v)
        a = r(a.transpose(1, 2).reshape(B, N, 768))
        tok = tok + F.linear(a, wq(g(p + "attn.proj.weight")), g(p + "attn.proj.bias"))
        h = r(F.layer_norm(tok, (768,), g(p + "norm2.weight"), g(p + "norm2.bias"), 1e-6))
        h = r(F.gelu(F.linear(h, wq(g(p + "mlp.fc1.weight")), g(p + "mlp.fc1.bias"))))
        tok = tok + F.linear(h, wq(g(p + "mlp.fc2.weight")), g(p + "mlp.fc2.bias"))
        taps[f"tokens_{i}"] = tok
        if i in (8, 11):
            hooked[i] = tok

    def readout(tk, n):
        pp = f"pretrained.act_postprocess{n}."
        tk = r(tk)                       # the hooked activation leaves the fp32 stream as a bf16 GEMM operand
        w = wq(g(pp + "0.project.0.weight"))
        cls_term = F.linear(tk[:, 0], w[:, 768:], g(pp + "0.project.0.bias"))       # fp32 [B,768]
        f = r(F.gelu(F.linear(tk[:, 1:], w[:, :768]) + cls_term[:, None, :]))
        f = f.transpose(1, 2).reshape(B, 768, gh, gw)
        return r(F.conv2d(f, wq(g(pp + "3.weight")), g(pp + "3.bias")))
    layer_1, layer_2 = feats[0], feats[1]
    layer_3 = readout(hooked[8], 3)
    layer_4 = readout(hooked[11], 4)
    layer_4 = r(F.conv2d(layer_4, wq(g("pretrained.act_postprocess4.4.weight")),
                         g("pretrained.act_postprocess4.4.bias"), stride=2, padding=1))
    taps.update(layer_1=layer_1, layer_2=layer_2, layer_3=layer_3, layer_4=layer_4)

    rn = [r(F.conv2d(l, wq(g(f"scratch.layer{i}_rn.weight")), None, padding=1))
          for i, l in zip((1, 2, 3, 4), (layer_1, layer_2, layer_3, layer_4))]
    for i in range(4):
        taps[f"layer_{i + 1}_rn"] = rn[i]

    def rcu(t, prefix):
        o = r(F.relu(F.conv2d(r(F.relu(t)), wq(g(prefix + "conv1.weight")), g(prefix + "conv1.bias"), padding=1)))
        return r(F.conv2d(o, wq(g(prefix + "conv2.weight")), g(prefix + "conv2.bias"), padding=1) + t)

    def up(t):
        return F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=True)

    def fusion_lowres(n, s_):
        """RCU2 then the (commuted) 1x1 out_conv at the block's input resolution."""
        p = f"scratch.refinenet{n}."
        y = rcu(s_, p + "resConfUnit2.")
        return r(F.conv2d(y, wq(g(p + "out_conv.weight")), g(p + "out_conv.bias")))

    z = fusion_lowres(4, rn[3])
    taps["path_4"] = r(up(z))
    for n, lrn in ((3, rn[2]), (2, rn[1]), (1, rn[0])):
        res = rcu(lrn, f"scratch.refinenet{n}.resConfUnit1.")
        s_ = r(up(z) + res)
        z = fusion_lowres(n, s_)
        taps[f"path_{n}"] = r(up(z))
    path_1 = taps["path_1"]

    o = r(F.conv2d(path_1, wq(g("scratch.output_conv.0.weight")), g("scratch.output_conv.0.bias"), padding=1))
    o = r(up(o))
    o = F.relu(F.conv2d(o, wq(g("scratch.output_conv.2.weight")), g("scratch.output_conv.2.bias"), padding=1))
    o = F.conv2d(o, g("scratch.output_conv.4.weight"), g("scratch.output_conv.4.bias"))   # fp32 weights
    taps["head_pre_relu"] = o
    if non_negative:
        o = F.relu(o)
    return o.squeeze(1)
