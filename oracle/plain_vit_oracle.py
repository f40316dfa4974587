"""TEST INFRASTRUCTURE — functional CPU restatement of the reference DPTs with a plain ViT/16 encoder (backbones
`vitl16_384` = DPT-Large and `vitb16_384`), the counterpart of oracle/dpt_oracle.py::forward_fp32 for the hybrid.

`forward_fp32(sd, x)` follows the reference dataflow operation by operation in plain PyTorch over a reference-layout
state_dict (citations are into the reference's omnidata_tools/torch/; "timm" = timm 0.4.12, restated in
oracle/timm_shim).  It is validated against the golden vectors of the UNMODIFIED reference class
(oracle/make_golden.py::make_large_golden, tests/test_plain_vit_oracle_cpu.py); with dtype=torch.float64 it is the
gradient truth of the plain-ViT train step's tests.  The decoder and head after the reassemble are the same
operations as the hybrid's restatement.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

P = "pretrained.model."


def forward_fp32(sd: Dict[str, torch.Tensor], x: torch.Tensor, taps: Optional[dict] = None,
                 non_negative: bool = True, dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """DPTDepthModel.forward (modules/midas/dpt_depth.py:106-107) with a plain ViT/16 encoder: timm PatchEmbed, cls,
    pos (resized off the 24 x 24 grid), the ViT blocks hooked at depth/4 - 1, depth/2 - 1, 3 depth/4 - 1, depth - 1
    (5/11/17/23 or 2/5/8/11), and the four readouts with act_postprocess1..4 (modules/midas/vit.py:185-318):
    ProjectReadout, conv1x1, then ConvTranspose 4/4 and 2/2, identity, conv3x3 s2."""
    taps = {} if taps is None else taps
    g = lambda k: sd[k].to(dtype)
    x = x.to(dtype)
    B = x.shape[0]
    D = sd[P + "cls_token"].shape[-1]
    heads = D // 64
    depth = len({k.split(".")[3] for k in sd if k.startswith(P + "blocks.")})
    hooks = tuple(depth // 4 * (j + 1) - 1 for j in range(4))

    # ---- forward_flex (modules/midas/vit.py:119-155): patch embedding, cls, pos, blocks (final norm is dead)
    tok = F.conv2d(x, g(P + "patch_embed.proj.weight"), g(P + "patch_embed.proj.bias"), stride=16)
    gh, gw = tok.shape[-2:]
    tok = tok.flatten(2).transpose(1, 2)
    tok = torch.cat((g(P + "cls_token").expand(B, -1, -1), tok), dim=1)
    pos = g(P + "pos_embed")
    if (gh, gw) != (24, 24):  # _resize_pos_embed (modules/midas/vit.py:102-116)
        grid = pos[0, 1:].reshape(1, 24, 24, -1).permute(0, 3, 1, 2)
        grid = F.interpolate(grid, size=(gh, gw), mode="bilinear")
        pos = torch.cat([pos[:, :1], grid.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)], dim=1)
    tok = tok + pos
    hooked = []
    for i in range(depth):
        p = f"{P}blocks.{i}."
        h = F.layer_norm(tok, (D,), g(p + "norm1.weight"), g(p + "norm1.bias"), 1e-6)
        qkv = F.linear(h, g(p + "attn.qkv.weight"), g(p + "attn.qkv.bias"))
        N = qkv.shape[1]
        q, k, v = qkv.reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
        a = ((q @ k.transpose(-2, -1)) * 0.125).softmax(dim=-1) @ v
        a = a.transpose(1, 2).reshape(B, N, D)
        tok = tok + F.linear(a, g(p + "attn.proj.weight"), g(p + "attn.proj.bias"))
        h = F.layer_norm(tok, (D,), g(p + "norm2.weight"), g(p + "norm2.bias"), 1e-6)
        h = F.gelu(F.linear(h, g(p + "mlp.fc1.weight"), g(p + "mlp.fc1.bias")))
        tok = tok + F.linear(h, g(p + "mlp.fc2.weight"), g(p + "mlp.fc2.bias"))
        if i in hooks:
            hooked.append(tok)
            taps[f"tokens_{i}"] = tok

    # ---- forward_vit reassemble (modules/midas/vit.py:61-99, 185-318)
    layers = []
    for n, tk in zip((1, 2, 3, 4), hooked):
        pp = f"pretrained.act_postprocess{n}."
        cls = tk[:, :1].expand(-1, tk.shape[1] - 1, -1)                      # ProjectReadout (vit.py:43-47)
        f = F.gelu(F.linear(torch.cat((tk[:, 1:], cls), -1), g(pp + "0.project.0.weight"),
                            g(pp + "0.project.0.bias")))
        f = f.transpose(1, 2).reshape(B, D, gh, gw)                          # Transpose + Unflatten
        f = F.conv2d(f, g(pp + "3.weight"), g(pp + "3.bias"))
        if n in (1, 2):                                                      # ConvTranspose2d(c, c, k, stride k)
            f = F.conv_transpose2d(f, g(pp + "4.weight"), g(pp + "4.bias"), stride=4 if n == 1 else 2)
        elif n == 4:
            f = F.conv2d(f, g(pp + "4.weight"), g(pp + "4.bias"), stride=2, padding=1)
        layers.append(f)
        taps[f"layer_{n}"] = f

    # ---- DPT.forward decoder (modules/midas/dpt_depth.py:73-83)
    rn = [F.conv2d(l, g(f"scratch.layer{i}_rn.weight"), None, padding=1) for i, l in zip((1, 2, 3, 4), layers)]
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
