"""DPT-Hybrid-384 (`vitb_rn50_384`) dense-prediction model, H100-native.

Drop-in for the reference's `modules/midas/dpt_depth.py::DPTDepthModel` (constructor kwargs,
`state_dict()` keys / shapes / order, `forward(x)` contract: float NCHW in, `[B,H,W]` (1 channel)
or `[B,C,H,W]` out, final ReLU when `non_negative`).  The arithmetic runs in the sm_90a kernels
of `omnidata_b200/csrc` through the C ABI (`include/omnidata_b200.h`); this file is host-side
orchestration only: weight pre-packing at load time, workspace management, launch order and
optional CUDA-graph replay.  There is no CPU / eager fallback — `forward` on a CPU tensor raises.

Reference call stack mirrored here (omnidata_tools/torch/): DPT.forward `modules/midas/dpt_depth.py:67-85`,
forward_vit / forward_flex `modules/midas/vit.py:61-155`, reassemble `vit.py:431-462`,
FeatureFusionBlock_custom / ResidualConvUnit_custom `modules/midas/blocks.py:231-341`,
head `dpt_depth.py:91-99`; encoder arithmetic is timm 0.4.12 `vit_base_resnet50_384` (`vit.py:483`).
"""
from __future__ import annotations

import math
from typing import Dict, List, NamedTuple, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import bwd, ops
from ._capi import OdbError

_STAGES = ((256, 3), (512, 4), (1024, 9))   # timm ResNetV2(layers=(3,4,9)) widths / depths
_FEATURES = 256
# Encoders behind the same decoder (modules/midas/blocks.py:12-47 _make_encoder, dpt_depth.py:41-45 hooks):
#   vitb_rn50_384  DPT-Hybrid: ResNetV2 stages 0/1 give layer_1/2, ViT-B blocks 8/11 give layer_3/4
#   vitl16_384     DPT-Large (SURVEY 8(f) rank 3): plain ViT-L/16, blocks 5/11/17/23 give layer_1..4
#                  (vit.py:185-290: conv1x1 then ConvTranspose 4x4/s4, 2x2/s2, identity, conv3x3/s2)
_ARCH = {
    "vitb_rn50_384": dict(embed=768, heads=12, depth=12, hybrid=True, hooks=(8, 11), rn_in=(256, 512, 768, 768)),
    "vitl16_384": dict(embed=1024, heads=16, depth=24, hybrid=False, hooks=(5, 11, 17, 23),
                       rn_in=(256, 512, 1024, 1024)),
    #   vitb16_384   plain ViT-B/16, blocks 2/5/8/11, reassemble widths 96/192/384/768 (vit.py:311-318); the 96
    #                channels are carried zero-padded to 128 internally (the GEMM N tile is a multiple of 64)
    "vitb16_384": dict(embed=768, heads=12, depth=12, hybrid=False, hooks=(2, 5, 8, 11),
                       rn_in=(96, 192, 384, 768)),
}

# Input sizes (H, W multiples of 32).  Inference takes up to MAX_PATCHES patches: the attention kernels take up to
# 4 097 tokens.  Training and x.grad take up to MAX_TRAIN_PATCHES: the attention backward materialises P and dS per
# (image, head) for up to 640 tokens.
MAX_PATCHES = 4096
MAX_TRAIN_PATCHES = 639
STEM_MAX_W = 1792          # DPT-Hybrid: the stem im2col stages 21 input rows of W + 5 floats in shared memory


def check_input_size(H: int, W: int, hybrid: bool, autograd: bool) -> None:
    """Raises ValueError, before anything is launched, for an input size the launch sequence cannot take: the
    differentiable forward (autograd) up to MAX_TRAIN_PATCHES patches, inference up to MAX_PATCHES."""
    patches = (H // 16) * (W // 16)
    if H % 32 or W % 32 or patches > MAX_TRAIN_PATCHES:
        if autograd:
            raise ValueError(f"H and W must be multiples of 32 with at most {MAX_TRAIN_PATCHES} patches for training "
                             f"and x.grad, got {H}x{W}")
        if H % 32 or W % 32 or patches > MAX_PATCHES:
            raise ValueError(f"H and W must be multiples of 32 with at most {MAX_PATCHES} patches, got {H}x{W}")
        # sizes beyond 639 patches: what the kernels of the launch sequence take
        if min(H, W) < 64:
            raise ValueError(f"H and W must be at least 64 (the 1/32 decoder map is upsampled from 2x2), got {H}x{W}")
        if hybrid and W > STEM_MAX_W:
            raise ValueError(f"DPT-Hybrid: W must be at most {STEM_MAX_W} (stem convolution), got {W}")


def _rn_pad(arch: dict) -> Tuple[int, ...]:
    """reassemble widths, zero-padded to the GEMM's N granularity"""
    return tuple((c + 63) // 64 * 64 for c in arch["rn_in"])


class GemmLayer(NamedTuple):
    """One GEMM layer of the DPT.  Parameter `weight` is read as [n][c][taps]; its forward operand is
    [n_pad][taps * c_pad], tap-major, the padded rows / columns zero.  `bias` names the bias parameter (None: no bias);
    `standardize`: timm StdConv2dSame weight standardisation (the ResNetV2 convolutions)."""
    key: str
    weight: str
    bias: Optional[str]
    n: int
    c: int
    taps: int
    n_pad: int
    c_pad: int
    standardize: bool


def _rcu_layers(n: int, u: int) -> List[GemmLayer]:
    p = f"scratch.refinenet{n}.resConfUnit{u}."
    return [GemmLayer(f"ff{n}.rcu{u}.c{cv}", f"{p}conv{cv}.weight", f"{p}conv{cv}.bias", 256, 256, 9, 256, 256, False)
            for cv in (1, 2)]


def gemm_layers(arch: dict) -> List[GemmLayer]:
    """Every GEMM layer of the DPT with encoder `arch` (an `_ARCH` entry) whose operands the packers build from a weight
    of the state dict, in the order of the train engine's packing tables.  Not listed: the hybrid's 7x7 stem (im2col
    operand) and the readout Linear layers (split into token and cls halves)."""
    L = []
    pm, D = "pretrained.model.", arch["embed"]
    rn_in, rn_pad = arch["rn_in"], _rn_pad(arch)
    if arch["hybrid"]:
        bb = pm + "patch_embed.backbone."
        cin = 64
        for s, (cout, depth) in enumerate(_STAGES):
            mid = cout // 4
            for b in range(depth):
                p = f"{bb}stages.{s}.blocks.{b}."
                if b == 0:
                    L.append(GemmLayer(f"s{s}b{b}.wd", p + "downsample.conv.weight", None, cout, cin, 1, cout, cin,
                                       True))
                c1 = cin if b == 0 else cout
                L.append(GemmLayer(f"s{s}b{b}.w1", p + "conv1.weight", None, mid, c1, 1, mid, c1, True))
                L.append(GemmLayer(f"s{s}b{b}.w2", p + "conv2.weight", None, mid, mid, 9, mid, mid, True))
                L.append(GemmLayer(f"s{s}b{b}.w3", p + "conv3.weight", None, cout, mid, 1, cout, mid, True))
            cin = cout
        c_proj = 1024
    else:
        c_proj = 3 * 16 * 16                        # Conv2d(3, D, 16, stride 16) over patchify's columns
    L.append(GemmLayer("proj", pm + "patch_embed.proj.weight", pm + "patch_embed.proj.bias", D, c_proj, 1, D, c_proj,
                       False))
    for i in range(arch["depth"]):
        p = f"{pm}blocks.{i}."
        for key, name, n, c in (("qkv", "attn.qkv", 3 * D, D), ("proj", "attn.proj", D, D),
                                ("fc1", "mlp.fc1", 4 * D, D), ("fc2", "mlp.fc2", D, 4 * D)):
            L.append(GemmLayer(f"blk{i}.{key}", p + name + ".weight", p + name + ".bias", n, c, 1, n, c, False))
    for n in ((3, 4) if arch["hybrid"] else (1, 2, 3, 4)):
        p = f"pretrained.act_postprocess{n}."
        L.append(GemmLayer(f"pp{n}", p + "3.weight", p + "3.bias", rn_in[n - 1], D, 1, rn_pad[n - 1], D, False))
    if not arch["hybrid"]:
        # ConvTranspose2d(c, c, k, stride k), weight [in][out][k][k] read as n = in, c = out, taps = (ky, kx): the
        # forward operand [in][(ky, kx, out)] is the input-gradient operand, the dgrad operand's tap blocks the
        # forward's per-phase 1x1 operands
        for n, k in ((1, 4), (2, 2)):
            p, c, cp = f"pretrained.act_postprocess{n}.", rn_in[n - 1], rn_pad[n - 1]
            L.append(GemmLayer(f"pp{n}t", p + "4.weight", p + "4.bias", c, c, k * k, cp, cp, False))
    L.append(GemmLayer("pp4s", "pretrained.act_postprocess4.4.weight", "pretrained.act_postprocess4.4.bias",
                       D, D, 9, D, D, False))
    for n in (1, 2, 3, 4):
        L.append(GemmLayer(f"rn{n}", f"scratch.layer{n}_rn.weight", None, 256, rn_in[n - 1], 9, 256, rn_pad[n - 1],
                           False))
    for n in (1, 2, 3, 4):
        p = f"scratch.refinenet{n}."
        L.append(GemmLayer(f"ff{n}.out", p + "out_conv.weight", p + "out_conv.bias", 256, 256, 1, 256, 256, False))
        for u in ((2,) if n == 4 else (1, 2)):      # refinenet4.resConfUnit1 is dead (blocks.py:328-330)
            L += _rcu_layers(n, u)
    L.append(GemmLayer("head0", "scratch.output_conv.0.weight", "scratch.output_conv.0.bias", 128, 256, 9, 128, 256,
                       False))
    # the train forward carries head conv2's 32 channels zero-padded to 64 (its unfused ReLU output feeds the backward)
    L.append(GemmLayer("head2", "scratch.output_conv.2.weight", "scratch.output_conv.2.bias", 32, 128, 9, 64, 128,
                       False))
    return L


def _forward_vectors(backbone: str) -> List[str]:
    """The parameters besides the GEMM layers' biases that dpt_forward reads as fp32 tensors: the norm affines, the cls
    token, the readout Linear biases and the head's final 1x1 conv (32 -> num_channels)."""
    return [k for k, _ in state_dict_spec(backbone=backbone)
            if (".norm" in k and not k.startswith("pretrained.model.norm."))   # the final ViT norm is dead (vit.py:153)
            or k.endswith(("cls_token", "0.project.0.bias")) or k.startswith("scratch.output_conv.4.")]


def _gemm_operand(w: torch.Tensor, layer: GemmLayer) -> torch.Tensor:
    """Forward operand of `layer`, fp32 [n_pad][taps * c_pad], from its weight `w`: standardised if the layer says so,
    read as [n][c][taps], zero-padded to [n_pad][c_pad], taken tap-major."""
    w = _std_weight(w) if layer.standardize else w.float()
    w = F.pad(w.reshape(layer.n, layer.c, layer.taps), (0, 0, 0, layer.c_pad - layer.c, 0, layer.n_pad - layer.n))
    return w.permute(0, 2, 1).reshape(layer.n_pad, -1)


def quantize_rows_e4m3(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(q e4m3 [n][k], s fp32 [n]) with w ~= q * s[:, None], per row n: amax = max |w[n]|, s = amax / 448,
    q = e4m3_rn_satfinite(w * (448 / amax)); an all-zero row gets s = 1 and q = 0.  The rule the fp8 mode's kernels
    apply to each token of a GEMM input, here for the weights (fp32 ops in torch)."""
    w = w.float()
    amax = w.abs().amax(dim=1)
    nz = amax > 0
    # tensor-by-tensor divisions: IEEE round-to-nearest quotients (a division by a Python scalar may be evaluated as a
    # product with its rounded reciprocal)
    c448 = torch.full_like(amax, 448.0)
    safe = torch.where(nz, amax, torch.ones_like(amax))
    s = torch.where(nz, safe / c448, torch.ones_like(amax))
    inv = torch.where(nz, c448 / safe, torch.zeros_like(amax))
    q = (w * inv[:, None]).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    return q.contiguous(), s.contiguous()


def _decoder_spec(add, num_channels: int, features: int, rn_in) -> None:
    for n, c in zip((1, 2, 3, 4), rn_in):
        add(f"scratch.layer{n}_rn.weight", features, c, 3, 3)
    for n in (1, 2, 3, 4):
        p = f"scratch.refinenet{n}."
        add(p + "out_conv.weight", features, features, 1, 1)
        add(p + "out_conv.bias", features)
        for u in (1, 2):                     # refinenet4.resConfUnit1 is dead (blocks.py:328-330)
            for cv in (1, 2):
                add(f"{p}resConfUnit{u}.conv{cv}.weight", features, features, 3, 3)
                add(f"{p}resConfUnit{u}.conv{cv}.bias", features)
    add("scratch.output_conv.0.weight", features // 2, features, 3, 3)
    add("scratch.output_conv.0.bias", features // 2)
    add("scratch.output_conv.2.weight", 32, features // 2, 3, 3)
    add("scratch.output_conv.2.bias", 32)
    add("scratch.output_conv.4.weight", num_channels, 32, 1, 1)
    add("scratch.output_conv.4.bias", num_channels)


def _vit_blocks_spec(add, pm: str, embed: int, depth: int) -> None:
    for i in range(depth):
        p = f"{pm}blocks.{i}."
        add(p + "norm1.weight", embed)
        add(p + "norm1.bias", embed)
        add(p + "attn.qkv.weight", 3 * embed, embed)
        add(p + "attn.qkv.bias", 3 * embed)
        add(p + "attn.proj.weight", embed, embed)
        add(p + "attn.proj.bias", embed)
        add(p + "norm2.weight", embed)
        add(p + "norm2.bias", embed)
        add(p + "mlp.fc1.weight", 4 * embed, embed)
        add(p + "mlp.fc1.bias", 4 * embed)
        add(p + "mlp.fc2.weight", embed, 4 * embed)
        add(p + "mlp.fc2.bias", embed)
    add(pm + "norm.weight", embed)           # dead in the reference forward (vit.py:153) but present
    add(pm + "norm.bias", embed)
    add(pm + "head.weight", 1000, embed)     # dead: ImageNet classifier of the timm model
    add(pm + "head.bias", 1000)


def _plain_vit_spec(num_channels: int, features: int, arch: dict) -> List[Tuple[str, Tuple[int, ...]]]:
    """DPT with a plain ViT encoder (`vitl16_384`): keys of the reference class instantiated with timm's
    vit_large_patch16_384 (vit.py:185-318), verified against it in tests/test_boundary_cpu.py."""
    spec: List[Tuple[str, Tuple[int, ...]]] = []

    def add(key, *shape):
        spec.append((key, tuple(shape)))

    D = arch["embed"]
    pm = "pretrained.model."
    add(pm + "cls_token", 1, 1, D)
    add(pm + "pos_embed", 1, 577, D)
    add(pm + "patch_embed.proj.weight", D, 3, 16, 16)
    add(pm + "patch_embed.proj.bias", D)
    _vit_blocks_spec(add, pm, D, arch["depth"])
    for n, c in zip((1, 2, 3, 4), arch["rn_in"]):
        p = f"pretrained.act_postprocess{n}."
        add(p + "0.project.0.weight", D, 2 * D)
        add(p + "0.project.0.bias", D)
        add(p + "3.weight", c, D, 1, 1)
        add(p + "3.bias", c)
        if n == 1:
            add(p + "4.weight", c, c, 4, 4)      # ConvTranspose2d(c, c, 4, stride 4): [in, out, kh, kw]
            add(p + "4.bias", c)
        elif n == 2:
            add(p + "4.weight", c, c, 2, 2)      # ConvTranspose2d(c, c, 2, stride 2)
            add(p + "4.bias", c)
        elif n == 4:
            add(p + "4.weight", c, c, 3, 3)      # Conv2d(c, c, 3, stride 2, padding 1)
            add(p + "4.bias", c)
    _decoder_spec(add, num_channels, features, arch["rn_in"])
    return spec


def state_dict_spec(num_channels: int = 1, features: int = _FEATURES,
                    backbone: str = "vitb_rn50_384") -> List[Tuple[str, Tuple[int, ...]]]:
    """(key, shape) in reference `state_dict()` order (SURVEY.md Appendix B; verified against the
    unmodified reference class in tests/test_boundary_cpu.py)."""
    if not _ARCH[backbone]["hybrid"]:
        return _plain_vit_spec(num_channels, features, _ARCH[backbone])
    spec: List[Tuple[str, Tuple[int, ...]]] = []

    def add(key, *shape):
        spec.append((key, tuple(shape)))

    arch = _ARCH[backbone]
    D = arch["embed"]
    pm = "pretrained.model."
    add(pm + "cls_token", 1, 1, D)
    add(pm + "pos_embed", 1, 577, D)
    bb = pm + "patch_embed.backbone."
    add(bb + "stem.conv.weight", 64, 3, 7, 7)
    add(bb + "stem.norm.weight", 64)
    add(bb + "stem.norm.bias", 64)
    cin = 64
    for s, (cout, depth) in enumerate(_STAGES):
        mid = cout // 4
        for b in range(depth):
            p = f"{bb}stages.{s}.blocks.{b}."
            if b == 0:
                add(p + "downsample.conv.weight", cout, cin, 1, 1)
                add(p + "downsample.norm.weight", cout)
                add(p + "downsample.norm.bias", cout)
            add(p + "conv1.weight", mid, cin if b == 0 else cout, 1, 1)
            add(p + "norm1.weight", mid)
            add(p + "norm1.bias", mid)
            add(p + "conv2.weight", mid, mid, 3, 3)
            add(p + "norm2.weight", mid)
            add(p + "norm2.bias", mid)
            add(p + "conv3.weight", cout, mid, 1, 1)
            add(p + "norm3.weight", cout)
            add(p + "norm3.bias", cout)
        cin = cout
    add(pm + "patch_embed.proj.weight", D, 1024, 1, 1)
    add(pm + "patch_embed.proj.bias", D)
    _vit_blocks_spec(add, pm, D, arch["depth"])
    for n in (3, 4):
        p = f"pretrained.act_postprocess{n}."
        add(p + "0.project.0.weight", D, 2 * D)
        add(p + "0.project.0.bias", D)
        add(p + "3.weight", D, D, 1, 1)
        add(p + "3.bias", D)
        if n == 4:
            add(p + "4.weight", D, D, 3, 3)
            add(p + "4.bias", D)
    _decoder_spec(add, num_channels, features, arch["rn_in"])
    return spec


def _std_weight(w: torch.Tensor, eps: float = 1e-8) -> torch.Tensor:
    """timm StdConv2dSame weight standardisation, folded offline for inference."""
    std, mean = torch.std_mean(w.float(), dim=[1, 2, 3], keepdim=True, unbiased=False)
    return (w.float() - mean) / (std + eps)


class _Workspace:
    """Named device buffers, allocated on first use and reused by every later forward.  A name asked for with another
    shape or dtype gets a new buffer: the training engine keeps one workspace across input shapes, while inference
    keeps one per (batch, height, width)."""

    def __init__(self, device):
        self.device = device
        self.bufs: Dict[str, torch.Tensor] = {}

    def get(self, name: str, shape, dtype=torch.bfloat16) -> torch.Tensor:
        t = self.bufs.get(name)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
            t = self.bufs[name] = torch.empty(tuple(shape), device=self.device, dtype=dtype)
        return t


class DPTDepthModel(nn.Module):
    """H100-native DPT-Hybrid; same constructor as the reference (`dpt_depth.py:27-35,88`)."""

    def __init__(self, path: Optional[str] = None, non_negative: bool = True, num_channels: int = 1,
                 backbone: str = "vitb_rn50_384", features: int = 256, readout: str = "project",
                 channels_last: bool = False, use_bn: bool = False, **kwargs):
        super().__init__()
        if backbone not in _ARCH:
            # reference: print + assert False (modules/midas/blocks.py:42-44)
            print(f"Backbone '{backbone}' not implemented")
            raise AssertionError(f"Backbone '{backbone}' not implemented")
        self.backbone = backbone
        self.arch = _ARCH[backbone]
        self._rn_pad = _rn_pad(self.arch)
        if features != 256 or readout != "project" or use_bn:
            raise NotImplementedError("only features=256, readout='project', use_bn=False (the Omnidata DPT-Hybrid)")
        self.non_negative = bool(non_negative)
        self.num_channels = int(num_channels)
        self.channels_last = channels_last        # a no-op in the reference as well (dpt_depth.py:68-69)
        self.use_cuda_graph = False
        self.keep_taps = False                    # tests: keep named intermediate activations
        self.taps: Dict[str, torch.Tensor] = {}
        # "bf16": wgmma tensor-core path (bf16 operands / storage, fp32 accumulation, fp32 ViT residual stream);
        # "fp32": correctness mode — every operand and activation fp32, contractions on the FP32 pipe with fp64
        #         combination of partial sums (the reference is fp32-only: requirements.txt:4, no autocast anywhere);
        # "fp8":  inference only — the bf16 path with the ViT blocks' four linear layers on e4m3 wgmma (per-token
        #         activation and per-channel weight scales; DESIGN.md §3 "Rounding points")
        self._precision = "bf16"
        self._packed = None
        self._packed_sig = None
        self._workspaces: Dict[Tuple[int, int, int], _Workspace] = {}
        self._graphs: Dict[Tuple[int, int, int], tuple] = {}
        self._build_parameters()
        self.register_load_state_dict_post_hook(lambda module, incompatible: module._invalidate())
        if path is not None:
            self.load(path)

    # ------------------------------------------------------------------ parameters / state_dict
    def _build_parameters(self):
        gen = torch.Generator().manual_seed(0)
        for key, shape in state_dict_spec(self.num_channels, backbone=self.backbone):
            *path, leaf = key.split(".")
            mod = self
            for name in path:
                child = mod._modules.get(name)
                if child is None:
                    child = nn.Module()
                    mod.add_module(name, child)
                mod = child
            if key.endswith("cls_token") or key.endswith("pos_embed"):
                t = torch.randn(shape, generator=gen) * 0.02
            elif leaf == "bias":
                t = torch.zeros(shape)
            elif len(shape) == 1:
                t = torch.ones(shape)
            else:
                fan_in = math.prod(shape[1:])
                t = torch.randn(shape, generator=gen) / math.sqrt(fan_in)
            mod.register_parameter(leaf, nn.Parameter(t))

    def load(self, path: str):
        """reference BaseModel.load (modules/midas/base_model.py:5-16)."""
        parameters = torch.load(path, map_location=torch.device("cpu"))
        if "optimizer" in parameters:
            parameters = parameters["model"]
        self.load_state_dict(parameters)

    @property
    def precision(self) -> str:
        return self._precision

    @precision.setter
    def precision(self, value: str):
        if value not in ("bf16", "fp32", "fp8"):
            raise ValueError("precision must be 'bf16', 'fp32' or 'fp8'")
        if value != self._precision:
            self._precision = value
            self._invalidate()
            self._workspaces.clear()

    def _invalidate(self):
        self._packed = None
        self._packed_sig = None
        self._graphs.clear()

    def refresh_weights(self):
        """Re-derive the packed kernel weights (and drop captured CUDA graphs) after the parameters changed.
        `forward` also detects in-place updates by itself (parameter version counters and storage pointers)."""
        self._invalidate()

    def _weights_signature(self):
        # in-place updates (optimizer steps on a flat buffer, broadcast copy_, EMA) bump `_version`;
        # re-pointed storage (flatten_parameters, .data = ...) changes `data_ptr`
        sig = 0
        for p in self.parameters():
            sig = (sig * 1000003 + p._version * 31 + p.data_ptr()) & 0xFFFFFFFFFFFFFFFF
        return sig

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self._invalidate()
        self._workspaces.clear()
        return out

    # ------------------------------------------------------------------ weight pre-pack (one-time)
    @torch.no_grad()
    def _prepack(self, device) -> dict:
        """The forward's operand table (schema: dpt_forward) from the state dict, in its own storage: packed state never
        aliases a parameter."""
        sd = {k: v.detach().to(device) for k, v in self.state_dict().items()}
        wdt = torch.float32 if self._precision == "fp32" else torch.bfloat16    # operand storage type of the GEMMs
        gemm = {}
        vec = {k: sd[k].float().clone() for k in _forward_vectors(self.backbone)}
        # refinenet4.resConfUnit1 is dead in the forward but packed (and broadcast) with the other decoder layers
        for layer in gemm_layers(self.arch) + _rcu_layers(4, 1):
            if layer.key == "head2":
                layer = layer._replace(n_pad=layer.n)      # unpadded: the fused head tail launches at block_n 32
            w = _gemm_operand(sd[layer.weight], layer)
            if self._precision == "fp8" and layer.key.startswith("blk"):
                # the ViT blocks' qkv / proj / fc1 / fc2: e4m3 with a per-output-channel scale
                gemm[layer.key], vec[layer.key + ".scale"] = quantize_rows_e4m3(w)
            elif layer.key in ("pp1t", "pp2t"):
                # ConvTranspose2d(c, c, k, stride k) (vit.py:216-225, 240-249): k*k independent 1x1 convolutions, one
                # per output phase t = (dy, dx): phases[t] = weight[:, :, dy, dx]^T, [out][in]
                w = w.view(layer.n_pad, layer.taps, layer.c_pad).permute(1, 2, 0)
                gemm[layer.key + ".phases"] = w.to(wdt).contiguous()
            else:
                gemm[layer.key] = w.to(wdt).contiguous()
            if layer.bias is not None:
                vec[layer.bias] = F.pad(sd[layer.bias].float(), (0, layer.n_pad - layer.n))
        if self.arch["hybrid"]:
            # stem 7x7: [64,3,7,7] -> [64, (ky,kx,c)=147] padded to 160 columns
            w = _std_weight(sd["pretrained.model.patch_embed.backbone.stem.conv.weight"]).permute(0, 2, 3, 1)
            gemm["stem"] = F.pad(w.reshape(64, 147), (0, 13)).to(wdt).contiguous()
        D = self.arch["embed"]
        for n in ((3, 4) if self.arch["hybrid"] else (1, 2, 3, 4)):
            wfull = sd[f"pretrained.act_postprocess{n}.0.project.0.weight"].to(wdt, copy=True)     # [D, 2D]
            gemm[f"ro{n}.full"] = wfull
            gemm[f"ro{n}.tok"] = wfull[:, :D].contiguous()                                # token half of the Linear
        pos = sd["pretrained.model.pos_embed"].float().clone()                              # [1,577,D] fp32 master copy
        return {"gemm": gemm, "vec": vec, "pos": pos, "pos_cache": {}}

    # ------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not x.is_cuda:
            raise OdbError("omnidata_b200.DPTDepthModel runs on a CUDA (sm_90a) device only; "
                           "there is no CPU fallback — move the model and input to cuda")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"expected input [B,3,H,W], got {tuple(x.shape)}")
        B, _, H, W = x.shape
        autograd = torch.is_grad_enabled() and (self.training or x.requires_grad)
        if autograd and self._precision == "fp8":
            raise ValueError("precision 'fp8' is inference-only: call the model under torch.no_grad() in eval() with "
                             "an input that does not require grad, or switch to 'bf16' / 'fp32' to train")
        check_input_size(H, W, self.arch["hybrid"], autograd)
        if autograd:
            # train() mode under autograd, or an input that requires grad in either mode: the
            # differentiable forward (activations kept for the backward kernels).  Any other eval() call, or any call
            # under torch.no_grad(), is the inference path below and returns a tensor that is not attached to an
            # autograd graph
            return self._forward_autograd(x)
        x = x.detach().float().contiguous()
        sig = self._weights_signature()
        if self._packed is None or sig != self._packed_sig:
            self._invalidate()
            self._packed = self._prepack(x.device)
            self._packed_sig = sig
        if self.use_cuda_graph and not self.keep_taps:
            out = self._forward_graph(x)
        else:
            out = self._forward_impl(x)
        return out.squeeze(dim=1)                     # dpt_depth.py:107

    def _forward_autograd(self, x: torch.Tensor) -> torch.Tensor:
        """Differentiable forward (train_depth.py:183-190 training_step): implemented by omnidata_b200.train."""
        from . import train
        return train.differentiable_forward(self, x)

    def _forward_graph(self, x: torch.Tensor) -> torch.Tensor:
        key = tuple(x.shape[i] for i in (0, 2, 3))
        entry = self._graphs.get(key)
        if entry is None:
            static_in = x.clone()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):                    # warm-up: allocate workspaces, configure kernels
                    self._forward_impl(static_in)
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_out = self._forward_impl(static_in)
            entry = (graph, static_in, static_out)
            self._graphs[key] = entry
        graph, static_in, static_out = entry
        static_in.copy_(x)
        graph.replay()
        return static_out.clone()

    @torch.no_grad()
    def _forward_impl(self, x: torch.Tensor) -> torch.Tensor:
        B, _, H, W = x.shape
        key = (B, H, W)
        ws = self._workspaces.get(key)
        if ws is None:
            ws = self._workspaces[key] = _Workspace(x.device)
        taps = self.taps if self.keep_taps else None
        if taps is not None:
            taps.clear()
        out = dpt_forward(x, self._packed, self.arch, self._precision, self.non_negative, self.num_channels, ws, taps=taps)
        if taps is not None:
            self.taps = {k: v.clone() for k, v in taps.items()}
        return out if (self.use_cuda_graph and not self.keep_taps) else out.clone()


def _debug_upsample(z: torch.Tensor) -> torch.Tensor:
    o = torch.empty((z.shape[0], 2 * z.shape[1], 2 * z.shape[2], z.shape[3]), device=z.device, dtype=z.dtype)
    ops.upsample2x_add(z, o)
    return o


def resize_pos_grid(pos: torch.Tensor, gh: int, gw: int) -> torch.Tensor:
    """Patch rows of the position embedding pos [1, 1 + 24*24, D] resized to a gh x gw patch grid: [gh*gw, D] (vit.py:102-116
    _resize_pos_embed, bilinear, align_corners=False).  The train engine's backward (bwd.pos_embed_resize_bwd) is the
    adjoint of exactly this map."""
    g = pos[0, 1:].reshape(1, 24, 24, -1).permute(0, 3, 1, 2)
    g = F.interpolate(g, size=(gh, gw), mode="bilinear")
    return g.permute(0, 2, 3, 1).reshape(gh * gw, -1)


def _pos_rows(pk, gh: int, gw: int, B: int):
    """(pos0 fp32 [D], patch rows fp32 [B, gh*gw, D]) for a gh x gw patch grid, cached in pk["pos_cache"]: they are
    derived from the weights, so they live with the packed weights.  Bilinear resize as vit.py:102-116 if needed."""
    cache = pk["pos_cache"]
    if (gh, gw) not in cache:
        pos = pk["pos"]
        grid = pos[0, 1:] if (gh, gw) == (24, 24) else resize_pos_grid(pos, gh, gw)
        cache[(gh, gw)] = (pos[0, 0].contiguous(), grid.float().contiguous())
    pos0, grid = cache[(gh, gw)]
    pos_b = cache.get((gh, gw, B))
    if pos_b is None:                                  # replicated per image: the patch GEMM's fp32 residual operand
        pos_b = cache[(gh, gw, B)] = grid.unsqueeze(0).expand(B, -1, -1).contiguous()
    return pos0, pos_b


def _resnet_features(x, pk, ws, buf, fp32: bool, taps, S):
    """ResNetV2 stem + stages of the hybrid encoder -> (layer_1, layer_2, stage-2 features)."""
    B, _, H, W = x.shape
    # ---------------- ResNetV2 stem + stages (timm; hooks at vit.py:363-368)
    h2, w2 = H // 2, W // 2
    n_gn = 1 + sum(3 * d + 1 for _, d in _STAGES)
    stats_pool = buf("gn_stats", (n_gn, B, 32, 2), torch.float32)
    gn_scratch = ws.bufs.get("gn_scratch")
    if gn_scratch is None:                             # zeroed once; the kernel leaves it zeroed
        # fp32 mode's statistics partials grow with B * H * W: the stem (64 ch at H/2) and stage 0 (256 ch at H/4)
        # need the most (4 MiB covers B = 56 at 384x384, B = 7 at 1024x1024)
        need = max(int(ops.lib().odb_groupnorm_scratch_bytes(B, hw, c, 32))
                   for hw, c in ((h2 * w2, 64), ((H // 4) * (W // 4), 256)))
        gn_scratch = ws.bufs["gn_scratch"] = torch.zeros(max(4 << 20, need), dtype=torch.uint8, device=x.device)
    stat_i = iter(range(n_gn))
    # fused statistics: the conv epilogue writes per-warp partial sums here (largest layer:
    # stage 0 at 96x96 -> 72 tiles x 4 quadrants x 32 groups x 2 per image)
    gn_part = buf("gn_partial", (B * ((H // 4) * (W // 4) // 32 + 64) * 4 * 32 * 2,), torch.float32)

    def conv_stats(fn, *args, out, **kw):
        """conv + GroupNorm statistics of its (unrounded) output.  Tensor-core path: partial sums in the conv
        epilogue + finalize; fp32 mode: the deterministic standalone statistics kernel."""
        st = stats_pool[next(stat_i)]
        if fp32:
            fn(*args, out, **kw)
            ops.groupnorm_stats(out, st, scratch=gn_scratch)
        else:
            fn(*args, out, gn_stats=(gn_part, st), **kw)
        return st

    cols = buf("stem_cols", (B * h2 * w2, 160))
    ops.stem_im2col(x, cols)
    s0 = buf("stem_conv", (B, h2, w2, 64))
    gemm, vec = pk["gemm"], pk["vec"]
    bb = "pretrained.model.patch_embed.backbone."
    st = conv_stats(ops.conv1x1, cols.view(B, h2, w2, 160), gemm["stem"], out=s0)
    t = buf("stem_pool", (B, h2 // 2, w2 // 2, 64))
    ops.stem_gn_relu_maxpool(s0, st, vec[bb + "stem.norm.weight"], vec[bb + "stem.norm.bias"], t)
    S["stem"] = (cols, s0, st, t)
    if taps is not None:
        taps["stem_conv"], taps["stem_pool"] = s0, t
    feats, blocks = [], []
    hh, ww = h2 // 2, w2 // 2
    for s, b in [(s, b) for s, (_, depth) in enumerate(_STAGES) for b in range(depth)]:
        cout, mid, stride = _STAGES[s][0], _STAGES[s][0] // 4, (2 if b == 0 and s > 0 else 1)
        ho, wo = hh // stride, ww // stride
        tag, p = f"s{s}b{b}", f"{bb}stages.{s}.blocks.{b}."
        gn = lambda norm: (vec[p + norm + ".weight"], vec[p + norm + ".bias"])      # GroupNorm affine
        # p: the block's parameter-name prefix, for the backward's gradient lookups
        rec = {"tag": tag, "p": p, "stride": stride, "t_in": t, "b": b, "s": s}
        shortcut, sc_stats = t, None
        if b == 0:
            d = buf(tag + "_ds", (B, ho, wo, cout))
            sc_stats = conv_stats(ops.conv1x1, t[:, ::stride, ::stride, :] if stride > 1 else t, gemm[tag + ".wd"],
                                  out=d)
            shortcut = d
            rec.update(d=d, std=sc_stats)
        y1 = buf(tag + "_y1", (B, hh, ww, mid))
        st1 = conv_stats(ops.conv1x1, t, gemm[tag + ".w1"], out=y1)
        a1 = buf(tag + "_a1", (B, hh, ww, mid))
        ops.groupnorm_apply(y1, st1, *gn("norm1"), a1, relu=True)
        y2 = buf(tag + "_y2", (B, ho, wo, mid))
        if stride == 1:
            st2 = conv_stats(ops.conv3x3, a1, gemm[tag + ".w2"], out=y2)
        else:
            st2 = conv_stats(lambda a, w_, o, **kw: ops.conv3x3_s2(a, w_, o, "same", **kw), a1, gemm[tag + ".w2"],
                             out=y2)
        a2 = buf(tag + "_a2", (B, ho, wo, mid))
        ops.groupnorm_apply(y2, st2, *gn("norm2"), a2, relu=True)
        y3 = buf(tag + "_y3", (B, ho, wo, cout))
        st3 = conv_stats(ops.conv1x1, a2, gemm[tag + ".w3"], out=y3)
        out = buf(tag + "_out", (B, ho, wo, cout))
        if b == 0:
            gd, bd = gn("downsample.norm")
            ops.groupnorm_apply(y3, st3, *gn("norm3"), out, relu=True, res=shortcut, res_stats=sc_stats, res_gamma=gd,
                                res_beta=bd)
        else:
            ops.groupnorm_apply(y3, st3, *gn("norm3"), out, relu=True, res=shortcut)
        rec.update(y1=y1, st1=st1, a1=a1, y2=y2, st2=st2, a2=a2, y3=y3, st3=st3, out=out)
        blocks.append(rec)
        t, hh, ww = out, ho, wo
        if taps is not None:
            taps[f"{tag}_out"] = out
        if b == _STAGES[s][1] - 1:
            feats.append(t)
    S["blocks"] = blocks
    return feats


def dpt_forward(x: torch.Tensor, pk: dict, arch: dict, precision: str, non_negative: bool, num_channels: int,
                ws: _Workspace, taps: Optional[dict] = None, save: Optional[dict] = None) -> torch.Tensor:
    """The launch sequence of one DPT forward, for inference (`DPTDepthModel`) and training (`train.TrainEngine`).

    `pk` is the operand table both packers fill (`DPTDepthModel._prepack`, `train.TrainEngine`):
      pk["gemm"]  GEMM operands by layer key: those of `gemm_layers(arch)` (the ConvTransposes "pp{n}t" are read as
                  "pp{n}t.phases" [k*k][c][c], one [out][in] 1x1 operand per output phase), the hybrid's "stem"
                  [64][160] (im2col columns), the readout Linear "ro{n}.full" [D][2D] and its token half "ro{n}.tok";
      pk["vec"]   fp32 tensors by parameter name: the layers' biases, zero-padded to n_pad where the forward reads the
                  layer padded, and the norm affines, cls token, readout biases and the head's last 1x1 conv;
                  precision "fp8": pk["gemm"]["blk{i}.qkv" / ".proj" / ".fc1" / ".fc2"] are e4m3 [n][c]
                  (`quantize_rows_e4m3`) and pk["vec"]["blk{i}.<layer>.scale"] their fp32 per-output-channel scales;
                  every other operand is as in "bf16";
      pk["pos"]   pos_embed in fp32 (inference), and pk["pos_cache"] the patch rows resized to a grid (`_pos_rows`).
    `ws` owns the activations, `taps` (inference diagnostics) receives named intermediates.  `x` is fp32 contiguous
    [B,3,H,W]; returns the fp32 NCHW output buffer.  With `save` given, every activation the hand-written backward reads
    is kept and recorded in it.  That changes the sequence at five points, marked (1)-(5) below: the backward needs each
    ViT block's activations, the attention's log-sum-exp, the pre-activations of the GELUs, and the head's intermediates
    that the fused epilogue never stores."""
    B, _, H, W = x.shape
    fp32, fp8 = precision == "fp32", precision == "fp8"
    if fp8 and save is not None:
        raise ValueError("precision 'fp8' is inference-only: the train forward takes 'bf16' or 'fp32'")
    adt = torch.float32 if fp32 else torch.bfloat16            # activation storage type (fp8: bf16 outside the GEMMs)
    f32 = torch.float32
    buf = lambda name, shape, dtype=None: ws.get(name, shape, adt if dtype is None else dtype)
    S = {} if save is None else save
    S.update(x=x, B=B, H=H, W=W)

    D, heads, depth, hooks = arch["embed"], arch["heads"], arch["depth"], arch["hooks"]
    gemm, vec = pk["gemm"], pk["vec"]
    pm = "pretrained.model."
    if arch["hybrid"]:
        layer_1, layer_2, f3 = _resnet_features(x, pk, ws, buf, fp32, taps, S)
        gh, gw = f3.shape[1], f3.shape[2]
        S["f3"] = f3
    else:
        gh, gw = H // 16, W // 16
    ntok = gh * gw + 1
    rows = B * ntok
    S.update(gh=gh, gw=gw, ntok=ntok)

    # ---------------- ViT buffers.  The residual stream is fp32 in BOTH precisions (timm Block.forward adds every
    # branch to an fp32 `x`; SURVEY.md C.1): the proj / fc2 epilogues read and write fp32, LayerNorm reads fp32.
    # xs[i] is block i's input, xm[i] its stream after the attention branch, xs[i + 1] its output.
    if save is None:
        # (1) the stream is updated in place, in one buffer per hooked block: the block after a hook writes its first
        # residual add into the next buffer, which leaves the hooked activation intact.  All blocks share one buffer set.
        tok = [buf(f"tok_{k}", (B, ntok, D), f32) for k in range(len(hooks))]
        xm = [tok[sum(h < i for h in hooks)] for i in range(depth)]
        xs = tok[:1] + xm
        h = buf("vit_h", (B, ntok, D))
        vit = [dict(h1=h, qkv=buf("vit_qkv", (B, ntok, 3 * D)), att=buf("vit_att", (B, ntok, D)), lse=None, h2=h,
                    u=None, mlp=buf("vit_mlp", (B, ntok, 4 * D)))] * depth
    else:
        xs = [buf(f"vit_x{i}", (B, ntok, D), f32) for i in range(depth + 1)]
        xm = [buf(f"vit_m{i}", (B, ntok, D), f32) for i in range(depth)]
        vit = [dict(h1=buf(f"vit_h1_{i}", (B, ntok, D)), qkv=buf(f"vit_qkv_{i}", (B, ntok, 3 * D)),
                    att=buf(f"vit_att_{i}", (B, ntok, D)),
                    # (2) bf16: the attention also writes the per-row log-sum-exp its backward starts from
                    lse=None if fp32 else buf(f"vit_lse_{i}", (B, heads, ntok), f32),
                    h2=buf(f"vit_h2_{i}", (B, ntok, D)), u=buf(f"vit_u_{i}", (B, ntok, 4 * D)),
                    mlp=buf(f"vit_mlp_{i}", (B, ntok, 4 * D))) for i in range(depth)]
    S.update(xs=xs, xm=xm, vit=vit)

    # ---------------- tokens: patch proj + cls + pos (vit.py:131-147)
    pos0, pos_b = _pos_rows(pk, gh, gw, B)
    ops.write_cls_row(xs[0], vec[pm + "cls_token"].view(-1), pos0)
    proj_b = vec[pm + "patch_embed.proj.bias"]
    if arch["hybrid"]:
        ops.linear(f3.view(B, 1, gh * gw, 1024), gemm["proj"], xs[0][:, 1:, :].unsqueeze(1), bias=proj_b,
                   residual=pos_b.unsqueeze(1))
    else:
        cols = buf("patch_cols", (B, 1, gh * gw, 3 * 16 * 16))
        ops.patchify(x, cols.view(B * gh * gw, -1), 16)
        ops.linear(cols, gemm["proj"], xs[0][:, 1:, :].unsqueeze(1), bias=proj_b, residual=pos_b.unsqueeze(1))
        S["cols"] = cols
    if taps is not None:
        taps["tokens_in"] = xs[0].clone()

    # ---------------- ViT blocks (vit.py:150-151); final norm is dead compute and skipped
    if fp8:
        # the e4m3 GEMM inputs and their row scales: one buffer each, every input consumed before the next is made
        qbuf, qs = buf("vit_q", (rows * 4 * D,), torch.float8_e4m3fn), buf("vit_qs", (rows,), f32)
        q1, q4 = qbuf[:rows * D].view(rows, D), qbuf.view(rows, 4 * D)
    for i, v in enumerate(vit):
        p, blk = f"{pm}blocks.{i}.", f"blk{i}."
        if fp8:
            ops.layernorm_e4m3(xs[i], vec[p + "norm1.weight"], vec[p + "norm1.bias"], q1.view(B, ntok, D), qs)
            ops.linear_fp8(q1, qs, gemm[blk + "qkv"], vec[blk + "qkv.scale"], v["qkv"].view(rows, -1),
                           bias=vec[p + "attn.qkv.bias"])
            ops.attention(v["qkv"], v["att"], heads=heads, scale=0.125)
            ops.rowquant_e4m3(v["att"].view(rows, -1), q1, qs)
            ops.linear_fp8(q1, qs, gemm[blk + "proj"], vec[blk + "proj.scale"], xm[i].view(rows, -1),
                           bias=vec[p + "attn.proj.bias"], residual=xs[i].view(rows, -1))
            ops.layernorm_e4m3(xm[i], vec[p + "norm2.weight"], vec[p + "norm2.bias"], q1.view(B, ntok, D), qs)
            mlp = v["mlp"].view(rows, -1)
            ops.linear_fp8(q1, qs, gemm[blk + "fc1"], vec[blk + "fc1.scale"], mlp, bias=vec[p + "mlp.fc1.bias"],
                           act=ops.ACT_GELU)
            ops.rowquant_e4m3(mlp, q4, qs)
            ops.linear_fp8(q4, qs, gemm[blk + "fc2"], vec[blk + "fc2.scale"], xs[i + 1].view(rows, -1),
                           bias=vec[p + "mlp.fc2.bias"], residual=xm[i].view(rows, -1))
            if taps is not None:
                taps[f"tokens_{i}"] = xs[i + 1].clone()
            continue
        ops.layernorm(xs[i], vec[p + "norm1.weight"], vec[p + "norm1.bias"], v["h1"])
        ops.linear(v["h1"].view(rows, -1), gemm[blk + "qkv"], v["qkv"].view(rows, -1), bias=vec[p + "attn.qkv.bias"])
        ops.attention(v["qkv"], v["att"], heads=heads, scale=0.125, lse=v["lse"])
        ops.linear(v["att"].view(rows, -1), gemm[blk + "proj"], xm[i].view(rows, -1), bias=vec[p + "attn.proj.bias"],
                   residual=xs[i].view(rows, -1))
        ops.layernorm(xm[i], vec[p + "norm2.weight"], vec[p + "norm2.bias"], v["h2"])
        h2, mlp = v["h2"].view(rows, -1), v["mlp"].view(rows, -1)
        fc1, fc1_b = gemm[blk + "fc1"], vec[p + "mlp.fc1.bias"]
        if save is None:
            ops.linear(h2, fc1, mlp, bias=fc1_b, act=ops.ACT_GELU)
        elif fp32:      # (3) the backward needs the pre-activation u as well as gelu(u)
            ops.linear(h2, fc1, v["u"].view(rows, -1), bias=fc1_b)
            bwd.gelu_fwd(v["u"], v["mlp"])
        else:           # (3) one pass: the pre-activation and gelu of the same fp32 value
            ops.linear(h2, fc1, v["u"].view(rows, -1), bias=fc1_b, out2=mlp, out2_act=ops.ACT_GELU)
        ops.linear(mlp, gemm[blk + "fc2"], xs[i + 1].view(rows, -1), bias=vec[p + "mlp.fc2.bias"],
                   residual=xm[i].view(rows, -1))
        if taps is not None:
            taps[f"tokens_{i}"] = xs[i + 1].clone()
    hooked = [xs[hk + 1] for hk in hooks]

    # ---------------- reassemble (vit.py:66-97, 185-290 / 431-462)
    def readout(tk32, n, cout):
        p = f"pretrained.act_postprocess{n}."
        tk = tk32
        if not fp32:                                   # the hooked activation leaves the fp32 stream as a bf16 operand
            tk = buf(f"ro{n}_tok", (B, ntok, D))
            ops.cast_f32_bf16(tk32, tk)
        cb = buf(f"ro{n}_cb", (B, D), f32)
        ops.readout_cls_bias(gemm[f"ro{n}.full"], vec[p + "0.project.0.bias"], tk, cb)
        r = buf(f"ro{n}_r", (B, 1, gh * gw, D))
        pre = None
        if save is None:
            ops.linear(tk[:, 1:, :].unsqueeze(1), gemm[f"ro{n}.tok"], r, bias=cb, bias_per_image=True, act=ops.ACT_GELU)
        else:           # (4) the backward needs the pre-activation: GELU by a separate kernel
            pre = buf(f"ro{n}_pre", (B, 1, gh * gw, D))
            ops.linear(tk[:, 1:, :].unsqueeze(1), gemm[f"ro{n}.tok"], pre, bias=cb, bias_per_image=True)
            bwd.gelu_fwd(pre, r)
        o = buf(f"pp{n}", (B, gh, gw, cout))
        ops.conv1x1(r.view(B, gh, gw, D), gemm[f"pp{n}"], o, bias=vec[p + "3.bias"])
        S[f"ro{n}"] = dict(tk=tk, tk32=tk32, pre=pre, r=r, o=o)
        return o

    def conv_transpose(t, n, k):
        """ConvTranspose2d(c, c, k, stride k): phase (dy, dx) of the output is a 1x1 convolution of the
        input, stored through a strided view of the output (no scatter kernel)."""
        c = t.shape[3]
        o = buf(f"pp{n}t", (B, gh * k, gw * k, c))
        phases, bias = gemm[f"pp{n}t.phases"], vec[f"pretrained.act_postprocess{n}.4.bias"]
        for dy in range(k):
            for dx in range(k):
                ops.conv1x1(t, phases[dy * k + dx], o[:, dy::k, dx::k, :], bias=bias)
        return o

    rn_in = _rn_pad(arch)
    if arch["hybrid"]:
        layer_3 = readout(hooked[0], 3, rn_in[2])
        u4 = readout(hooked[1], 4, rn_in[3])
    else:
        layer_1 = conv_transpose(readout(hooked[0], 1, rn_in[0]), 1, 4)
        layer_2 = conv_transpose(readout(hooked[1], 2, rn_in[1]), 2, 2)
        layer_3 = readout(hooked[2], 3, rn_in[2])
        u4 = readout(hooked[3], 4, rn_in[3])
    layer_4 = buf("pp4s", (B, gh // 2, gw // 2, rn_in[3]))
    ops.conv3x3_s2(u4, gemm["pp4s"], layer_4, "sym1", bias=vec["pretrained.act_postprocess4.4.bias"])
    S["layers"] = (layer_1, layer_2, layer_3, layer_4)

    # ---------------- scratch.layerN_rn (dpt_depth.py:73-76): raw + relu copies feed the RCUs
    rn_raw, rn_relu = [], []
    for n, l in zip((1, 2, 3, 4), S["layers"]):
        shp = (B, l.shape[1], l.shape[2], _FEATURES)
        raw, rl = buf(f"rn{n}_raw", shp), buf(f"rn{n}_relu", shp)
        ops.conv3x3(l, gemm[f"rn{n}"], raw, out2=rl)
        rn_raw.append(raw)
        rn_relu.append(rl)
    S.update(rn_raw=rn_raw, rn_relu=rn_relu)

    # ---------------- RefineNet fusion (dpt_depth.py:78-81; blocks.py:263-341)
    def rcu(n, u, x_raw, x_relu, out):
        key, p = f"ff{n}.rcu{u}.c", f"scratch.refinenet{n}.resConfUnit{u}.conv"
        tmid = buf(f"ff{n}_rcu{u}_t", x_raw.shape)
        ops.conv3x3(x_relu, gemm[key + "1"], tmid, bias=vec[p + "1.bias"], act=ops.ACT_RELU)   # relu(conv1(relu(x)))
        ops.conv3x3(tmid, gemm[key + "2"], out, bias=vec[p + "2.bias"], residual=x_raw)       # conv2(.) + x
        S[f"ff{n}.rcu{u}"] = dict(x_raw=x_raw, x_relu=x_relu, tmid=tmid)

    def fusion_tail(n, s_raw, s_relu):
        """RCU2, then the 1x1 out_conv at the input resolution (it commutes with the bilinear
        upsample: the interpolation weights sum to one)."""
        y = buf(f"ff{n}_y", s_raw.shape)
        rcu(n, 2, s_raw, s_relu, y)
        z = buf(f"ff{n}_z", s_raw.shape)
        ops.conv1x1(y, gemm[f"ff{n}.out"], z, bias=vec[f"scratch.refinenet{n}.out_conv.bias"])
        S[f"ff{n}"] = dict(y=y, z=z)
        return z

    z = fusion_tail(4, rn_raw[3], rn_relu[3])
    if taps is not None:
        taps["path_4"] = _debug_upsample(z)
    for n in (3, 2, 1):
        l_raw, l_relu = rn_raw[n - 1], rn_relu[n - 1]
        res = buf(f"ff{n}_res", l_raw.shape)
        rcu(n, 1, l_raw, l_relu, res)
        s_raw, s_relu = buf(f"ff{n}_s", l_raw.shape), buf(f"ff{n}_s_relu", l_raw.shape)
        ops.upsample2x_add(z, s_raw, res=res, out_relu=s_relu)         # up(path) + RCU1(layer_rn)
        z = fusion_tail(n, s_raw, s_relu)
        if taps is not None and n > 1:
            taps[f"path_{n}"] = _debug_upsample(z)
    path_1 = buf("path_1", (B, z.shape[1] * 2, z.shape[2] * 2, _FEATURES))
    ops.upsample2x_add(z, path_1)

    # ---------------- head (dpt_depth.py:91-99)
    h1 = buf("head_h1", (B, path_1.shape[1], path_1.shape[2], _FEATURES // 2))
    ops.conv3x3(path_1, gemm["head0"], h1, bias=vec["scratch.output_conv.0.bias"])
    h1u = buf("head_h1u", (B, H, W, _FEATURES // 2))
    ops.upsample2x_add(h1, h1u)
    out = buf("out", (B, num_channels, H, W), f32)
    w2, b2 = gemm["head2"], vec["scratch.output_conv.2.bias"]
    w4, b4 = vec["scratch.output_conv.4.weight"].view(num_channels, 32), vec["scratch.output_conv.4.bias"]
    if save is not None:
        # (5) unfused: the backward needs relu(conv2) (32 channels carried zero-padded to 64) and the output map
        a = buf("head_a", (B, H, W, 64))
        ops.conv3x3(h1u, w2, a, bias=b2, act=ops.ACT_RELU)
        bwd.head_tail_fwd(a, w4, b4, out, non_negative)
        S["head"] = dict(path_1=path_1, h1=h1, h1u=h1u, a=a, out=out, w4=w4)
    elif fp32:
        # correctness mode: the 128 -> 32 conv (+ReLU) on the FP32 pipe, then the 1x1 conv (+ReLU) to NCHW
        h2 = buf("head_h2", (B, H, W, 32))
        ops.conv3x3(h1u, w2, h2, bias=b2, act=ops.ACT_RELU)
        pre = buf("head_pre", (B, num_channels, H, W), f32) if taps is not None else None
        ops.head_tail_f32(h2, w4, b4, out, relu=non_negative, pre=pre)
        if taps is not None:
            taps["head_pre_relu"] = pre
    else:
        ops.conv3x3(h1u, w2, None, bias=b2, head=(w4, b4, out, non_negative))

    if taps is not None:
        for hk, tk in zip(hooks, hooked):
            taps[f"tokens_{hk}"] = tk
        taps.update(layer_1=layer_1, layer_2=layer_2, layer_3=layer_3, layer_4=layer_4, path_1=path_1,
                    layer_1_rn=rn_raw[0], layer_2_rn=rn_raw[1], layer_3_rn=rn_raw[2], layer_4_rn=rn_raw[3])
    return out
