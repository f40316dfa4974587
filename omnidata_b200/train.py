"""Train steps of the DPT depth and surface-normal models, every backbone (train_depth.py:183-190 training_step, :261-279
_shared_step, :381-383 Adam, :424-426 DDP; train_normal.py:247-265 for the normal loss): differentiable forward +
hand-written backward over the kernels of this package.  DepthTrainStep (num_channels=1) and NormalTrainStep
(num_channels=3) differ only in their loss and inputs; engine, trainable set, all-reduce, clip + Adam and CUDA-graph
capture are _FlatTrainStep's.

`TrainEngine(model)` owns flat fp32 parameter / gradient buffers (the model's nn.Parameters become views), re-packs the
GEMM operands from the fp32 master weights every step (odb_pack_weight: cast, ResNetV2 weight standardisation, dgrad
layout), runs the forward keeping every activation the backward needs, and the backward.  The forward is the inference
launch sequence, `model.dpt_forward`, fed this engine's operand table and a `save` dict; it differs from inference at five
points, all because the backward needs values inference never stores: per-block ViT buffers, the attention's log-sum-exp,
the pre-activations of the fc1 and readout GELUs, and the unfused head's intermediates.  The backward:
  * dgrad of every conv / linear layer = odb_conv_gemm with the re-packed (in/out swapped, 180-degree rotated) weight;
    stride-2 convolutions scatter through parity-plane output views;
  * wgrad = odb_conv_wgrad (wgmma, both operands MN-major straight from the channels-last tensors; fp32 twin);
  * attention backward = odb_attention_bwd; LayerNorm / GroupNorm / GELU / ReLU / bilinear / max-pool / head backward and
    bias gradients = the kernels of csrc/bwd_ops.cu;
  * the plain ViTs' ConvTranspose reassembles: one dgrad and one wgrad with k taps on k row views of the output gradient.
The DPT-Hybrid (vitb_rn50_384), DPT-Large (vitl16_384) and the plain ViT-B DPT (vitb16_384) share this engine: only the
front end (ResNetV2 + stem vs patch embedding) and the reassemble of layer_1 / layer_2 are backbone-specific.
The engine takes H and W multiples of 32 with at most 639 patches (inference takes up to 4 096).  Off the pretrained
24 x 24 patch grid the forward resizes pos_embed's patch rows from this step's fp32 master weights with the function
inference uses (model.resize_pos_grid), and the backward takes their gradient through the adjoint of that bilinear
resize (odb_pos_embed_resize_bwd, no atomics).
`precision="fp32"` runs the same orchestration on the FP32-pipe twins: the mode the gradient-parity tests use against
torch.autograd of the reference arithmetic.  `differentiable_forward(model, x)` wraps the engine in a
torch.autograd.Function so that `loss(model(x)).backward()` fills `p.grad` (and `x.grad` when x requires grad) like the
reference module would.
requires_grad is honoured per tensor: `backward_plan` walks the network's DAG (_backward_graph) and the backward forms
only the weight / bias / norm-affine gradients of trainable tensors and only the activation gradients that some trainable
tensor or x.grad needs; the forward re-packs frozen operands only when they changed.  With every tensor trainable the
launch sequence is the full one, and every gradient a partial backward forms is bit-identical to the full backward's.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from . import bwd, ops
from ._capi import OdbError
from .model import (_ARCH, _STAGES, MAX_TRAIN_PATCHES, DPTDepthModel, _forward_vectors, _Workspace, check_input_size,
                    dpt_forward, gemm_layers, resize_pos_grid)


def _parity_dgrad_plan(mode: str):
    """Stride-2 3x3 convolution, gradient w.r.t. the input: for input parity plane (py, px) the list of
    (tap index t = ky*3+kx, dy, dx): dX[2p + py, 2q + px] += W_t^T dY[p + dy, q + dx]."""
    def axis(par):
        if mode == "same":          # i = 2o + k
            return [(0, 0), (2, -1)] if par == 0 else [(1, 0)]
        if mode == "sym1":          # i = 2o + k - 1
            return [(1, 0)] if par == 0 else [(0, 1), (2, 0)]
        raise ValueError(mode)
    plan = {}
    for py in (0, 1):
        for px in (0, 1):
            plan[(py, px)] = [(ky * 3 + kx, dy, dx) for ky, dy in axis(py) for kx, dx in axis(px)]
    return plan


def parity_dgrad_operands(wb: torch.Tensor, n_pad: int, mode: str) -> dict:
    """Operands of the stride-2 3x3 input gradient, one small convolution per input parity plane: wb is the layer's
    dgrad operand [c][9 * n_pad] (tap slot 8 - t holds W_t^T, odb_pack_weight).  -> {(py, px): (weight
    [c][len(taps) * n_pad], taps)}; convolving dY with `taps` and that weight gives dX[:, py::2, px::2, :]."""
    operands = {}
    for plane, taps_ in _parity_dgrad_plan(mode).items():
        cat = torch.cat([wb[:, (8 - t) * n_pad:(9 - t) * n_pad] for t, _, _ in taps_], dim=1).contiguous()
        operands[plane] = (cat, [(0, dx, dy) for _, dy, dx in taps_])
    return operands


_BB = "pretrained.model.patch_embed.backbone."
_PM = "pretrained.model."


def _backward_graph(arch: dict) -> List[Tuple[Tuple[str, ...], Tuple[str, ...], str]]:
    """The DPT forward of backbone `arch` (model._ARCH) as a DAG over the activations whose gradients the backward forms:
    (parameters, input activations, output activation) per op, in forward order.  "x" is the input image; parameter-free
    ops (ReLU + add, attention, upsampling, the layer_N taps) carry no parameters.  Tensors no op names (the timm
    classifier head, the final ViT norm, refinenet4.resConfUnit1) are dead: the output does not depend on them."""
    ops = []

    def op(params, ins, out):
        ops.append((tuple(params), tuple(ins), out))

    if arch["hybrid"]:
        _resnet_graph(op)
    else:
        op([_PM + "patch_embed.proj.weight", _PM + "patch_embed.proj.bias", _PM + "cls_token", _PM + "pos_embed"], ["x"],
           "vit.x0")
    for i in range(arch["depth"]):
        p, v, x = f"{_PM}blocks.{i}.", f"vit{i}.", f"vit.x{i}"
        op([p + "norm1.weight", p + "norm1.bias"], [x], v + "h1")
        op([p + "attn.qkv.weight", p + "attn.qkv.bias"], [v + "h1"], v + "qkv")
        op([], [v + "qkv"], v + "att")
        op([p + "attn.proj.weight", p + "attn.proj.bias"], [v + "att", x], v + "xm")
        op([p + "norm2.weight", p + "norm2.bias"], [v + "xm"], v + "h2")
        op([p + "mlp.fc1.weight", p + "mlp.fc1.bias"], [v + "h2"], v + "u")
        op([p + "mlp.fc2.weight", p + "mlp.fc2.bias"], [v + "u", v + "xm"], f"vit.x{i + 1}")
    readouts = (3, 4) if arch["hybrid"] else (1, 2, 3, 4)
    for n, hook in zip(readouts, arch["hooks"]):
        q = f"pretrained.act_postprocess{n}."
        op([q + "0.project.0.weight", q + "0.project.0.bias"], [f"vit.x{hook + 1}"], f"ro{n}.r")
        op([q + "3.weight", q + "3.bias"], [f"ro{n}.r"], f"pp{n}.o")
    if not arch["hybrid"]:                                           # the ConvTranspose reassembles of layer_1 / layer_2
        for n in (1, 2):
            q = f"pretrained.act_postprocess{n}."
            op([q + "4.weight", q + "4.bias"], [f"pp{n}.o"], f"layer_{n}")
    op([], ["pp3.o"], "layer_3")
    op(["pretrained.act_postprocess4.4.weight", "pretrained.act_postprocess4.4.bias"], ["pp4.o"], "layer_4")
    _decoder_graph(op)
    return ops


def _resnet_graph(op):
    """The DPT-Hybrid's ResNetV2 stem and stages, then its 1x1 patch projection (the front end of _backward_graph)."""
    op([_BB + "stem.conv.weight"], ["x"], "stem.s0")
    op([_BB + "stem.norm.weight", _BB + "stem.norm.bias"], ["stem.s0"], "stem.out")
    prev = "stem.out"
    for s, (_, depth) in enumerate(_STAGES):
        for b in range(depth):
            p, t = f"{_BB}stages.{s}.blocks.{b}.", f"s{s}b{b}"
            for i, (src, dst) in enumerate(((prev, "y1"), ("a1", "y2"), ("a2", "y3")), start=1):
                op([p + f"conv{i}.weight"], [src if i == 1 else f"{t}.{src}"], f"{t}.{dst}")
                op([p + f"norm{i}.weight", p + f"norm{i}.bias"], [f"{t}.{dst}"], f"{t}.{('a1', 'a2', 'r')[i - 1]}")
            skip = prev
            if b == 0:
                op([p + "downsample.conv.weight"], [prev], f"{t}.d")
                op([p + "downsample.norm.weight", p + "downsample.norm.bias"], [f"{t}.d"], f"{t}.dn")
                skip = f"{t}.dn"
            op([], [f"{t}.r", skip], f"{t}.out")
            prev = f"{t}.out"
        if s < 2:
            op([], [prev], f"layer_{s + 1}")                        # stage outputs 0 and 1 feed the decoder
    op([], [prev], "f3")
    op([_PM + "patch_embed.proj.weight", _PM + "patch_embed.proj.bias", _PM + "cls_token", _PM + "pos_embed"], ["f3"],
       "vit.x0")


def _decoder_graph(op):
    """scratch.layerN_rn, the RefineNet fusion blocks and the head (the back end of _backward_graph)."""
    for n in (1, 2, 3, 4):
        op([f"scratch.layer{n}_rn.weight"], [f"layer_{n}"], f"rn{n}.o")

    def rcu(n, u, x, out):
        q = f"scratch.refinenet{n}.resConfUnit{u}."
        op([q + "conv1.weight", q + "conv1.bias"], [x], f"ff{n}.rcu{u}.t")
        op([q + "conv2.weight", q + "conv2.bias"], [f"ff{n}.rcu{u}.t", x], out)
    for n in (4, 3, 2, 1):
        s_in = "rn4.o"
        if n < 4:
            rcu(n, 1, f"rn{n}.o", f"ff{n}.res")
            op([], [f"ff{n}.res", f"ff{n + 1}.z"], f"ff{n}.s")
            s_in = f"ff{n}.s"
        rcu(n, 2, s_in, f"ff{n}.y")
        op([f"scratch.refinenet{n}.out_conv.weight", f"scratch.refinenet{n}.out_conv.bias"], [f"ff{n}.y"], f"ff{n}.z")
    op(["scratch.output_conv.0.weight", "scratch.output_conv.0.bias"], ["ff1.z"], "head.h1")
    op(["scratch.output_conv.2.weight", "scratch.output_conv.2.bias"], ["head.h1"], "head.a")
    op(["scratch.output_conv.4.weight", "scratch.output_conv.4.bias"], ["head.a"], "out")


class BackwardPlan:
    """What one backward computes.  grad(name): the parameter's gradient is formed (it is trainable); act(name): the
    gradient w.r.t. that activation of _backward_graph is formed, which is the case iff x.grad is wanted or some
    trainable tensor lies upstream of it.  `full`: every tensor trainable, the backward's complete launch sequence."""

    def __init__(self, trainable: frozenset, acts: Dict[str, bool], full: bool, want_dx: bool):
        self.trainable, self.acts, self.full, self.want_dx = trainable, acts, full, want_dx

    def grad(self, name: str) -> bool:
        return name in self.trainable

    def act(self, name: str) -> bool:
        return self.acts[name]


def backward_plan(param_names, trainable=None, want_dx: bool = False, backbone: str = "vitb_rn50_384") -> BackwardPlan:
    """The backward plan of the DPT with encoder `backbone` for the trainable tensors `trainable` (names; None = all of
    param_names) and, if want_dx, the gradient w.r.t. the input image."""
    names = list(param_names)
    ops = _backward_graph(_ARCH[backbone])
    known = set(names)
    for params, _, _ in ops:
        for p in params:
            if p not in known:
                raise ValueError(f"backward_plan: parameter {p} of the {backbone} DPT is missing from param_names")
    T = frozenset(names) if trainable is None else frozenset(trainable)
    unknown = T - known
    if unknown:
        raise ValueError(f"backward_plan: unknown parameter names {sorted(unknown)[:3]}")
    up = {"x": bool(want_dx)}
    for params, ins, out in ops:
        up[out] = any(p in T for p in params) or any(up[i] for i in ins)
    return BackwardPlan(T, up, trainable is None or T == known, bool(want_dx))


def trainable_segments(names: List[str], sizes: List[int], trainable) -> List[Tuple[int, int]]:
    """[start, end) ranges of the flat buffers (state_dict order, padded sizes) holding exactly the trainable tensors
    (slices of adjacent trainable tensors merged): the segment table of the clip and Adam kernels."""
    segs, off = [], 0
    for n, s in zip(names, sizes):
        if n in trainable:
            if segs and segs[-1][1] == off:
                segs[-1] = (segs[-1][0], off + s)
            else:
                segs.append((off, off + s))
        off += s
    return segs


def select_buckets(buckets, names: List[str], sizes: List[int], trainable):
    """The all-reduce buckets (plan_grad_buckets) that hold at least one trainable tensor."""
    starts, off = [], 0
    for n, s in zip(names, sizes):
        if n in trainable:
            starts.append(off)
        off += s
    return [(s, e, tag) for s, e, tag in buckets if any(s <= o < e for o in starts)]


class TrainEngine:
    def __init__(self, model: DPTDepthModel, precision: str = "bf16"):
        if precision == "fp8":
            raise ValueError("precision 'fp8' is inference-only: training and gradients take 'bf16' or 'fp32'")
        if precision not in ("bf16", "fp32"):
            raise ValueError("precision must be 'bf16' or 'fp32'")
        self.model = model
        self.backbone, self.hybrid = model.backbone, model.arch["hybrid"]
        self.D, self.heads, self.depth, self.hooks = (model.arch[k] for k in ("embed", "heads", "depth", "hooks"))
        self.rn_in, self.rn_pad = model.arch["rn_in"], model._rn_pad
        # the readouts the hooked blocks feed, in hook order (act_postprocess1..4; the hybrid's layer_1/2 come from ResNetV2)
        self.readouts = (3, 4) if self.hybrid else (1, 2, 3, 4)
        self.precision = precision
        self.fp32 = precision == "fp32"
        self.adt = torch.float32 if self.fp32 else torch.bfloat16
        p0 = next(model.parameters())
        if not p0.is_cuda:
            raise OdbError("TrainEngine: the model must live on a CUDA device (no CPU path)")
        self.device = p0.device
        self.C = model.num_channels
        self.non_negative = model.non_negative
        # ---- flat fp32 master parameters / gradients (16-byte aligned slices, state_dict order)
        names, params = zip(*model.named_parameters())
        sizes = [(p.numel() + 3) // 4 * 4 for p in params]
        self.flat = torch.zeros(sum(sizes), device=self.device, dtype=torch.float32)
        self.flat_grad = torch.zeros_like(self.flat)
        self.P: Dict[str, torch.Tensor] = {}
        self.G: Dict[str, torch.Tensor] = {}
        off = 0
        with torch.no_grad():
            for name, p, n in zip(names, params, sizes):
                self.flat[off:off + p.numel()].copy_(p.data.reshape(-1).float())
                p.data = self.flat[off:off + p.numel()].view_as(p.data)
                self.P[name] = p.data
                self.G[name] = self.flat_grad[off:off + p.numel()].view_as(p.data)
                off += n
        self.param_names = list(names)
        self.params = dict(zip(names, params))                       # the model's nn.Parameters (requires_grad, _version)
        self._plans: Dict[tuple, BackwardPlan] = {}
        self._packed_sig: Dict[str, tuple] = {}                     # source parameter -> (version, pointer) last packed
        self._pack_tables: Dict[tuple, bwd.PackTable] = {}
        self._unpack_cache: Dict[frozenset, dict] = {}
        self.plane_w = {}
        self.ws = _Workspace(self.device)
        self.bufs = self.ws.bufs
        self._build_layer_table()
        self.pk = self._forward_operands()
        self.saved = None

    # ------------------------------------------------------------------ buffers
    def buf(self, name: str, shape, dtype=None) -> torch.Tensor:
        return self.ws.get(name, shape, self.adt if dtype is None else dtype)

    # ------------------------------------------------------------------ weight table / per-step packing
    def _build_layer_table(self):
        """The GEMM layers (model.gemm_layers): fwd [n_pad][taps*c_pad], bwd [c_pad][taps*n_pad] operand buffers are
        allocated once and re-filled every step.  Padded rows / columns are zero and their gradients are dropped by the
        unpack pass."""
        self.layers = gemm_layers(self.model.arch)
        self.layer = {L.key: L for L in self.layers}
        self.W: Dict[str, Tuple[torch.Tensor, torch.Tensor]] = {}
        for L in self.layers:
            fwd = torch.zeros((L.n_pad, L.taps * L.c_pad), device=self.device, dtype=self.adt)
            bwd_ = torch.zeros((L.c_pad, L.taps * L.n_pad), device=self.device, dtype=self.adt)
            self.W[L.key] = (fwd, bwd_)
        # packed-layout wgrad scratch (the readouts' Linear halves, the stem)
        D = self.D
        self.gp = torch.empty(D * 9 * D, device=self.device, dtype=torch.float32)
        # one-launch packing of all layers; packed-layout gradient buffers of the layers that need the unpack pass
        # (3x3 taps, weight standardisation or padding), converted by ONE launch per all-reduce bucket
        self.pack_table = self._new_pack_table(self.layers)
        self.gp_layer: Dict[str, torch.Tensor] = {}
        groups = {"decoder": [], "resnet": []}
        for L in self.layers:
            if L.taps == 1 and not L.standardize and L.n_pad == L.n and L.c_pad == L.c:
                continue                                           # written straight into the flat gradient
            gp = torch.zeros((L.n_pad, L.taps * L.c_pad), device=self.device, dtype=torch.float32)
            self.gp_layer[L.key] = gp
            tag = "resnet" if "backbone" in L.weight else "decoder"
            groups[tag].append((L.weight, (gp, self.P[L.weight], self.G[L.weight], L.n, L.c, L.taps, L.c_pad,
                                           L.standardize)))
        self.unpack_groups = groups
        self.unpack_tables = {t: bwd.UnpackTable([it for _, it in v]) for t, v in groups.items() if v}
        self.zb = torch.zeros(4096, device=self.device, dtype=torch.float32)               # zero "bias" of the dgrad convs:
        #   selects the straight-line (bias / bias + residual) epilogues of the tensor-core kernel

    def _new_pack_table(self, layers) -> bwd.PackTable:
        return bwd.PackTable([(self.P[L.weight], *self.W[L.key], L.n, L.c, L.taps, L.n_pad, L.c_pad, L.standardize)
                              for L in layers], self.adt)

    def _forward_operands(self) -> dict:
        """The forward's operand table (schema: model.dpt_forward) as the engine's persistent tensors: the GEMM operands
        pack() refills in place, and views of the flat fp32 master weights, or zero-padded copies that pack() refreshes
        where the forward reads a bias padded (head conv2, vitb16_384's 96-wide layer_1)."""
        gemm = {L.key: self.W[L.key][0] for L in self.layers}
        vec = {name: self.P[name] for name in _forward_vectors(self.backbone)}
        for L in self.layers:
            if L.bias is not None:
                padded = L.n_pad != L.n
                vec[L.bias] = self.buf(f"w.pad.{L.bias}", (L.n_pad,), torch.float32) if padded else self.P[L.bias]
        if self.hybrid:
            gemm["stem"] = self.buf("w.stem", (64, 160))
        D = self.D
        for n in self.readouts:
            gemm[f"ro{n}.full"] = self.buf(f"w.ro{n}.full", (D, 2 * D))
            gemm[f"ro{n}.tok"] = self.buf(f"w.ro{n}.tok", (D, D))
        if not self.hybrid:
            for n, k in ((1, 4), (2, 2)):                           # filled by pack() from the dgrad operand
                cp = self.rn_pad[n - 1]
                gemm[f"pp{n}t.phases"] = self.buf(f"w.pp{n}t.phases", (k * k, cp, cp))
        # pos_cache: filled by every forward() with that step's rows
        return {"gemm": gemm, "vec": vec, "pos_cache": {}}

    def _stale(self, trainable) -> set:
        """Source parameters whose derived forward operands must be (re)built: every trainable one (FlatAdam writes the
        master weights through raw pointers, bumping no version counter) and every frozen one whose version counter or
        storage changed since it was last packed (load_state_dict, copy_, re-pointed .data: DPTDepthModel's rule)."""
        out = set()
        for name, p in self.params.items():
            if trainable is None or name in trainable:
                out.add(name)
                self._packed_sig.pop(name, None)                    # re-checked if the tensor is frozen later
            else:
                sig = (p._version, p.data_ptr())
                if self._packed_sig.get(name) != sig:
                    out.add(name)
                    self._packed_sig[name] = sig
        return out

    def pack_table_for(self, keys: tuple) -> bwd.PackTable:
        """The one-launch packing of the GEMM layers `keys` (cached: the table's device copy is made once, outside any
        CUDA-graph capture)."""
        if len(keys) == len(self.layers):
            return self.pack_table
        tab = self._pack_tables.get(keys)
        if tab is None:
            tab = self._pack_tables[keys] = self._new_pack_table([L for L in self.layers if L.key in keys])
        return tab

    @torch.no_grad()
    def pack(self, trainable=None):
        """fp32 master weights -> GEMM operands.  trainable None: all of them (every step: the optimizer just changed
        them); else only those of the trainable tensors and of frozen tensors changed since their last packing."""
        if trainable is None:
            self._packed_sig.clear()
        stale = None if trainable is None else self._stale(trainable)
        fresh = (lambda name: True) if stale is None else (lambda name: name in stale)
        keys = tuple(L.key for L in self.layers if fresh(L.weight))
        if keys:
            self.pack_table_for(keys).run()
        P, gemm, vec = self.P, self.pk["gemm"], self.pk["vec"]
        bb = "pretrained.model.patch_embed.backbone."
        # stem 7x7 (3 input channels): [64,3,7,7] -> standardise -> [64, (ky,kx,c)=147] padded to 160 columns
        if self.hybrid and fresh(bb + "stem.conv.weight"):
            w = P[bb + "stem.conv.weight"]
            std_, mean = torch.std_mean(w, dim=[1, 2, 3], keepdim=True, unbiased=False)
            ws = ((w - mean) / (std_ + 1e-8)).permute(0, 2, 3, 1).reshape(64, 147)
            stem = gemm["stem"]
            stem.zero_()
            stem[:, :147].copy_(ws)
        for L in self.layers:                                        # the biases the forward reads zero-padded
            if L.bias is not None and L.n_pad != L.n and fresh(L.bias):
                vec[L.bias].zero_()
                vec[L.bias][:L.n].copy_(P[L.bias])
        # ProjectReadout Linear(2D -> D): token half as a GEMM operand (fwd / bwd), whole matrix for the cls kernel
        D = self.D
        for n in self.readouts:
            if not fresh(f"pretrained.act_postprocess{n}.0.project.0.weight"):
                continue
            wfull = P[f"pretrained.act_postprocess{n}.0.project.0.weight"]
            gemm[f"ro{n}.full"].copy_(wfull)
            gemm[f"ro{n}.tok"].copy_(wfull[:, :D])
            tokb = self.buf(f"w.ro{n}.tokT", (D, D))
            tokb.copy_(wfull[:, :D].t())
            clsT = self.buf(f"w.ro{n}.clsT", (D, D), torch.float32)
            clsT.copy_(wfull[:, D:].t())
        if not self.hybrid:
            for n, k in ((1, 4), (2, 2)):
                if f"pp{n}t" in keys:
                    # the forward's per-phase operands W[:, :, ky, kx]^T [out][in] = the tap blocks of the dgrad
                    # operand, bwd[out][(k*k-1-t)*cp + in]
                    cp = self.rn_pad[n - 1]
                    gemm[f"pp{n}t.phases"].copy_(self.W[f"pp{n}t"][1].view(cp, k * k, cp).permute(1, 0, 2).flip(0))
        # stride-2 3x3 convolutions: per-parity-plane dgrad operands cut out of the rotated dgrad weight
        for key, mode in (("s1b0.w2", "same"), ("s2b0.w2", "same"), ("pp4s", "sym1")):
            if key not in keys:
                continue
            for plane, op in parity_dgrad_operands(self.W[key][1], self.layer[key].n_pad, mode).items():
                self.plane_w[(key, plane)] = op

    # ------------------------------------------------------------------ small helpers
    def _wgrad(self, key: str, views, taps, dy, n_rows: Optional[int] = None):
        """weight gradient of layer `key` into the flat gradient buffer (through the weight standardisation); nothing
        for a frozen weight."""
        L = self.layer[key]
        if not self._plan.grad(L.weight):
            return
        if key not in self.gp_layer:
            # linear / 1x1 layer without weight standardisation: the packed gradient layout IS the parameter layout
            bwd.conv_wgrad(views, taps, dy, self.G[L.weight].view(L.n, L.c))
            return
        bwd.conv_wgrad(views, taps, dy, self.gp_layer[key])        # converted to parameter layout by the bucket's unpack launch

    def _bias_grad(self, pname: str, dy):
        if not self._plan.grad(pname):
            return
        g = self.G[pname]
        if dy.shape[-1] == g.numel():
            bwd.colsum(dy.reshape(-1, dy.shape[-1]), g.view(1, -1))
        else:                                                   # padded output channels (head conv2, vitb16 layer_1)
            tmp = self.buf(f"tmp.bias{dy.shape[-1]}", (1, dy.shape[-1]), torch.float32)
            bwd.colsum(dy.reshape(-1, dy.shape[-1]), tmp)
            g.copy_(tmp[0, :g.numel()])

    def _param_grads(self, wname: str, bname: str):
        """(dgamma, dbeta) outputs of a norm / the head tail: None, None when both are frozen; a frozen one of a pair
        whose other half trains gets a scratch buffer (the kernels form both or neither)."""
        tw, tb = self._plan.grad(wname), self._plan.grad(bname)
        if not (tw or tb):
            return None, None
        G = self.G
        dw = G[wname] if tw else self.buf(f"tmp.dparam_w{G[wname].numel()}", G[wname].shape, torch.float32)
        db = G[bname] if tb else self.buf(f"tmp.dparam_b{G[bname].numel()}", G[bname].shape, torch.float32)
        return dw, db

    def plan_for(self, trainable, want_dx: bool) -> BackwardPlan:
        key = (trainable, bool(want_dx))
        plan = self._plans.get(key)
        if plan is None:
            plan = self._plans[key] = backward_plan(self.param_names, trainable, want_dx, self.backbone)
        return plan

    def _unpack(self, tag: str, plan: BackwardPlan):
        """The packed-layout -> parameter-layout conversion of bucket `tag`, for the trainable weights only (one table per
        trainable set, cached)."""
        tab = self._unpack_tables_for(plan).get(tag)
        if tab is not None:
            tab.run()

    def _unpack_tables_for(self, plan: BackwardPlan) -> dict:
        if plan.full:
            return self.unpack_tables
        tabs = self._unpack_cache.get(plan.trainable)
        if tabs is None:
            tabs = {}
            for tag, v in self.unpack_groups.items():
                items = [it for pn, it in v if pn in plan.trainable]
                if items:
                    tabs[tag] = bwd.UnpackTable(items)
            self._unpack_cache[plan.trainable] = tabs
        return tabs

    def prepare(self, trainable=None):
        """Builds the packing / unpacking tables and the plans of a trainable set up front (a CUDA-graph capture cannot
        create them)."""
        for want_dx in (False, True):
            plan = self.plan_for(trainable, want_dx)
        self._unpack_tables_for(plan)
        if trainable is not None:
            keys = tuple(L.key for L in self.layers if L.weight in trainable)
            if keys:
                self.pack_table_for(keys)

    def _zb(self, w: torch.Tensor):
        """zero bias vector for a dgrad convolution with weight `w` [n_out][K] (tensor-core path only)."""
        return None if self.fp32 else self.zb[: w.shape[0]]

    # ------------------------------------------------------------------ forward (activations kept)
    @torch.no_grad()
    def forward(self, x: torch.Tensor, trainable=None) -> torch.Tensor:
        """The model's forward (the launch sequence of model.dpt_forward) on this step's weights; every activation the
        backward reads is recorded in self.saved.  trainable (names; None = all): the operands of frozen tensors are
        re-packed only when those tensors changed (pack)."""
        if not x.is_cuda or x.dim() != 4 or x.shape[1] != 3:
            raise OdbError("TrainEngine.forward: CUDA input [B,3,H,W] required")
        x = x.detach().float().contiguous()
        B, _, H, W = x.shape
        check_input_size(H, W, self.model.arch["hybrid"], autograd=True)
        gh, gw = H // 16, W // 16
        self.pack(trainable)
        # the patch rows of this step's pos_embed (resized from the fp32 master weights as inference resizes them),
        # replicated per image: the patch GEMM's residual operand
        pos = self.P["pretrained.model.pos_embed"]
        grid = pos[0, 1:] if (gh, gw) == (24, 24) else resize_pos_grid(pos, gh, gw)
        pos_b = self.buf("pos_expanded", (B, gh * gw, pos.shape[-1]), torch.float32)
        pos_b.copy_(grid.unsqueeze(0).expand(B, -1, -1))
        self.pk["pos_cache"] = {(gh, gw): (pos[0, 0], grid), (gh, gw, B): pos_b}
        self.saved = {}
        return dpt_forward(x, self.pk, self.model.arch, self.precision, self.non_negative, self.C, self.ws,
                           save=self.saved)

    # ------------------------------------------------------------------ backward
    def _gemm_bwd(self, key: str, dy, x, dx=None, bias: bool = True):
        """Backward of GEMM layer `key` (one input view, the taps of its table entry) with output gradient dy and input
        x: the input gradient into dx (skipped when dx is None), the weight gradient and, unless `bias` is False (formed
        elsewhere), the bias gradient."""
        L = self.layer[key]
        taps = bwd.TAPS_1 if L.taps == 1 else bwd.TAPS_3X3
        if dx is not None:
            w = self.W[key][1]
            ops.conv_gemm([dy], taps, w, dx, bias=self._zb(w))
        self._wgrad(key, [x], taps, dy)
        if bias and L.bias is not None:
            self._bias_grad(L.bias, dy)

    def _dgrad_s2(self, key: str, dy, dx):
        """gradient w.r.t. the input of a stride-2 3x3 convolution: one small convolution per input parity plane,
        stored through a strided view of dx."""
        for (py, px) in ((0, 0), (0, 1), (1, 0), (1, 1)):
            w, taps = self.plane_w[(key, (py, px))]
            ops.conv_gemm([dy], taps, w, dx[:, py::2, px::2, :], bias=self._zb(w))

    def _conv_transpose_bwd(self, n: int, k: int, dout, u):
        """Backward of layer_n's ConvTranspose2d(c, c, k, stride k) (plain ViTs), out[b, k*y+ky, k*x+kx, o] =
        sum_i u[b, y, x, i] W[i, o, ky, kx] + bias[o].  Row k*y+ky of the channels-last dout is contiguous over (kx, o),
        so dout is k views [B, gh, gw, k*c], one per ky: the input gradient is one convolution with k taps (K = k*k*c)
        and the weight gradient one wgrad with k taps, no scatter.  -> gradient w.r.t. u (None when not needed)."""
        B, H, W, cp = dout.shape
        views = [dout.view(B, H // k, k, W // k, k * cp)[:, :, ky] for ky in range(k)]
        taps = [(ky, 0, 0) for ky in range(k)]
        du = None
        if self._plan.act(f"pp{n}.o"):
            w = self.W[f"pp{n}t"][0]                                  # [in][(ky, kx, out)]
            du = self.buf(f"g.pp{n}", u.shape)
            ops.conv_gemm(views, taps, w, du, bias=self._zb(w))
        self._wgrad(f"pp{n}t", views, taps, u)                         # [in][(ky, kx, out)] = the parameter's layout
        self._bias_grad(f"pretrained.act_postprocess{n}.4.bias", dout)
        return du

    @torch.no_grad()
    def backward(self, dout: torch.Tensor, on_ready=None, dx: Optional[torch.Tensor] = None, trainable=None):
        """dout: gradient w.r.t. the forward's output [B,C,H,W] fp32.  Fills self.flat_grad: the slices of the trainable
        tensors (`trainable`: names; None = all 368, the complete launch sequence).  The slices of frozen tensors are not
        written, and no work is done that only they or unwanted activations need (backward_plan).
        on_ready(tag) is called when a contiguous range of the flat gradient is final (plan_grad_buckets): the
        data-parallel train step launches that range's all-reduce while the rest of the backward runs.
        dx (optional, fp32 contiguous [B,3,H,W]) receives the gradient w.r.t. the input image."""
        ready = on_ready if on_ready is not None else (lambda tag: None)
        S, P, G, Wt, buf = self.saved, self.P, self.G, self.W, self.buf
        if S is None:
            raise OdbError("TrainEngine.backward: call forward first")
        plan = self._plan = self.plan_for(trainable, dx is not None)
        need, T = plan.act, plan.grad
        B, H, W = S["B"], S["H"], S["W"]
        f32 = torch.float32
        dout = dout.detach().float().contiguous().view(B, self.C, H, W)
        hd = S["head"]
        # ---- head
        da = dh1 = dpath = None
        w4, b4 = "scratch.output_conv.4.weight", "scratch.output_conv.4.bias"
        if need("head.a") or T(w4) or T(b4):
            da = buf("g.head_a", hd["a"].shape)
            dw4, db4 = self._param_grads(w4, b4)
            bwd.head_tail_bwd(dout, hd["out"], hd["a"], hd["w4"], da, None if dw4 is None else dw4.view(self.C, 32), db4,
                              self.non_negative)
        dh1u = buf("g.head_h1u", hd["h1u"].shape) if need("head.h1") else None
        self._gemm_bwd("head2", da, hd["h1u"], dh1u)
        if need("head.h1"):
            dh1 = buf("g.head_h1", hd["h1"].shape)
            bwd.upsample2x_bwd(dh1u, dh1)
        if need("ff1.z"):
            dpath = buf("g.path_1", hd["path_1"].shape)
        self._gemm_bwd("head0", dh1, hd["path_1"], dpath)

        # ---- RefineNet fusion blocks
        def rcu_bwd(n, u_, d_out, dx, x_name):
            """d_out: gradient w.r.t. the RCU output; dx <- gradient w.r.t. its (pre-ReLU) input `x_name` when needed."""
            r = S[f"ff{n}.rcu{u_}"]
            need_t = need(f"ff{n}.rcu{u_}.t")
            dt = buf(f"g.ff{n}_rcu{u_}_t", r["tmid"].shape) if need_t else None
            self._gemm_bwd(f"ff{n}.rcu{u_}.c2", d_out, r["tmid"], dt)
            if need_t:
                bwd.mask_add(dt, dt, mask=r["tmid"])                    # through relu(conv1 + b1)
                dxr = buf(f"g.ff{n}_rcu{u_}_x", r["x_raw"].shape) if need(x_name) else None
                self._gemm_bwd(f"ff{n}.rcu{u_}.c1", dt, r["x_relu"], dxr)
            if need(x_name):
                bwd.mask_add(dx, dxr, a=d_out, mask=r["x_relu"])        # skip + through relu(x)

        d_rn = [None] * 4
        if need("ff1.z"):
            dz = buf("g.ff1_z", S["ff1"]["z"].shape)
            bwd.upsample2x_bwd(dpath, dz)
        for n in (1, 2, 3, 4):
            if not need(f"ff{n}.z"):                                    # nor anything of the later fusion blocks
                break
            f = S[f"ff{n}"]
            dy = buf(f"g.ff{n}_y", f["y"].shape) if need(f"ff{n}.y") else None
            self._gemm_bwd(f"ff{n}.out", dz, f["y"], dy)
            if dy is None:
                continue
            s_name = "rn4.o" if n == 4 else f"ff{n}.s"
            ds_ = buf(f"g.ff{n}_s", f["y"].shape) if need(s_name) else None
            rcu_bwd(n, 2, dy, ds_, s_name)
            if n == 4:
                d_rn[3] = ds_
            else:
                if need(f"ff{n}.res"):
                    dr = buf(f"g.rn{n}_raw", f["y"].shape) if need(f"rn{n}.o") else None
                    rcu_bwd(n, 1, ds_, dr, f"rn{n}.o")                  # res = RCU1(layer_rn): d res = d s
                    d_rn[n - 1] = dr
                if need(f"ff{n + 1}.z"):
                    dz = buf(f"g.ff{n + 1}_z", S[f"ff{n + 1}"]["z"].shape)
                    bwd.upsample2x_bwd(ds_, dz)
        # ---- scratch.layerN_rn
        d_layers = [None] * 4
        for n in (1, 2, 3, 4):
            l = S["layers"][n - 1]
            if need(f"layer_{n}"):
                d_layers[n - 1] = buf(f"g.layer_{n}", l.shape)
            self._gemm_bwd(f"rn{n}", d_rn[n - 1], l, d_layers[n - 1])
        # ---- reassemble: act_postprocess4.4 (stride 2), the ConvTransposes of layer_1 / layer_2 (plain ViTs), then the
        # readouts
        gh, gw, ntok, D = S["gh"], S["gw"], S["ntok"], self.D
        u4 = S["ro4"]["o"]
        du4 = None
        if need("pp4.o"):
            du4 = buf("g.pp4", u4.shape)
            self._dgrad_s2("pp4s", d_layers[3], du4)
        planes = [u4[:, py::2, px::2, :] for py in range(2) for px in range(2)]
        self._wgrad("pp4s", planes, ops._parity_taps("sym1"), d_layers[3])
        self._bias_grad("pretrained.act_postprocess4.4.bias", d_layers[3])
        d_pp = {3: d_layers[2], 4: du4}                              # gradient w.r.t. act_postprocessN.3's output
        if not self.hybrid:
            for n, k in ((2, 2), (1, 4)):
                if need(f"layer_{n}"):
                    d_pp[n] = self._conv_transpose_bwd(n, k, d_layers[n - 1], S[f"ro{n}"]["o"])

        def readout_bwd(n, do, tokens):
            """-> gradient w.r.t. the hooked tokens `tokens`, activation type [B, ntok, D] (None when not needed)."""
            r = S[f"ro{n}"]
            pp = f"pretrained.act_postprocess{n}."
            dr = buf(f"g.ro{n}_r", r["r"].shape) if need(f"ro{n}.r") else None
            self._gemm_bwd(f"pp{n}", do, r["r"].view(B, gh, gw, D), None if dr is None else dr.view(B, gh, gw, D))
            if dr is None:
                return None
            bwd.gelu_bwd(dr, r["pre"], dr)
            dtk = None
            if need(tokens):
                dtk = buf(f"g.ro{n}_tok", (B, ntok, D))
                ops.linear(dr, self.bufs[f"w.ro{n}.tokT"], dtk[:, 1:, :].unsqueeze(1))
            tw, wname = T(pp + "0.project.0.weight"), pp + "0.project.0.weight"
            gw_ = G[wname]
            gp = self.gp[: D * D].view(D, D)
            if tw:
                bwd.conv_wgrad([r["tk"][:, 1:, :].unsqueeze(1)], bwd.TAPS_1, dr, gp)
                gw_[:, :D].copy_(gp)
            # cls half: cb[b] = W[:, D:] tok[b, 0] + bias, added to every token of image b
            dcb = buf(f"g.ro{n}_cb", (B, D), f32)
            bwd.colsum(dr.view(B, gh * gw, D), dcb, batches=B)
            if T(pp + "0.project.0.bias"):
                bwd.colsum(dcb, G[pp + "0.project.0.bias"].view(1, -1))
            if tw:
                tok0 = buf(f"ro{n}_tok0", (B, D), f32)
                tok0.copy_(r["tk"][:, 0, :])
                bwd.conv_wgrad([tok0.view(1, 1, B, D)], bwd.TAPS_1, dcb.view(1, 1, B, D), gp)
                gw_[:, D:].copy_(gp)
            if dtk is not None:
                dt0 = buf(f"g.ro{n}_tok0", (B, D), f32)
                ops.linear(dcb, self.bufs[f"w.ro{n}.clsT"], dt0)
                dtk[:, 0, :].copy_(dt0)
            return dtk

        dtk = {}                                                     # hooked block -> gradient w.r.t. its output tokens
        for n, hook in reversed(list(zip(self.readouts, self.hooks))):
            if need(f"pp{n}.o"):
                dtk[hook] = readout_bwd(n, d_pp[n], f"vit.x{hook + 1}")
        self._unpack("decoder", plan)
        ready("decoder")
        # ---- ViT blocks (fp32 stream gradient ds, activation-type copy ds16 for the GEMMs)
        pm = "pretrained.model."
        rows = B * ntok
        xs, xm, vit = S["xs"], S["xm"], S["vit"]
        ds = buf("g.vit_ds", (B, ntok, D), f32)
        ds_b = buf("g.vit_ds_b", (B, ntok, D), f32)
        ds16 = buf("g.vit_ds16", (B, ntok, D)) if not self.fp32 else None
        hooked, depth = self.hooks, self.depth                       # blocks whose output gradient gets a readout gradient
        if need(f"vit.x{depth}"):                                    # every backbone hooks its last block
            bwd.add_cast(None, dtk[depth - 1], ds, ds16)
        for i in range(depth - 1, -1, -1):
            p, q = f"{pm}blocks.{i}.", f"vit{i}."
            v = vit[i]
            if i == depth // 2 - 1:
                ready("vit_hi")
            if not need(f"vit.x{i + 1}"):                            # nothing of this block or below is wanted
                continue
            if i in hooked and i != depth - 1:                       # the hooked tokens also feed a readout
                bwd.add_cast(ds, dtk[i], ds, ds16)
            g16 = ds if self.fp32 else ds16
            # mlp: x_{i+1} = xm + fc2(gelu(fc1(LN2(xm))))
            dmlp = buf("g.vit_mlp", v["mlp"].shape) if need(q + "u") else None
            self._gemm_bwd(f"blk{i}.fc2", g16.view(rows, -1), v["mlp"].view(rows, -1),
                           None if dmlp is None else dmlp.view(rows, -1), bias=False)
            if i in hooked and T(p + "mlp.fc2.bias"):                # else: written by block i+1's norm1 backward
                bwd.colsum(ds.view(rows, -1), G[p + "mlp.fc2.bias"].view(1, -1))
            if need(q + "u"):
                bwd.gelu_bwd(dmlp, v["u"], dmlp)
                dh = buf("g.vit_h", v["h2"].shape) if need(q + "h2") else None
                self._gemm_bwd(f"blk{i}.fc1", dmlp.view(rows, -1), v["h2"].view(rows, -1),
                               None if dh is None else dh.view(rows, -1))
            if not need(q + "h2"):
                continue
            # ds_b = gradient at attn.proj's output: its column sums are proj's bias gradient (same pass)
            dg, db = self._param_grads(p + "norm2.weight", p + "norm2.bias")
            bwd.layernorm_bwd(dh, xm[i], P[p + "norm2.weight"], ds, ds_b, ds16, dg, db,
                              dcolsum=G[p + "attn.proj.bias"] if T(p + "attn.proj.bias") else None)
            if not need(q + "xm"):
                continue
            g16 = ds_b if self.fp32 else ds16
            # attention: xm = x_i + proj(attn(qkv(LN1(x_i))))
            datt = buf("g.vit_att", v["att"].shape) if need(q + "att") else None
            self._gemm_bwd(f"blk{i}.proj", g16.view(rows, -1), v["att"].view(rows, -1),
                           None if datt is None else datt.view(rows, -1), bias=False)
            if not need(q + "att"):
                continue
            dqkv = buf("g.vit_qkv", v["qkv"].shape)
            bwd.attention_bwd(v["qkv"], v["att"], datt, v["lse"], dqkv, heads=self.heads, scale=0.125)
            self._gemm_bwd(f"blk{i}.qkv", dqkv.view(rows, -1), v["h1"].view(rows, -1),
                           dh.view(rows, -1) if need(q + "h1") else None)
            if not need(q + "h1"):
                continue
            # ds = gradient at block i-1's output = at its mlp.fc2 output, unless a hook adds to it first
            fc2_bias = f"{pm}blocks.{i - 1}.mlp.fc2.bias"
            fc2_bias = G[fc2_bias] if i >= 1 and (i - 1) not in hooked and T(fc2_bias) else None
            dg, db = self._param_grads(p + "norm1.weight", p + "norm1.bias")
            bwd.layernorm_bwd(dh, xs[i], P[p + "norm1.weight"], ds_b, ds, ds16, dg, db, dcolsum=fc2_bias)
        # ---- tokens: cls / pos_embed, patch projection
        df3 = None
        if need("vit.x0"):
            gpos = G[pm + "pos_embed"]
            want_pos, want_cls = T(pm + "pos_embed"), T(pm + "cls_token")
            if (gh, gw) == (24, 24) and want_pos:
                bwd.colsum(ds.view(B, ntok * D), gpos.view(1, -1))
                row0 = gpos[0, 0]
            elif want_pos or want_cls:                               # through the forward's resize of the patch rows
                dgrid = buf("g.pos_rows", (ntok, D), f32)
                bwd.colsum(ds.view(B, ntok * D), dgrid.view(1, -1))
                row0 = dgrid[0]
                if want_pos:
                    gpos[0, 0].copy_(dgrid[0])
                    bwd.pos_embed_resize_bwd(dgrid[1:], gh, gw, gpos[0, 1:])
                    row0 = gpos[0, 0]
            if want_cls:
                G[pm + "cls_token"].view(-1).copy_(row0)
            g16 = ds if self.fp32 else ds16
            dtok = g16[:, 1:, :].unsqueeze(1)
            # the bias gradient sums the patch rows of ds (below)
            if self.hybrid:
                f3 = S["f3"]
                df3 = buf("g.f3", f3.shape) if need("f3") else None
                self._gemm_bwd("proj", dtok, f3.view(B, 1, gh * gw, 1024),
                               None if df3 is None else df3.view(B, 1, gh * gw, 1024), bias=False)
            else:                                                    # Conv2d(3, D, 16, stride 16) = GEMM over patchify's columns
                cols = S["cols"]
                dcols = buf("g.patch_cols", cols.shape) if dx is not None else None
                self._gemm_bwd("proj", dtok, cols, dcols, bias=False)
                if dx is not None:
                    bwd.patch_input_grad(dcols.view(B * gh * gw, -1), dx)
            if T(pm + "patch_embed.proj.bias"):
                tmpb = buf("tmp.projbias", (B, D), f32)
                bwd.colsum(ds[:, 1:, :], tmpb, batches=B)
                bwd.colsum(tmpb, G[pm + "patch_embed.proj.bias"].view(1, -1))
        ready("vit_lo")
        if not self.hybrid:
            return self.flat_grad

        # ---- ResNetV2 bottlenecks, last to first
        d_out = df3
        for rec in reversed(S["blocks"]):
            tag, p, stride = rec["tag"], rec["p"], rec["stride"]
            s, b = rec["s"], rec["b"]
            # stage outputs also feed the decoder
            if (s, b) == (1, _STAGES[1][1] - 1) and need("layer_2"):
                bwd.mask_add(d_out, d_layers[1], a=d_out)
            if (s, b) == (0, _STAGES[0][1] - 1) and need("layer_1"):
                bwd.mask_add(d_out, d_layers[0], a=d_out)
            if not need(f"{tag}.out"):                                # nothing of this block or before it is wanted
                continue
            in_name = f"s{s}b{b - 1}.out" if b > 0 else (f"s{s - 1}b{_STAGES[s - 1][1] - 1}.out" if s > 0 else "stem.out")
            out, t_in = rec["out"], rec["t_in"]
            g = buf(f"g.{tag}_g", out.shape)
            bwd.mask_add(g, d_out, mask=out)                             # through the block's final ReLU
            dy3 = dy2 = dy1 = None
            if need(f"{tag}.r"):
                dy3 = buf(f"g.{tag}_y3", out.shape)
                dg, db = self._param_grads(p + "norm3.weight", p + "norm3.bias")
                bwd.groupnorm_bwd(g, rec["y3"], rec["st3"], P[p + "norm3.weight"], dy3, dg, db)
            da2 = buf(f"g.{tag}_a2", rec["a2"].shape) if need(f"{tag}.a2") else None
            self._gemm_bwd(tag + ".w3", dy3, rec["a2"], da2)
            if need(f"{tag}.a2"):
                dy2 = buf(f"g.{tag}_y2", rec["y2"].shape)
                dg, db = self._param_grads(p + "norm2.weight", p + "norm2.bias")
                bwd.groupnorm_bwd(da2, rec["y2"], rec["st2"], P[p + "norm2.weight"], dy2, dg, db, mask=rec["a2"])
            a1 = rec["a1"]
            need_a1 = need(f"{tag}.a1")
            da1 = buf(f"g.{tag}_a1", a1.shape) if need_a1 else None
            if stride == 1:
                self._gemm_bwd(tag + ".w2", dy2, a1, da1)
            else:
                if need_a1:
                    self._dgrad_s2(tag + ".w2", dy2, da1)
                planes = [a1[:, py::2, px::2, :] for py in range(2) for px in range(2)]
                self._wgrad(tag + ".w2", planes, ops._parity_taps("same"), dy2)
            if need_a1:
                dy1 = buf(f"g.{tag}_y1", rec["y1"].shape)
                dg, db = self._param_grads(p + "norm1.weight", p + "norm1.bias")
                bwd.groupnorm_bwd(da1, rec["y1"], rec["st1"], P[p + "norm1.weight"], dy1, dg, db, mask=a1)
            need_in = need(in_name)
            dt_in = buf(f"g.{tag}_in", t_in.shape) if need_in else None
            if b == 0:
                dd = None
                if need(f"{tag}.dn"):
                    dd = buf(f"g.{tag}_ds", rec["d"].shape)
                    dg, db = self._param_grads(p + "downsample.norm.weight", p + "downsample.norm.bias")
                    bwd.groupnorm_bwd(g, rec["d"], rec["std"], P[p + "downsample.norm.weight"], dd, dg, db)
                if stride > 1:                                       # the strided 1x1 conv: through strided views
                    if need_in:
                        dt_in.zero_()
                        ops.conv1x1(dd, Wt[tag + ".wd"][1], dt_in[:, ::stride, ::stride, :], bias=self._zb(Wt[tag + ".wd"][1]))
                    self._wgrad(tag + ".wd", [t_in[:, ::stride, ::stride, :]], bwd.TAPS_1, dd)
                else:
                    self._gemm_bwd(tag + ".wd", dd, t_in, dt_in)
            # w1: its input gradient adds to the shortcut's (b = 0) or to the skip connection's (b > 0)
            if need_in:
                w1 = Wt[tag + ".w1"][1]
                ops.conv1x1(dy1, w1, dt_in, residual=dt_in if b == 0 else g, bias=self._zb(w1))
            self._wgrad(tag + ".w1", [t_in], bwd.TAPS_1, dy1)
            d_out = dt_in
        # ---- stem
        bb = "pretrained.model.patch_embed.backbone."
        if need("stem.out"):
            cols, s0, st0, t = S["stem"]
            g_s0 = buf("g.stem_gn", s0.shape)
            bwd.stem_pool_bwd(d_out, s0, st0, P[bb + "stem.norm.weight"], P[bb + "stem.norm.bias"], g_s0)
            ds0 = buf("g.stem_conv", s0.shape)
            dg, db = self._param_grads(bb + "stem.norm.weight", bb + "stem.norm.bias")
            bwd.groupnorm_bwd(g_s0, s0, st0, P[bb + "stem.norm.weight"], ds0, dg, db)
            if dx is not None:
                bwd.stem_input_grad(ds0, self.pk["gemm"]["stem"], dx)
            if T(bb + "stem.conv.weight"):
                gp = self.gp[: 64 * 160].view(64, 160)
                h2, w2 = H // 2, W // 2
                bwd.conv_wgrad([cols.view(B, h2, w2, 160)], bwd.TAPS_1, ds0, gp)
                g147 = buf("tmp.stem_g", (64, 147), f32)
                g147.copy_(gp[:, :147])
                bwd.unpack_wgrad(g147, P[bb + "stem.conv.weight"], G[bb + "stem.conv.weight"], 64, 3, 49, 3, True)
        self._unpack("resnet", plan)
        ready("resnet")
        return self.flat_grad


def _trainable_names(names: List[str], flags) -> Optional[frozenset]:
    """requires-grad flags aligned with names -> the trainable set (None when every tensor trains)."""
    flags = tuple(bool(f) for f in flags)
    return None if all(flags) else frozenset(n for n, f in zip(names, flags) if f)


class _DptFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, engine, x, *params):
        ctx.trainable = _trainable_names(engine.param_names, ctx.needs_input_grad[2:])
        out = engine.forward(x, trainable=ctx.trainable)
        ctx.engine = engine
        ctx.x_shape, ctx.x_dtype = x.shape, x.dtype
        return out.clone()

    @staticmethod
    def backward(ctx, grad_out):
        """Gradients of the tensors that require grad only: None (no work, no copy) for frozen ones."""
        eng = ctx.engine
        want = ctx.needs_input_grad[2:]
        if not ctx.needs_input_grad[1] and not any(want):
            return (None,) * len(ctx.needs_input_grad)
        dx = None
        if ctx.needs_input_grad[1]:
            B, _, H, W = ctx.x_shape
            dx = torch.empty((B, 3, H, W), device=grad_out.device, dtype=torch.float32)
        eng.backward(grad_out, dx=dx, trainable=ctx.trainable)
        grads = tuple(eng.G[n].clone() if w else None for n, w in zip(eng.param_names, want))
        if dx is not None:
            dx = dx.reshape(ctx.x_shape).to(ctx.x_dtype)
        return (None, dx) + grads


def differentiable_forward(model: DPTDepthModel, x: torch.Tensor) -> torch.Tensor:
    """model(x) under autograd: returns a tensor whose backward fills p.grad of every parameter that requires grad and,
    when x requires grad, x.grad (the gradient w.r.t. the input image, in x's dtype).  Only those gradients are computed
    (backward_plan); the GEMM operands of frozen parameters are re-packed only when the parameters change."""
    if x.dim() == 4:
        check_input_size(x.shape[2], x.shape[3], model.arch["hybrid"], autograd=True)
    eng = getattr(model, "_train_engine", None)
    if eng is None or eng.fp32 != (model.precision == "fp32"):
        eng = TrainEngine(model, precision=model.precision)
        object.__setattr__(model, "_train_engine", eng)
    params = [p for _, p in model.named_parameters()]
    out = _DptFunction.apply(eng, x, *params)
    return out.squeeze(dim=1)


# ====================================================================================== the train step
def plan_grad_buckets(names: List[str], sizes: List[int]) -> List[Tuple[int, int, str]]:
    """Contiguous [start, end) ranges of the flat gradient buffer (state_dict order, padded sizes) in the order the
    backward COMPLETES them, so that each range can be all-reduced while the rest of the backward still runs, for a
    model of `depth` ViT blocks:
      DPT-Hybrid: decoder + reassemble (scratch.*, act_postprocess*) -> ViT blocks depth/2.. -> ViT blocks ..depth/2-1 +
      patch projection -> cls / pos_embed + the ResNetV2 stem and stages;
      plain ViTs: decoder + reassemble -> ViT blocks depth/2.. -> cls / pos_embed, patch embedding, ViT blocks ..depth/2-1.
    Returns (start, end, ready_after) with ready_after in {"decoder", "vit_hi", "vit_lo", "resnet"}."""
    offs, off = {}, 0
    for n, s in zip(names, sizes):
        offs[n] = (off, off + s)
        off += s
    total = off

    def first(pred):
        return min(offs[n][0] for n in names if pred(n))
    block = lambda n: int(n.split(".")[3]) if n.startswith("pretrained.model.blocks.") else -1
    depth = max(block(n) for n in names) + 1
    b_blocks = first(lambda n: n.startswith("pretrained.model.blocks."))
    b_proj = first(lambda n: n.startswith("pretrained.model.patch_embed.proj."))
    b_half = first(lambda n: block(n) >= depth // 2)
    b_tail = first(lambda n: n.startswith("pretrained.model.norm.") or n.startswith("pretrained.act_postprocess") or
                   n.startswith("scratch."))
    assert b_proj < b_blocks < b_half < b_tail
    if not any(n.startswith(_BB) for n in names):                    # plain ViT: nothing precedes the patch embedding
        return [(b_tail, total, "decoder"), (b_half, b_tail, "vit_hi"), (0, b_half, "vit_lo")]
    return [(b_tail, total, "decoder"), (b_half, b_tail, "vit_hi"), (b_proj, b_half, "vit_lo"), (0, b_proj, "resnet")]


class _FlatTrainStep:
    """What the fused train steps of the DPT-Hybrid share whatever the task: one process per GPU; forward -> the task's
    loss and its gradient w.r.t. the network output -> backward -> gradient all-reduce (data parallel, as the reference's
    PL DDP, train_depth.py:424-426: mean over ranks, bucketed, overlapped with the rest of the backward on a
    communication stream) -> clip_grad_norm_ -> Adam on the flat fp32 master weights.  step() returns the task's losses
    followed by the gradient norm before clipping, fp32 on the device, with no host synchronisation.

    The trainable set is the parameters that require grad when the step is constructed (the reference's
    `Adam(filter(lambda p: p.requires_grad, model.parameters()))`): the backward forms only their gradients, the clip
    norm and Adam cover only them, only the all-reduce buckets holding them are reduced, and frozen parameters and
    their moments are never written.  Changing requires_grad afterwards is an error (step() raises ValueError):
    construct a new step for a new set.

    A task subclass sets CHANNELS (the model's num_channels it trains) and `self.loss`, validates its inputs, and
    implements _loss_and_grad; a task with host-side inputs beyond the target tensors stages them for the captured
    step through _stage_extra / _refill_extra."""

    CHANNELS = 0
    _RING = 4           # host staging slots: the CPU may run at most _RING - 1 replays ahead of the GPU

    def __init__(self, model: DPTDepthModel, lr: float, clip: Optional[float], precision: str, input_size):
        import torch.distributed as dist
        from .optim import FlatAdam
        name = type(self).__name__
        if (input_size[0] // 16) * (input_size[1] // 16) > MAX_TRAIN_PATCHES:
            raise ValueError(f"{name}: training takes at most {MAX_TRAIN_PATCHES} patches, got input_size "
                             f"{tuple(input_size)}")
        if model.num_channels != self.CHANNELS:
            raise ValueError(f"{name} trains a model with num_channels={self.CHANNELS}, got num_channels="
                             f"{model.num_channels}")
        self.engine = TrainEngine(model, precision)
        eng = self.engine
        self.input_size = tuple(input_size)
        self._flag_params = [eng.params[n] for n in eng.param_names]
        self._flags = tuple(p.requires_grad for p in self._flag_params)
        if not any(self._flags):
            raise ValueError(f"{name}: no parameter requires grad")
        self.trainable = _trainable_names(eng.param_names, self._flags)
        sizes = [(eng.P[n].numel() + 3) // 4 * 4 for n in eng.param_names]
        segments = None if self.trainable is None else trainable_segments(eng.param_names, sizes, self.trainable)
        self.opt = FlatAdam(self.engine.flat, lr=lr, segments=segments)
        self.clip = clip
        self.dist = dist if (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1) else None
        self.world = self.dist.get_world_size() if self.dist else 1
        self.buckets = plan_grad_buckets(eng.param_names, sizes)
        if self.trainable is not None:
            self.buckets = select_buckets(self.buckets, eng.param_names, sizes, self.trainable)
        eng.prepare(self.trainable)
        self._frozen_sig = self._frozen_signature()
        self.comm_stream = torch.cuda.Stream(eng.device) if self.dist else None
        self.global_step = 0
        self.allreduce_bytes = sum(e - s for s, e, _ in self.buckets) * 4 if self.dist else 0
        self._hooks_done: Dict[str, torch.cuda.Event] = {}
        # The eager step issues ~1150 launches from Python and is host-bound at batch 16; with use_cuda_graph the whole
        # launch sequence (forward, loss, backward, clip, Adam) is captured once per input shape (and task key) and
        # replayed.  Single-process by default; graph_collectives=True also captures the NCCL all-reduces (fork / join
        # of the communication stream inside the capture).
        self.use_cuda_graph = False
        self.graph_collectives = False
        self._graphs: Dict[tuple, dict] = {}

    def _allreduce_bucket(self, tag: str):
        """called by the backward when the range `tag` of the flat gradient is final"""
        hit = [(s, e) for s, e, t in self.buckets if t == tag]
        if self.dist is None or not hit:                          # (a bucket of frozen tensors is not reduced)
            return
        s, e = hit[0]
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.engine.device))
        with torch.cuda.stream(self.comm_stream):
            self.comm_stream.wait_event(ev)
            self.dist.all_reduce(self.engine.flat_grad[s:e], op=self.dist.ReduceOp.AVG)

    def _check_trainable_set(self):
        if tuple(p.requires_grad for p in self._flag_params) != self._flags:
            name = type(self).__name__
            raise ValueError(f"{name}: requires_grad of the model's parameters changed since the step was "
                             f"constructed; construct a new {name} for a new trainable set")

    def _graph_mode(self) -> bool:
        return self.use_cuda_graph and (self.dist is None or self.graph_collectives)

    def _run(self, rgb, targets: tuple, extra, graph_key: tuple) -> torch.Tensor:
        """One validated step: rgb and the target tensors, the task's `extra` (passed to _loss_and_grad), and what
        besides the input shapes selects a captured graph."""
        if self._graph_mode():
            with torch.cuda.device(self.engine.device):             # capture / replay on the engine's device and stream
                return self._step_graph(rgb, targets, extra, graph_key)
        res = self._launch_sequence(rgb, targets, extra, scalars_on_device=False)
        self.global_step += 1
        return res

    def _loss_and_grad(self, out: torch.Tensor, targets: tuple, extra):
        """-> (losses fp32 [k], d loss / d out) of the network output `out`."""
        raise NotImplementedError

    def _launch_sequence(self, rgb, targets: tuple, extra, scalars_on_device: bool) -> torch.Tensor:
        eng = self.engine
        out = eng.forward(rgb, trainable=self.trainable)              # [B,C,H,W]
        losses, dpred = self._loss_and_grad(out, targets, extra)
        eng.backward(dpred, on_ready=self._allreduce_bucket, trainable=self.trainable)
        if self.dist is not None:
            torch.cuda.current_stream(eng.device).wait_stream(self.comm_stream)
        norm = self.opt.step(eng.flat_grad, max_norm=self.clip, scalars_on_device=scalars_on_device)
        k = losses.numel()
        res = torch.empty(k + 1, device=eng.device, dtype=torch.float32)
        res[:k].copy_(losses)
        res[k:k + 1].copy_(norm.reshape(1) if norm is not None else torch.zeros(1, device=eng.device))
        return res

    # ------------------------------------------------------------------ captured step
    def _stage_extra(self, g: dict, extra):
        """Capture time: device copies of the task's host inputs in graph `g` (and their pinned staging buffers in
        g["host"]); returns the `extra` the captured launch sequence reads."""
        return extra

    def _refill_extra(self, g: dict, h: dict, extra):
        """Before each replay: this step's host inputs through the staging slot `h` into graph `g`'s device copies."""

    def _capture(self, rgb, targets: tuple, extra) -> dict:
        eng, dev = self.engine, self.engine.device
        g = {"rgb": rgb.detach().float().contiguous().clone(),
             "targets": tuple(t.detach().float().contiguous().clone() for t in targets), "slot": 0,
             "host": [dict(scal=torch.zeros(2, dtype=torch.float32).pin_memory(), done=None) for _ in range(self._RING)]}
        extra = self._stage_extra(g, extra)
        # one eager step first (workspaces, kernel attributes, NCCL channels): a training step changes the weights and
        # the optimizer state, so both are put back before the capture
        snap = (eng.flat.clone(), self.opt.exp_avg.clone(), self.opt.exp_avg_sq.clone(), self.opt.step_count)
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            self.opt.stage_step_scalars(g["host"][0]["scal"])
            self._launch_sequence(g["rgb"], g["targets"], extra, scalars_on_device=True)
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        eng.flat.copy_(snap[0]); self.opt.exp_avg.copy_(snap[1]); self.opt.exp_avg_sq.copy_(snap[2])
        self.opt.step_count = snap[3]
        del snap
        graph = torch.cuda.CUDAGraph()
        # with NCCL in the capture, other threads of the process (the process group's watchdog) keep making CUDA calls:
        # restrict the capture's error checking to this thread
        mode = "thread_local" if self.dist is not None else "global"
        with torch.cuda.graph(graph, capture_error_mode=mode):
            g["res"] = self._launch_sequence(g["rgb"], g["targets"], extra, scalars_on_device=True)
        g["graph"] = graph
        g["scratch"] = bwd._SCRATCH.buf        # the shared kernel workspace the captured launches point into stays alive
        return g

    def _frozen_signature(self):
        """(version, pointer) of every frozen parameter: the captured step packs only the trainable layers, so a change
        of a frozen one (load_state_dict, copy_) invalidates the graphs."""
        if self.trainable is None:
            return None
        return tuple((p._version, p.data_ptr()) for n, p in zip(self.engine.param_names, self._flag_params)
                     if n not in self.trainable)

    def _step_graph(self, rgb, targets: tuple, extra, graph_key: tuple) -> torch.Tensor:
        sig = self._frozen_signature()
        if sig != self._frozen_sig:
            self._graphs.clear()                                     # re-captured below, re-packing the changed operands
            self._frozen_sig = sig
        shapes = (tuple(rgb.shape),) + tuple(tuple(t.shape) for t in targets)
        key = shapes + tuple(graph_key)
        g = self._graphs.get(key)
        if g is None:
            # the engine's activation buffers are re-allocated when the input shape changes: graphs of other shapes
            # would replay into freed memory
            for k in [k for k in self._graphs if k[:len(shapes)] != shapes]:
                del self._graphs[k]
            g = self._graphs[key] = self._capture(rgb, targets, extra)
        h = g["host"][g["slot"]]
        g["slot"] = (g["slot"] + 1) % self._RING
        if h["done"] is not None:
            h["done"].synchronize()                                 # the replay that last read this staging slot has run
        g["rgb"].copy_(rgb)
        for dst, t in zip(g["targets"], targets):
            dst.copy_(t)
        self._refill_extra(g, h, extra)
        self.opt.stage_step_scalars(h["scal"])
        g["graph"].replay()
        h["done"] = torch.cuda.Event()
        h["done"].record(torch.cuda.current_stream(self.engine.device))
        self.global_step += 1
        return g["res"].clone()


class DepthTrainStep(_FlatTrainStep):
    """The train step of the depth model (num_channels=1).  step(rgb, depth_gt, mask_float): forward -> clamp + MiDaS SSI
    + gradient-matching + virtual normal loss (DepthStepLoss) -> backward -> bucketed gradient all-reduce ->
    clip_grad_norm_(10) -> Adam(lr) on the flat fp32 master weights (train_depth.py:381-383,
    Trainer(gradient_clip_val=10)).  Trainable set, data parallelism and CUDA-graph replay: _FlatTrainStep."""

    CHANNELS = 1

    def __init__(self, model: DPTDepthModel, lr: float = 1e-5, clip: Optional[float] = 10.0, precision: str = "bf16",
                 input_size=(384, 384)):
        from .losses import DepthStepLoss
        super().__init__(model, lr, clip, precision, input_size)
        self.loss = DepthStepLoss(input_size)

    @torch.no_grad()
    def step(self, rgb: torch.Tensor, depth_gt: torch.Tensor, mask_float: torch.Tensor, points=None,
             full_mix: Optional[bool] = None) -> torch.Tensor:
        """-> fp32 [5] on the device: (loss, ssi, reg, vn, gradient norm before clipping); no host synchronisation.
        rgb [B,3,H,W], depth_gt and mask_float [B,1,H,W] with (H, W) = the step's input_size; `points`: host index
        arrays in [0, H*W)."""
        from .losses import check_vnl_points
        self._check_trainable_set()
        H, W = self.input_size
        if rgb.dim() != 4 or tuple(rgb.shape[1:]) != (3, H, W):
            raise ValueError(f"DepthTrainStep: rgb must be [B,3,{H},{W}] (the step's input_size), got {tuple(rgb.shape)}")
        B = rgb.shape[0]
        for name, t in (("depth_gt", depth_gt), ("mask_float", mask_float)):
            if tuple(t.shape[-2:]) != (H, W) or t.numel() != B * H * W:
                raise ValueError(f"DepthTrainStep: {name} must be [{B},1,{H},{W}], got {tuple(t.shape)}")
        if points is not None:
            check_vnl_points(points, H, W)
        if full_mix is None:
            full_mix = self.global_step >= 15000                     # train_depth.py:274-279
        full_mix = bool(full_mix)
        if self._graph_mode() and full_mix and points is None:
            points = self.loss.vnl.select_index()                   # host NumPy RNG, the reference's call sequence
        return self._run(rgb, (depth_gt, mask_float), (points, full_mix), (full_mix,))

    def _loss_and_grad(self, out, targets, extra):
        (depth_gt, mask_float), (points, full_mix) = targets, extra
        return self.loss(out, depth_gt, mask_float, full_mix=full_mix, points=points)

    def _stage_extra(self, g, extra):
        """the VNL index arrays: device copies the captured loss gathers at, refilled through pinned slots"""
        points, full_mix = extra
        g["pts"] = None
        if full_mix:
            arrs = [np.ascontiguousarray(q, dtype=np.int32) for q in points]
            g["pts"] = [torch.from_numpy(a).to(self.engine.device) for a in arrs]
            for h in g["host"]:
                h["pts"] = [torch.empty(a.shape, dtype=torch.int32).pin_memory() for a in arrs]
        return g["pts"], full_mix

    def _refill_extra(self, g, h, extra):
        points, full_mix = extra
        if full_mix:
            for dst, hp, q in zip(g["pts"], h["pts"], points):
                hp.copy_(torch.from_numpy(np.ascontiguousarray(q, dtype=np.int32)))
                dst.copy_(hp, non_blocking=True)


class NormalTrainStep(_FlatTrainStep):
    """The train step of the surface-normal model (num_channels=3, hubconf.surface_normal_dpt_hybrid_384).
    step(rgb, normal_gt, mask_float): forward -> clamp + masked L1 + masked cosine angular loss, loss = cos + 10 l1
    (NormalStepLoss, the arithmetic of train_normal.py:247-265) -> backward -> bucketed gradient all-reduce ->
    clip_grad_norm_(clip) -> Adam(lr) on the flat fp32 master weights.  lr and clip default to DepthTrainStep's.
    Trainable set, data parallelism and CUDA-graph replay: _FlatTrainStep."""

    CHANNELS = 3

    def __init__(self, model: DPTDepthModel, lr: float = 1e-5, clip: Optional[float] = 10.0, precision: str = "bf16",
                 input_size=(384, 384)):
        from .losses import NormalStepLoss
        super().__init__(model, lr, clip, precision, input_size)
        self.loss = NormalStepLoss()

    @torch.no_grad()
    def step(self, rgb: torch.Tensor, normal_gt: torch.Tensor, mask_float: torch.Tensor) -> torch.Tensor:
        """-> fp32 [4] on the device: (loss, l1, cos, gradient norm before clipping); no host synchronisation.
        rgb and normal_gt [B,3,H,W], mask_float [B,1,H,W] with (H, W) = the step's input_size."""
        self._check_trainable_set()
        H, W = self.input_size
        if rgb.dim() != 4 or tuple(rgb.shape[1:]) != (3, H, W):
            raise ValueError(f"NormalTrainStep: rgb must be [B,3,{H},{W}] (the step's input_size), got {tuple(rgb.shape)}")
        B = rgb.shape[0]
        for name, t, c in (("normal_gt", normal_gt, 3), ("mask_float", mask_float, 1)):
            if tuple(t.shape) != (B, c, H, W):
                raise ValueError(f"NormalTrainStep: {name} must be [{B},{c},{H},{W}], got {tuple(t.shape)}")
        return self._run(rgb, (normal_gt, mask_float), None, ())

    def _loss_and_grad(self, out, targets, extra):
        return self.loss(out, *targets)
