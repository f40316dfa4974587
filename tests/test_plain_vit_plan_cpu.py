"""Backward plan, all-reduce buckets and C-ABI signature of the plain-ViT DPTs' train step (vitl16_384, vitb16_384)."""
from pathlib import Path

import pytest

from omnidata_b200 import train
from omnidata_b200.model import _ARCH, state_dict_spec

ROOT = Path(__file__).resolve().parents[1]
PLAIN = ("vitl16_384", "vitb16_384")
DEAD = ("pretrained.model.norm.", "pretrained.model.head.", "scratch.refinenet4.resConfUnit1.")


def _names(backbone):
    return [k for k, _ in state_dict_spec(1, backbone=backbone)]


@pytest.mark.parametrize("backbone", PLAIN)
def test_dag_names_every_live_parameter(backbone):
    names = _names(backbone)
    named = {p for params, _, _ in train._backward_graph(_ARCH[backbone]) for p in params}
    live = {n for n in names if not n.startswith(DEAD)}
    assert named == live
    plan = train.backward_plan(names, None, False, backbone)
    assert plan.full and not plan.act("x") and plan.act("vit.x0") and plan.act("layer_1")


@pytest.mark.parametrize("backbone", PLAIN)
def test_frozen_encoder_leaves_no_vit_gradient(backbone):
    names = _names(backbone)
    depth = _ARCH[backbone]["depth"]
    plan = train.backward_plan(names, {n for n in names if n.startswith("scratch.")}, False, backbone)
    assert not any(plan.grad(n) for n in names if n.startswith("pretrained."))
    assert not any(plan.act(a) for a in [f"vit.x{i}" for i in range(depth + 1)] + [f"ro{n}.r" for n in (1, 2, 3, 4)])
    assert not any(plan.act(f"pp{n}.o") for n in (1, 2, 3, 4))
    assert all(plan.act(f"layer_{n}") is False for n in (1, 2, 3, 4))
    assert plan.act("ff1.z") and plan.act("rn1.o")


@pytest.mark.parametrize("backbone", PLAIN)
def test_want_dx_alone_reaches_the_image(backbone):
    names = _names(backbone)
    plan = train.backward_plan(names, set(), True, backbone)
    assert not plan.trainable and plan.act("x") and plan.act("vit.x0") and plan.act("pp1.o") and plan.act("layer_1")
    assert not train.backward_plan(names, set(), False, backbone).act("vit.x0")


def _sizes(backbone):
    import math
    return [(math.prod(s) + 3) // 4 * 4 for _, s in state_dict_spec(1, backbone=backbone)]


@pytest.mark.parametrize("backbone", PLAIN)
def test_buckets_cover_the_flat_buffer_and_split_at_half_depth(backbone):
    names, sizes = _names(backbone), _sizes(backbone)
    buckets = train.plan_grad_buckets(names, sizes)
    assert [t for _, _, t in buckets] == ["decoder", "vit_hi", "vit_lo"]
    spans = sorted((s, e) for s, e, _ in buckets)
    assert spans[0][0] == 0 and spans[-1][1] == sum(sizes)
    assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
    offs, off = {}, 0
    for n, s in zip(names, sizes):
        offs[n] = off
        off += s
    half = _ARCH[backbone]["depth"] // 2
    vit_lo = [b for b in buckets if b[2] == "vit_lo"][0]
    assert vit_lo[1] == offs[f"pretrained.model.blocks.{half}.norm1.weight"]


def test_hybrid_buckets_unchanged():
    names, sizes = _names("vitb_rn50_384"), _sizes("vitb_rn50_384")
    offs, off = {}, 0
    for n, s in zip(names, sizes):
        offs[n] = off
        off += s
    expect = [(offs["pretrained.model.norm.weight"], off, "decoder"),
              (offs["pretrained.model.blocks.6.norm1.weight"], offs["pretrained.model.norm.weight"], "vit_hi"),
              (offs["pretrained.model.patch_embed.proj.weight"], offs["pretrained.model.blocks.6.norm1.weight"], "vit_lo"),
              (0, offs["pretrained.model.patch_embed.proj.weight"], "resnet")]
    assert train.plan_grad_buckets(names, sizes) == expect


def test_patch_input_grad_signature_matches_header():
    import ctypes as C
    from omnidata_b200 import _capi
    text = (ROOT / "include" / "omnidata_b200.h").read_text()
    assert "int odb_patch_input_grad(const void* dcols, float* dx, int32_t b, int32_t h, int32_t w, int32_t patch, " \
           "int32_t dtype,\n                         void* stream);" in text
    res, args = _capi._SIGNATURES["odb_patch_input_grad"]
    assert res is C.c_int and args == [C.c_void_p] * 2 + [C.c_int32] * 5 + [C.c_void_p]
