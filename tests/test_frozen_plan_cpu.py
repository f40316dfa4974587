"""Backward plan of a partly frozen DPT-Hybrid (train.backward_plan), and the segment / bucket selection of the train
step: pure functions over the parameter names, no GPU needed."""
import pytest

from omnidata_b200 import optim, train
from omnidata_b200.model import DPTDepthModel

BB = "pretrained.model.patch_embed.backbone."
DEAD = ("pretrained.model.head.", "pretrained.model.norm.", "scratch.refinenet4.resConfUnit1.")


@pytest.fixture(scope="module")
def model_params():
    m = DPTDepthModel(backbone="vitb_rn50_384")
    names = [n for n, _ in m.named_parameters()]
    sizes = [(p.numel() + 3) // 4 * 4 for _, p in m.named_parameters()]
    return names, sizes


def _acts(plan, prefix):
    return {a: v for a, v in plan.acts.items() if a.startswith(prefix)}


def test_all_trainable_is_todays_plan(model_params):
    names, _ = model_params
    for want_dx in (False, True):
        plan = train.backward_plan(names, None, want_dx)
        assert plan.full and len(names) == 368
        assert all(plan.grad(n) for n in names)
        # every activation gradient the backward forms today (the input's only when x.grad is wanted)
        assert all(v for a, v in plan.acts.items() if a != "x") and plan.act("x") == want_dx
        assert train.backward_plan(names, set(names), want_dx).full


def test_encoder_frozen(model_params):
    names, _ = model_params
    plan = train.backward_plan(names, {n for n in names if n.startswith("scratch.")}, False)
    assert not plan.full
    # the four layerN_rn convolutions: weight gradients, no gradient w.r.t. their inputs
    assert all(plan.act(f"rn{n}.o") and not plan.act(f"layer_{n}") for n in (1, 2, 3, 4))
    assert not any(v for a, v in plan.acts.items() if not (a.startswith(("ff", "head.", "rn")) or a == "out"))
    assert all(plan.act(a) for a in ("head.a", "head.h1", "ff1.z", "ff4.z", "ff4.rcu2.t", "ff1.rcu1.t"))
    assert not plan.grad("pretrained.act_postprocess4.4.weight") and plan.grad("scratch.layer1_rn.weight")


def test_top_blocks_and_decoder(model_params):
    names, _ = model_params
    keep = tuple(f"pretrained.model.blocks.{i}." for i in (8, 9, 10, 11)) + ("scratch.",)
    plan = train.backward_plan(names, {n for n in names if n.startswith(keep)}, False)
    # stops at block 8's input; layer_1 / layer_2 get no gradient; nothing in the ResNetV2
    assert plan.act("vit8.h1") and not plan.act("vit.x8") and not plan.act("vit7.u")
    assert not plan.act("layer_1") and not plan.act("layer_2")
    assert plan.act("layer_3") and plan.act("layer_4")                 # readouts pass the gradient to blocks 8 / 11
    assert not any(v for a, v in plan.acts.items() if a.startswith(("s0", "s1", "s2", "stem")) or a in ("f3", "vit.x0"))


def test_everything_frozen_input_gradient(model_params):
    names, _ = model_params
    plan = train.backward_plan(names, set(), True)
    assert all(plan.acts.values())                                     # every dgrad down to the image
    assert not any(plan.grad(n) for n in names)                        # no wgrad, colsum, unpack or norm affine
    plan = train.backward_plan(names, set(), False)
    assert not any(plan.acts.values())


def test_frozen_weight_trainable_bias(model_params):
    names, _ = model_params
    b = "scratch.refinenet2.out_conv.bias"
    plan = train.backward_plan(names, {b}, False)
    assert plan.grad(b) and not plan.grad("scratch.refinenet2.out_conv.weight")
    assert plan.act("ff2.z") and plan.act("ff1.z") and plan.act("head.a")
    assert not plan.act("ff2.y") and not plan.act("rn2.o") and not plan.act("ff3.z")
    g = BB + "stages.1.blocks.2.norm2.bias"                            # half of a norm's affine pair
    plan = train.backward_plan(names, {g}, False)
    assert plan.act("s1b2.a2") and not plan.act("s1b2.y2") and plan.act("f3") and not plan.act("s1b1.out")


def test_only_pos_embed_and_cls_token(model_params):
    names, _ = model_params
    plan = train.backward_plan(names, {"pretrained.model.pos_embed", "pretrained.model.cls_token"}, False)
    assert plan.act("vit.x0") and plan.act("vit.x12") and plan.act("vit0.h1")
    assert not plan.act("f3") and not any(v for a, v in plan.acts.items() if a.startswith(("s0", "s1", "s2", "stem")))


def test_dead_tensors_need_nothing(model_params):
    names, _ = model_params
    dead = [n for n in names if n.startswith(DEAD)]
    assert len(dead) == 8
    plan = train.backward_plan(names, set(dead), False)
    assert plan.grad(dead[0]) and not any(plan.acts.values())


def test_plan_rejects_unknown_names(model_params):
    names, _ = model_params
    with pytest.raises(ValueError):
        train.backward_plan(names, {"no.such.tensor"}, False)


def test_segments_cover_exactly_the_trainable_tensors(model_params):
    names, sizes = model_params
    offs, o = {}, 0
    for n, s in zip(names, sizes):
        offs[n] = (o, o + s)
        o += s
    for trainable in ({n for n in names if n.startswith("scratch.")},
                      {n for n in names if n.endswith(".bias")},
                      {"pretrained.model.pos_embed", "scratch.output_conv.4.bias"}):
        segs = train.trainable_segments(names, sizes, trainable)
        covered = set()
        for s, e in segs:
            covered |= {n for n in names if s <= offs[n][0] and offs[n][1] <= e}
            assert all(not (s < offs[n][1] and offs[n][0] < e) for n in names if n not in trainable)
        assert covered == trainable
        assert all(segs[k][1] < segs[k + 1][0] for k in range(len(segs) - 1))       # merged, ascending
        assert optim.check_segments(segs, o) == sum(offs[n][1] - offs[n][0] for n in trainable)
    assert train.trainable_segments(names, sizes, set(names)) == [(0, o)]


def test_check_segments_rejects_bad_tables():
    for bad in ([], [(0, 8), (4, 12)], [(2, 8)], [(0, 6), (8, 12)], [(0, 100)], [(8, 8)]):
        with pytest.raises(ValueError):
            optim.check_segments(bad, 64)
    assert optim.check_segments([(0, 8), (16, 19)], 64) == 11


def test_buckets_without_trainable_tensors_are_dropped(model_params):
    names, sizes = model_params
    buckets = train.plan_grad_buckets(names, sizes)
    sel = train.select_buckets(buckets, names, sizes, {n for n in names if n.startswith("scratch.")})
    assert [t for *_, t in sel] == ["decoder"]
    keep = {n for n in names if n.startswith(("pretrained.model.blocks.10.", BB + "stem."))}
    assert [t for *_, t in train.select_buckets(buckets, names, sizes, keep)] == ["vit_hi", "resnet"]
    assert train.select_buckets(buckets, names, sizes, set(names)) == buckets
    assert train.select_buckets(buckets, names, sizes, set()) == []
