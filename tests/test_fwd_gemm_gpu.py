"""The forward GEMMs and attention of the three DPTs against float64 at every geometry the models launch.

Every ops.conv_gemm and ops.attention launch of a real forward is recorded by wrapping the two entry points: the
inference forward (DPTDepthModel in eval mode) and the train forward (TrainEngine.forward, which differs at the five
points marked in model.dpt_forward), for the DPT-Hybrid (`vitb_rn50_384`), DPT-Large (`vitl16_384`) and the plain
ViT-B (`vitb16_384`), in bf16 and fp32, at batch 2 and four input sizes.  Added to those: the hybrid at batch 32
(bench.py's inference workload), the hybrid and DPT-Large train forwards at batch 16 (the train benchmarks), where
the tile planner (make_plan in csrc/conv_gemm.cu) picks 256-wide N tiles for nearly every layer, and the surface-normal
model (head_c = 3).  Each distinct geometry (shapes, strides, aliasing, flags) is replayed on seeded operands in
guarded buffers (oracle/guard.py): every output element written, nothing else changed (inputs, guard bands, and the
GroupNorm partial-sum buffer beyond the rows the plan names), a second run bit-identical, and each output compared with
oracle/gemm_oracle.py per element.

Bounds, "measured X, bound Y" with X the largest value over every case of this file, measured on an NVIDIA H100 80GB
HBM3 with a 400 W power limit (the inputs are seeded, so the numbers repeat).  tau is the error over the magnitude of
the sum an fp32-accumulated element is made of, tau = |kernel - ref| / (|x| |W| + |bias| + |residual|):
  * bf16 output: |k - ref| <= 0.5 ulp + tau * scale, the one rounding of the fp32 result: measured tau 6.4e-7,
    bound 2e-6.  A GELU output (and the GELU out2 copy) gets one ulp and tau * max|gelu'| (1.13) * scale: measured
    4.2e-8, bound 2e-7.  The relu out2 copy equals relu(out) exactly.
  * fp32 output from bf16 operands (the ViT residual stream, EPI_BIAS_RES_F32): no rounding term, measured tau 6.5e-7,
    bound 2e-6.  fp32 mode (the FP32-pipe twin): measured tau 2.3e-7, bound 5e-7.
  * GroupNorm statistics of the unrounded conv result: mean error over the group's rms measured 3.7e-7, bound 5e-7;
    rstd relative error measured 2.2e-6, bound 3e-6 (var = E[x^2] - mean^2 from fp32 partial sums).
  * head tail (relu(conv + bias) -> 1x1 conv -> relu, fp32 NCHW): error over (scale of the conv) |w| + |b|: measured
    5.4e-8, bound 2e-7.
  * attention bf16, against the rounded oracle (P rounded as the kernel rounds it): an element passes within one bf16
    ulp plus ATT_ABS = 1e-3 x the rms of its image and head block; a rounding flip of P moves a few elements further:
    measured fraction 2.6e-5, bound 5e-5, and no element beyond 3.7 such units, bound 8.  Against the exact result:
    measured rel-L2 2.25e-3, bound 4e-3.  lse (log2-sum-exp, the backward's starting point): measured max abs error
    1.4e-6, bound 5e-6.  fp32 against the exact result: measured rel-L2 8.4e-8, bound 2e-7.
"""
import ctypes as C

import pytest
import torch

from oracle import gemm_oracle as G
from oracle.guard import checked_launch, geometry, materialize, same_storage, ulp_bf16

pytestmark = pytest.mark.gpu

TAU = {"bf16": 2e-6, "gelu": 2e-7, "f32out": 2e-6, "fp32": 5e-7, "head": 2e-7}
GN_MEAN, GN_RSTD = 5e-7, 3e-6
ATT_ABS, ATT_FLIPS, ATT_MAX, ATT_EXACT, ATT_LSE, ATT_F32 = 1e-3, 5e-5, 8.0, 4e-3, 5e-6, 2e-7
GELU_SLOPE = 1.13                      # max |gelu'(x)| = 1.1289 (at x = sqrt(2))

SIZES = [(384, 384), (320, 480), (64, 96), (96, 1664)]
BACKBONES = ["vitb_rn50_384", "vitl16_384", "vitb16_384"]
SEEN = {}                              # (block_n, pair, halo, epilogue) -> launches, over every recording of the run


def dev():
    return torch.device("cuda:0")


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-300))


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    print("(block_n, cta pair, halo, epilogue) -> launches: " +
          ", ".join(f"{k}: {v}" for k, v in sorted(SEEN.items(), key=str)))


# ------------------------------------------------------------------------------------------ recording
def _model(backbone, num_channels):
    from omnidata_b200 import synthetic
    from omnidata_b200.model import DPTDepthModel, state_dict_spec
    model = DPTDepthModel(backbone=backbone, num_channels=num_channels)
    sd = synthetic.make_state_dict(0, num_channels, spec=state_dict_spec(num_channels, backbone=backbone))
    model.load_state_dict(sd, strict=True)
    return model.to(dev())


def _epilogue(ts, flags, plan):
    """The epilogue body odb_conv_gemm selects (the launch_fast conditions of its host code) for a bf16 launch."""
    act, _, out2_act, head_relu = flags
    out, res = ts["out"], ts["residual"]
    if head_relu is not None:
        return "head"
    if out.dtype == torch.float32:
        return "bias_res_f32"
    fast = not plan[3] & 2 and plan[2] >= 64 and out2_act is None
    if fast and ts["bias"] is None and ts["gn_partial"] is not None and res is None and act == 0:
        return "gn"
    if fast and ts["bias"] is not None and ts["gn_partial"] is None:
        if res is None:
            return ("bias", "bias_relu", "bias_gelu")[act]
        if act == 0 and G.as4(res).shape[0] == G.as4(out).shape[0]:
            return "bias_res"
    return "generic"


def _record(backbone, size, precision, batch, mode, num_channels=1):
    """One forward (mode "eval": DPTDepthModel inference; "train": TrainEngine.forward) -> {key: launches} and
    {key: plan} for every distinct conv_gemm / attention launch."""
    from omnidata_b200 import _capi, ops
    from omnidata_b200.train import TrainEngine
    H, W = size
    model = _model(backbone, num_channels)
    g = torch.Generator(device="cpu").manual_seed(H * 7 + W + batch)
    x = (torch.rand(batch, 3, H, W, generator=g) * 2 - 1).to(dev())
    geoms, plans, last = {}, {}, {}
    conv0, attn0 = ops.conv_gemm, ops.attention
    lib = _capi.lib()
    launch0 = lib.odb_conv_gemm
    modeled = {"bias", "bias_per_image", "residual", "act", "out2", "out2_act", "gn_stats", "head"}

    def launch(desc, stream):                         # the planner's choice for the launch being recorded
        if desc._obj.in_dtype == _capi.DTYPE_BF16:
            plan = (C.c_int32 * 4)()
            _capi.check(lib.odb_conv_gemm_plan(desc, plan), "odb_conv_gemm_plan")
            last["plan"] = tuple(plan)
        return launch0(desc, stream)

    def conv(views, taps, weight, out, **kw):
        extra = set(kw) - modeled
        assert not extra, f"conv_gemm flags the replay does not model: {sorted(extra)}"
        gn, head = kw.get("gn_stats"), kw.get("head")
        ts = {f"v{i}": v for i, v in enumerate(views)}
        ts.update(weight=weight, out=out, bias=kw.get("bias"), residual=kw.get("residual"), out2=kw.get("out2"),
                  gn_partial=gn[0] if gn else None, gn_stats=gn[1] if gn else None,
                  head_w=head[0] if head else None, head_b=head[1] if head else None, head_out=head[2] if head else None)
        flags = (kw.get("act", 0), bool(kw.get("bias_per_image", False)),
                 kw.get("out2_act", ops.ACT_RELU) if kw.get("out2") is not None else None,
                 bool(head[3]) if head else None)
        key = ("conv", geometry(ts), tuple(map(tuple, taps)), flags)
        last.pop("plan", None)
        r = conv0(views, taps, weight, out, **kw)
        if "plan" in last:
            plans[key] = last["plan"]
            combo = last["plan"][2:3] + (bool(last["plan"][3] & 1), bool(last["plan"][3] & 2), _epilogue(ts, flags, last["plan"]))
            SEEN[combo] = SEEN.get(combo, 0) + 1
        geoms[key] = geoms.get(key, 0) + 1
        return r

    def attention(qkv, out, heads=12, scale=0.125, lse=None):
        key = ("attn", geometry(dict(qkv=qkv, out=out, lse=lse)), (), (heads, scale))
        geoms[key] = geoms.get(key, 0) + 1
        return attn0(qkv, out, heads=heads, scale=scale, lse=lse)

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ops, "conv_gemm", conv)
        mp.setattr(ops, "attention", attention)
        mp.setattr(lib, "odb_conv_gemm", launch)
        if mode == "eval":
            model.eval()
            model.precision = precision
            with torch.no_grad():
                model(x)
        else:
            TrainEngine(model.train(), precision).forward(x)
        torch.cuda.synchronize()
    del model
    torch.cuda.empty_cache()
    return geoms, plans


# ------------------------------------------------------------------------------------------ checks
def _tau(k, ref, scale, rounding_ulps):
    """max over elements of (|k - ref| - rounding_ulps bf16 ulps) / scale."""
    err = (k.double() - ref).abs()
    if rounding_ulps:
        err = (err - rounding_ulps * torch.maximum(ulp_bf16(k), ulp_bf16(ref))).clamp_min(0)
    return float((err / scale.clamp_min(1e-30)).max())


def check_conv(key, plan, seed):
    """Replays one recorded conv_gemm launch -> {class: worst value}."""
    from omnidata_b200 import ops
    _, geom, taps, (act, bias_per_image, out2_act, head_relu) = key
    bufs, ts = materialize(geom, gen(seed))
    views = [ts[f"v{i}"] for i in range(4) if f"v{i}" in ts]
    taps = list(taps)
    w, out, bias, res, out2 = ts["weight"], ts["out"], ts["bias"], ts["residual"], ts["out2"]
    gpart, gstats, hw, hb, hout = ts["gn_partial"], ts["gn_stats"], ts["head_w"], ts["head_b"], ts["head_out"]
    if hout is not None:
        grid = (hout.shape[0], hout.shape[2], hout.shape[3])
    else:
        grid = tuple(G.as4(out).shape[:3])
    # the references, from the operands before the launch (the residual may be the output itself)
    ref = G.conv_gemm_ref(views, taps, w, grid, bias=bias, residual=res, act=act, bias_per_image=bias_per_image,
                          out2_act=out2_act)
    ref, ref2 = ref if out2_act is not None else (ref, None)
    scale = G.conv_acc_ref(views, taps, w, grid, absolute=True)
    if bias is not None:
        scale = scale + (bias.double().abs()[:, None, None, :] if bias_per_image else bias.double().abs())
    if res is not None:
        scale = scale + (res.double().abs().unsqueeze(0) if res.dim() == 3 else G.as4(res).double().abs())
    outs = [t for t in (out, out2, gstats, hout) if t is not None]
    if gpart is not None:
        # the partial sums the plan names: [B][tiles_y * tiles_x][4 quadrants][groups][2]; the rest must stay as it is
        outs.append(gpart[:grid[0] * plan[0] * plan[1] * 4 * 32 * 2])
    kw = dict(bias=bias, bias_per_image=bias_per_image, residual=res, act=act)
    if out2 is not None:
        kw.update(out2=out2, out2_act=out2_act)
    if gpart is not None:
        kw.update(gn_stats=(gpart, gstats))
    if hout is not None:
        kw.update(head=(hw, hb, hout, head_relu))
    got = checked_launch(bufs, outs, lambda: ops.conv_gemm(views, taps, w, out, **kw),
                         prefill_nan=not same_storage(res, out))
    got = dict(zip([id(t) for t in outs], got))
    r = {}
    if hout is not None:
        hscale = scale @ hw.double().abs().t() + hb.double().abs()
        r["head"] = _tau(got[id(hout)], G.head_tail_ref(ref, hw, hb, head_relu), hscale.permute(0, 3, 1, 2), 0)
        assert r["head"] <= TAU["head"], r
        return r
    k = G.as4(got[id(out)])
    if views[0].dtype == torch.float32:
        cls, ulps, slope = "fp32", 0, 1.0
    elif out.dtype == torch.float32:
        cls, ulps, slope = "f32out", 0, 1.0
    elif act == 2:
        cls, ulps, slope = "gelu", 1, GELU_SLOPE
    else:
        cls, ulps, slope = "bf16", 0.5, 1.0
    r[cls] = _tau(k, ref, slope * scale, ulps)
    if out2 is not None:
        k2 = G.as4(got[id(out2)])
        if out2_act == ops.ACT_RELU:
            assert torch.equal(k2, torch.relu(k)), "the relu copy is not relu(out)"
        else:
            r["gelu"] = max(r.get("gelu", 0.0), _tau(k2, ref2, GELU_SLOPE * scale, 1))
    if gstats is not None:
        st = got[id(gstats)].double()
        gref = G.gn_stats_ref(ref)
        b = ref.shape[0]
        rms = ref.reshape(b, -1, 32, ref.shape[-1] // 32).transpose(1, 2).reshape(b, 32, -1).pow(2).mean(-1).sqrt()
        r["gn mean"] = float(((st[..., 0] - gref[..., 0]).abs() / rms).max())
        r["gn rstd"] = float(((st[..., 1] - gref[..., 1]).abs() / gref[..., 1]).max())
        assert r["gn mean"] <= GN_MEAN and r["gn rstd"] <= GN_RSTD, r
    assert all(r[c] <= TAU[c] for c in r if c in TAU), r
    return r


def check_attention(key, seed):
    from omnidata_b200 import ops
    _, geom, _, (heads, scale) = key
    bufs, ts = materialize(geom, gen(seed))
    qkv, out, lse = ts["qkv"], ts["out"], ts["lse"]
    outs = [out] if lse is None else [out, lse]
    got = checked_launch(bufs, outs, lambda: ops.attention(qkv, out, heads=heads, scale=scale, lse=lse))
    exact = G.attention_ref(qkv, heads, scale=scale)
    k = got[0].double()
    if qkv.dtype == torch.float32:
        r = {"fp32 exact": rel(k, exact)}
        assert r["fp32 exact"] <= ATT_F32, r
        return r
    rnd = G.attention_ref(qkv, heads, rounded=True, scale=scale)
    b, t, _ = qkv.shape
    err = (k - rnd).abs().view(b, t, heads, -1)
    rms = rnd.view(b, t, heads, -1).pow(2).mean(dim=(1, 3), keepdim=True).sqrt()      # per image and head
    units = err / (ulp_bf16(rnd).view(b, t, heads, -1) + ATT_ABS * rms)
    r = {"exact": rel(k, exact), "flips": float((units > 1).double().mean()), "worst": float(units.max())}
    if lse is not None:
        r["lse"] = float((got[1].double() - G.lse_ref(qkv, heads, scale)).abs().max())
    assert r["exact"] <= ATT_EXACT and r["flips"] <= ATT_FLIPS and r["worst"] <= ATT_MAX, r
    assert r.get("lse", 0.0) <= ATT_LSE, r
    return r


def _replay_recording(backbone, size, precision, batch, mode, num_channels=1):
    geoms, plans = _record(backbone, size, precision, batch, mode, num_channels)
    kinds = {k[0] for k in geoms}
    assert kinds == {"conv", "attn"}, kinds
    worst = {}
    for i, key in enumerate(geoms):
        res = check_conv(key, plans.get(key), i) if key[0] == "conv" else check_attention(key, i)
        cls = "attention" if key[0] == "attn" else "conv"
        for m, v in res.items():
            worst[f"{cls} {m}"] = max(worst.get(f"{cls} {m}", 0.0), v)
    print(f"{backbone} c{num_channels} {mode} batch {batch} {size} {precision}: {len(geoms)} distinct geometries of "
          f"{sum(geoms.values())} launches; worst " + ", ".join(f"{k} {v:.2e}" for k, v in sorted(worst.items())))


# ------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("mode", ["eval", "train"])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("size", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
@pytest.mark.parametrize("backbone", BACKBONES)
def test_every_forward_geometry(backbone, size, precision, mode):
    _replay_recording(backbone, size, precision, 2, mode)


# (backbone, batch, mode): bench.py's inference workload, and the train forwards the train benchmarks time
# (bench.py --config 4, profiles/plain_vit_train.py).  Past these batches every layer already fills the SMs with
# 256-wide tiles, so the planner's choices no longer change.
BENCH_CASES = [("vitb_rn50_384", 32, "eval"), ("vitb_rn50_384", 16, "train"), ("vitl16_384", 16, "train")]


@pytest.mark.parametrize("backbone,batch,mode", BENCH_CASES, ids=[f"{b}-b{n}-{m}" for b, n, m in BENCH_CASES])
def test_benchmark_forward_geometry(backbone, batch, mode):
    _replay_recording(backbone, (384, 384), "bf16", batch, mode)


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_normal_model_forward_geometry(mode):
    """The surface-normal model: the fused head tail with head_c = 3."""
    _replay_recording("vitb_rn50_384", (320, 480), "bf16", 2, mode, num_channels=3)
