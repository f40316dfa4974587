"""Backward and train step of the plain-ViT DPTs (DPT-Large `vitl16_384`, plain ViT-B `vitb16_384`) on the GPU.

Checkers: float64 torch.autograd of the plain-ViT oracle (oracle/plain_vit_oracle.py::forward_fp32, pinned to the
UNMODIFIED reference class's golden vectors in tests/test_plain_vit_oracle_cpu.py) with the same seeded weights; torch
permutations and float64 einsums for the two new backward operations (patch-embedding input gradient, ConvTranspose
dgrad / wgrad); torch.optim.Adam + clip_grad_norm_ for the optimizer step.  The bounds are the DPT-Hybrid's
(tests/test_train_sizes_gpu.py, tests/test_bwd_gemm_gpu.py, tests/test_optim_gpu.py)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
PLAIN = ["vitl16_384", "vitb16_384"]
REL_WGRAD = {torch.bfloat16: 1e-4, torch.float32: 4.5e-7}
REL_DGRAD = {torch.bfloat16: 4e-3, torch.float32: 4e-7}
DEAD = ("pretrained.model.norm.", "pretrained.model.head.", "scratch.refinenet4.resConfUnit1.")


def dev():
    return torch.device("cuda:0")


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield


def _sd(backbone, c=1):
    from omnidata_b200.model import state_dict_spec
    from omnidata_b200.synthetic import make_state_dict
    return make_state_dict(0, c, spec=state_dict_spec(c, backbone=backbone))


def _model(backbone, precision, sd=None, c=1):
    from omnidata_b200.model import DPTDepthModel
    m = DPTDepthModel(backbone=backbone, num_channels=c)
    m.load_state_dict(_sd(backbone, c) if sd is None else sd, strict=True)
    m = m.to(dev()).train()
    m.precision = precision
    return m


def _inputs(h, w, batch=1, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.rand(batch, 3, h, w, generator=g) * 2 - 1
    R = torch.randn(batch, h, w, generator=torch.Generator(device="cpu").manual_seed(123 + seed)).to(dev())
    return x, R


def _engine_grads(model, x, R, need_x_grad=False):
    for p in model.parameters():
        p.grad = None
    xi = x.to(dev()).clone().requires_grad_(need_x_grad)
    y = model(xi)
    assert y.requires_grad
    (y * R).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}
    return y.detach(), grads, (xi.grad.detach().clone() if need_x_grad else None)


def _reference_grads(sd, x, R, dtype=torch.float64, autocast=False, want_x=False):
    from oracle import plain_vit_oracle
    leaves = {k: v.to(dev()).to(dtype).requires_grad_(True) for k, v in sd.items()}
    xi = x.to(dev()).to(dtype).requires_grad_(want_x)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        y = plain_vit_oracle.forward_fp32(leaves, xi, dtype=dtype)
    ins = list(leaves.values()) + ([xi] if want_x else [])
    grads = torch.autograd.grad((y.to(dtype) * R.to(dtype)).sum(), ins, allow_unused=True)
    g = {k: (gg if gg is not None else torch.zeros_like(leaves[k])) for k, gg in zip(leaves, grads)}
    return y.detach(), g, (grads[-1] if want_x else None)


def _compare(g_ref, g_mine, per_tensor_tol, global_tol, min_cos):
    worst, num, dot, n1, n2 = [], 0.0, 0.0, 0.0, 0.0
    assert set(g_ref) == set(g_mine)
    for k, gr in g_ref.items():
        gm, gr = g_mine[k].double(), gr.double()
        if float(gr.norm()) == 0.0:            # dead parameters (timm classifier head / final norm, refinenet4.resConfUnit1)
            assert float(gm.norm()) == 0.0, k
            continue
        worst.append((float((gm - gr).norm() / gr.norm()), k))
        num += float((gm - gr).pow(2).sum())
        dot += float((gm * gr).sum()); n1 += float(gm.pow(2).sum()); n2 += float(gr.pow(2).sum())
    worst.sort(reverse=True)
    glob, cos = (num / n2) ** 0.5, dot / (n1 * n2) ** 0.5
    print(f"global rel-L2 {glob:.3e}, cosine {cos:.7f}; worst tensors: " + ", ".join(f"{k} {e:.2e}" for e, k in worst[:6]))
    assert glob <= global_tol and cos >= min_cos, (glob, cos)
    assert worst[0][0] <= per_tensor_tol, worst[:6]
    return glob


# ------------------------------------------------------------------------------------------ the two new operations
@pytest.mark.parametrize("h,w", [(384, 384), (320, 480)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_patch_input_grad_is_the_permutation(dtype, h, w):
    from omnidata_b200 import bwd
    b, gh, gw = 2, h // 16, w // 16
    dcols = torch.randn(b * gh * gw, 768, generator=torch.Generator(device="cuda").manual_seed(h + w), device=dev()).to(dtype)
    dx = torch.full((b, 3, h, w), float("nan"), device=dev())
    bwd.patch_input_grad(dcols, dx)
    ref = dcols.float().view(b, gh, gw, 3, 16, 16).permute(0, 3, 1, 4, 2, 5).reshape(b, 3, h, w)
    torch.cuda.synchronize()
    assert torch.equal(dx, ref)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("backbone", PLAIN)
def test_conv_transpose_bwd_matches_float64(backbone, precision):
    """The input, weight and bias gradients of layer_1's ConvTranspose 4/4 and layer_2's 2/2 at the step's shapes (batch
    2, 384x384 and 320x480), against float64 on the same operands."""
    from omnidata_b200.train import TrainEngine
    eng = TrainEngine(_model(backbone, precision), precision)
    eng.pack()
    eng._plan = eng.plan_for(None, False)
    adt = eng.adt
    for gh, gw in ((24, 24), (20, 30)):
        for n, k in ((1, 4), (2, 2)):
            c, cp = eng.rn_in[n - 1], eng.rn_pad[n - 1]
            g = torch.Generator(device="cuda").manual_seed(n * 100 + gh)
            u = torch.randn(2, gh, gw, cp, generator=g, device=dev())
            dout = torch.randn(2, k * gh, k * gw, cp, generator=g, device=dev())
            u[..., c:] = 0                                           # padded channels carry zeros, as in the forward
            dout[..., c:] = 0
            u, dout = u.to(adt), dout.to(adt)
            du = eng._conv_transpose_bwd(n, k, dout, u)
            torch.cuda.synchronize()
            Wf = eng.W[f"pp{n}t"][0].double().view(cp, k, k, cp)     # [in][ky][kx][out]
            d6 = dout.double().view(2, gh, k, gw, k, cp)
            du_ref = torch.einsum("byYxXo,iYXo->byxi", d6, Wf)
            gw_ref = torch.einsum("byxi,byYxXo->iYXo", u.double(), d6)
            e_d, e_w = rel(du, du_ref), rel(eng.gp_layer[f"pp{n}t"], gw_ref.reshape(cp, -1))
            e_b = rel(eng.G[f"pretrained.act_postprocess{n}.4.bias"], d6.sum(dim=(0, 1, 2, 3, 4))[:c])
            print(f"{backbone} {precision} layer_{n} {gh}x{gw}: dgrad {e_d:.2e}, wgrad {e_w:.2e}, bias {e_b:.2e}")
            assert e_d <= REL_DGRAD[adt] and e_w <= REL_WGRAD[adt] and e_b <= 1e-6
            assert not bool(du[..., c:].any())                       # padded input channels get no gradient


# ------------------------------------------------------------------------------------------ whole network
@pytest.mark.parametrize("backbone", PLAIN)
def test_network_backward_fp32_mode(backbone):
    """fp32 mode against float64 autograd of the oracle at 320x480 (off the 24 x 24 grid: the pos_embed resize adjoint
    runs), with the DPT-Hybrid's bounds at that size: output <= 1e-5, global <= 1e-3, every tensor <= 5e-3, cosine
    >= 0.999999; the head's backward with the engine's ReLU masks put into the float64 head <= 1e-5; x.grad <= 5e-3."""
    from oracle import plain_vit_oracle
    h, w = 320, 480
    sd = _sd(backbone)
    x, R = _inputs(h, w)
    model = _model(backbone, "fp32", sd)
    y, g, dx = _engine_grads(model, x, R, need_x_grad=True)
    y_ref, g_ref, dx_ref = _reference_grads(sd, x, R, want_x=True)
    err_y, err_x = rel(y, y_ref), rel(dx, dx_ref)
    print(f"{backbone} fp32 mode {h}x{w}: output {err_y:.2e}, x.grad {err_x:.2e}")
    assert err_y <= 1e-5 and err_x <= 5e-3
    _compare(g_ref, g, per_tensor_tol=5e-3, global_tol=1e-3, min_cos=0.999999)
    heads = ["scratch.output_conv.0.weight", "scratch.output_conv.0.bias", "scratch.output_conv.2.weight",
             "scratch.output_conv.2.bias", "scratch.output_conv.4.weight", "scratch.output_conv.4.bias"]
    hd = model._train_engine.saved["head"]
    m2 = (hd["a"][..., :32] > 0).permute(0, 3, 1, 2).double()
    m4 = (hd["out"] > 0).double()
    taps = {}
    with torch.no_grad():
        plain_vit_oracle.forward_fp32({k: v.to(dev()).double() for k, v in sd.items()}, x.to(dev()).double(), taps=taps,
                                dtype=torch.float64)
    p = {k: sd[k].to(dev()).double().requires_grad_(True) for k in heads}
    o = F.conv2d(taps["path_1"], p[heads[0]], p[heads[1]], padding=1)
    o = F.interpolate(o, scale_factor=2, mode="bilinear", align_corners=True)
    o = F.conv2d(o, p[heads[2]], p[heads[3]], padding=1) * m2
    o = F.conv2d(o, p[heads[4]], p[heads[5]]) * m4
    g_head = dict(zip(heads, torch.autograd.grad((o.squeeze(1) * R.double()).sum(), [p[k] for k in heads])))
    num = sum(float((g[k].double() - g_head[k]).pow(2).sum()) for k in heads)
    e_msk = (num / sum(float(g_head[k].pow(2).sum()) for k in heads)) ** 0.5
    print(f"  head with the engine's ReLU masks: {e_msk:.2e}")
    assert e_msk <= 1e-5


@pytest.mark.parametrize("backbone", PLAIN)
def test_network_backward_bf16_mode(backbone):
    """bf16: global error <= 1.6 x stock autocast measured live; bit-reproducible; batch-independent and eval() ==
    train() bit for bit for x.grad."""
    h, w = 384, 384
    sd = _sd(backbone)
    x, R = _inputs(h, w)
    model = _model(backbone, "bf16", sd)
    _, g, dx1 = _engine_grads(model, x, R, need_x_grad=True)
    _, g_ref, _ = _reference_grads(sd, x, R)
    mine = _compare(g_ref, g, per_tensor_tol=10.0, global_tol=10.0, min_cos=0.0)
    _, g_ac, _ = _reference_grads(sd, x, R, torch.float32, autocast=True)
    stock = _compare(g_ref, g_ac, per_tensor_tol=10.0, global_tol=10.0, min_cos=0.0)
    print(f"{backbone} bf16 mode: global rel-L2 {mine:.3e}; stock autocast(bf16) autograd {stock:.3e}")
    assert mine <= 1.6 * stock, (mine, stock)
    _, g2, _ = _engine_grads(model, x, R)
    assert all(torch.equal(g[k], g2[k]) for k in g)
    x2, R2 = _inputs(h, w, batch=2, seed=5)
    x2[0], R2[0] = x[0], R[0]
    _, _, dx2 = _engine_grads(model, x2, R2, need_x_grad=True)
    assert torch.equal(dx1[0], dx2[0])
    model.eval()
    _, _, dx_eval = _engine_grads(model, x, R, need_x_grad=True)
    assert torch.equal(dx_eval, dx1)


@pytest.mark.parametrize("backbone", PLAIN)
def test_frozen_sets(backbone):
    """The encoder frozen, and everything frozen with x.grad wanted: every returned gradient equals the full backward's
    bit for bit, frozen p.grad stays None, and the frozen slices of the flat gradient are never written."""
    x, R = _inputs(384, 384)
    model = _model(backbone, "bf16")
    _, g_full, dx_full = _engine_grads(model, x, R, need_x_grad=True)
    eng = model._train_engine
    for frozen, want_x in ((lambda n: n.startswith("pretrained."), False), (lambda n: True, True)):
        for n, p in model.named_parameters():
            p.requires_grad_(not frozen(n))
        eng.flat_grad.fill_(float("nan"))
        if want_x:
            xi = x.to(dev()).clone().requires_grad_(True)
            (model(xi) * R).sum().backward()
            assert torch.equal(xi.grad, dx_full)
        else:
            for p in model.parameters():
                p.grad = None
            _engine_grads(model, x, R)
        torch.cuda.synchronize()
        for n, p in model.named_parameters():
            if frozen(n):
                assert p.grad is None, n
                assert bool(torch.isnan(eng.G[n]).all()), n
            elif not n.startswith(DEAD):                             # no backward writes a dead tensor's zero slice
                assert torch.equal(p.grad, g_full[n]), n
        for p in model.parameters():
            p.requires_grad_(True)
            p.grad = None


def test_depth_train_step_vitl():
    """DepthTrainStep on DPT-Large: clip + Adam after one step match clip_grad_norm_ + torch.optim.Adam; three steps at
    lr 1e-6 lower the loss; eager and CUDA-graph replay are bit-identical; at 320x480 it learns and is deterministic."""
    import numpy as np
    from omnidata_b200.train import DepthTrainStep
    LR = 1e-6
    for h, w in ((384, 384), (320, 480)):
        g = torch.Generator(device="cpu").manual_seed(9)
        rgb = (torch.rand(2, 3, h, w, generator=g) * 2 - 1).to(dev())
        gt = torch.rand(2, 1, h, w, generator=g).to(dev())
        mask = (torch.rand(2, 1, h, w, generator=g) > 0.1).float().to(dev())
        runs = []
        for graph in (False, True, False):
            step = DepthTrainStep(_model("vitl16_384", "bf16"), lr=LR, clip=10.0, precision="bf16", input_size=(h, w))
            step.use_cuda_graph = graph
            w0 = step.engine.flat.clone()
            np.random.seed(11)
            hist = []
            for i in range(3):
                hist.append(step.step(rgb, gt, mask, full_mix=True).cpu())
                if i == 0 and not graph and not runs:
                    torch.cuda.synchronize()
                    gr = step.engine.flat_grad.cpu()
                    ref_p = torch.nn.Parameter(w0.cpu())
                    ref_p.grad = gr.clone()
                    exact = float(gr.double().norm())
                    print(f"vitl16_384 {h}x{w}: gradient norm {float(hist[0][4]):.6e} (float64 {exact:.6e})")
                    assert abs(float(hist[0][4]) - exact) <= 1e-6 * exact
                    # clip_grad_norm_'s arithmetic with the float64 norm: torch's own fp32 norm over these 343M values
                    # on the CPU put the clipped gradient 1.8 % off (measured)
                    ref_p.grad.mul_(min(1.0, 10.0 / (exact + 1e-6)))
                    ref = torch.optim.Adam([ref_p], lr=LR)
                    ref.step()
                    st = ref.state[ref_p]
                    rt = 1e-4
                    assert torch.allclose(step.opt.exp_avg.cpu(), st["exp_avg"], rtol=rt,
                                          atol=rt * float(st["exp_avg"].abs().max()))
                    assert torch.allclose(step.opt.exp_avg_sq.cpu(), st["exp_avg_sq"], rtol=2 * rt, atol=1e-20)
                    assert float((step.engine.flat.cpu() - ref_p.detach()).abs().max()) <= 5e-7
            torch.cuda.synchronize()
            assert all(torch.isfinite(t).all() for t in hist)
            assert float(hist[-1][0]) < float(hist[0][0])
            runs.append((hist, step.engine.flat.clone()))
            del step
        for hist, flat in runs[1:]:
            assert all(torch.equal(a, b) for a, b in zip(hist, runs[0][0])) and torch.equal(flat, runs[0][1])


def test_normal_train_step_plain_vit():
    """NormalTrainStep on a num_channels=3 plain ViT-B DPT: three steps learn, finite and deterministic."""
    from omnidata_b200.train import NormalTrainStep
    g = torch.Generator(device="cpu").manual_seed(4)
    rgb = (torch.rand(2, 3, 384, 384, generator=g) * 2 - 1).to(dev())
    gt = F.normalize(torch.randn(2, 3, 384, 384, generator=g), dim=1).mul(0.5).add(0.5).to(dev())
    mask = (torch.rand(2, 1, 384, 384, generator=g) > 0.1).float().to(dev())
    runs = []
    for _ in range(2):
        step = NormalTrainStep(_model("vitb16_384", "bf16", c=3), lr=1e-6)
        hist = [step.step(rgb, gt, mask).cpu() for _ in range(3)]
        torch.cuda.synchronize()
        assert all(torch.isfinite(t).all() for t in hist) and float(hist[-1][0]) < float(hist[0][0])
        runs.append((hist, step.engine.flat.clone()))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0])) and torch.equal(runs[0][1], runs[1][1])
    assert math.isfinite(float(runs[0][0][0][0]))
