"""The surface-normal model (num_channels=3, final ReLU) trained by the fused train step, on the GPU box.

  * NormalStepLoss (the step's sync-free loss launch sequence) against the autograd-facing normal_step_losses and
    against float64 autograd of the oracle's restatement of train_normal.py:247-265;
  * the 3-channel network backward against float64 autograd of oracle/dpt_oracle.py::forward_fp32 (shipped
    non_negative=True), in both precisions, with the golden input and the R-weighted loss of test_train_gpu.py;
  * NormalTrainStep: its gradient is autograd's, its clip + Adam is torch's, it learns, it is deterministic, its
    CUDA-graph replay is its eager step, it honours frozen tensors, it runs off the pretrained grid, and it checks its
    inputs before any launch."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

LR = 1e-6
SIZES = [(384, 384), (320, 480)]


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


# ------------------------------------------------------------------------------------------ loss sequence
def _loss_inputs(size):
    """loss_oracle.normal_loss_inputs (about 10 % of the predictions outside [0, 1]) cut to size."""
    from oracle import loss_oracle
    h, w = size
    pred, gt, mf = loss_oracle.normal_loss_inputs(0, 2, max(h, w))
    return tuple(t[:, :, :h, :w].contiguous() for t in (pred, gt, mf))


@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_normal_step_loss_matches_autograd(size):
    from omnidata_b200 import losses
    from oracle import loss_oracle
    pred, gt, mf = _loss_inputs(size)
    assert float(((pred < 0) | (pred > 1)).float().mean()) > 0.05                 # the clamp matters
    p = pred.to(dev()).requires_grad_(True)
    ref = losses.normal_step_losses(p, gt.to(dev()), mf.to(dev()))
    ref["normal_loss"].backward()
    fn = losses.NormalStepLoss()
    out, dpred = fn(pred.to(dev()), gt.to(dev()), mf.to(dev()))
    out, dpred = out.clone(), dpred.clone()
    torch.cuda.synchronize()
    assert out.shape == (3,) and dpred.shape == pred.shape
    for i, k in enumerate(("normal_loss", "l1_loss", "cos_loss")):
        assert rel(out[i], ref[k].detach()) <= 1e-6, k
    assert rel(dpred, p.grad) <= 1e-6
    # float64 autograd of the oracle: the bound of test_losses_gpu.py::test_normal_losses_backward
    p64 = pred.double().requires_grad_(True)
    tot, l1, cos = loss_oracle.normal_step(p64, gt.double(), mf.double())
    tot.backward()
    assert rel(out[0].cpu(), tot.detach()) <= 1e-6
    assert rel(dpred.cpu(), p64.grad) <= 1e-5
    out2, dpred2 = fn(pred.to(dev()), gt.to(dev()), mf.to(dev()))
    torch.cuda.synchronize()
    assert torch.equal(out2, out) and torch.equal(dpred2, dpred)


def test_normal_step_loss_is_capturable():
    """one fixed launch sequence, no synchronisation or allocation: a CUDA graph of it replays the eager bits"""
    from omnidata_b200 import losses
    pred, gt, mf = (t.to(dev()) for t in _loss_inputs((384, 384)))
    fn = losses.NormalStepLoss()
    ref = [t.clone() for t in fn(pred, gt, mf)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn(pred, gt, mf)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, dpred = fn(pred, gt, mf)
    out.zero_(); dpred.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref[0]) and torch.equal(dpred, ref[1])


# ------------------------------------------------------------------------------------------ 3-channel network backward
def _compare(g_ref, g_mine):
    """-> (global rel-L2, cosine, worst per-tensor rel-L2, its name) over all 368 tensors (dead ones must be zero)."""
    assert set(g_ref) == set(g_mine) and len(g_ref) == 368
    worst, num, den, dot, n1 = [(0.0, "")], 0.0, 0.0, 0.0, 0.0
    for k, gr in g_ref.items():
        gm, gr = g_mine[k].double(), gr.double()
        if float(gr.norm()) == 0.0:
            assert float(gm.norm()) == 0.0, k
            continue
        worst.append((float((gm - gr).norm() / gr.norm()), k))
        num += float((gm - gr).pow(2).sum()); den += float(gr.pow(2).sum())
        dot += float((gm * gr).sum()); n1 += float(gm.pow(2).sum())
    worst.sort(reverse=True)
    glob, cos = (num / den) ** 0.5, dot / (n1 * den) ** 0.5
    print(f"global rel-L2 {glob:.3e}, cosine {cos:.7f}; worst tensors: " + ", ".join(f"{k} {e:.2e}" for e, k in worst[:5]))
    return glob, cos, worst[0][0], worst[0][1]


def _oracle_grads(sd, x, R, dtype=torch.float64, autocast=False):
    from oracle import dpt_oracle
    leaves = {k: v.to(dev()).to(dtype).requires_grad_(True) for k, v in sd.items()}
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        y = dpt_oracle.forward_fp32(leaves, x.to(dev()), non_negative=True, dtype=dtype)
    grads = torch.autograd.grad((y.to(dtype) * R.to(dtype)).sum(), list(leaves.values()), allow_unused=True)
    return y.detach(), {k: (g if g is not None else torch.zeros_like(leaves[k])) for k, g in zip(leaves, grads)}


def _model_c3(sd, precision):
    from omnidata_b200.model import DPTDepthModel
    model = DPTDepthModel(backbone="vitb_rn50_384", num_channels=3)            # non_negative=True, as shipped
    model.load_state_dict(sd, strict=True)
    model = model.to(dev()).train()
    model.precision = precision
    return model


def _engine_grads(model, x, R):
    y = model(x.to(dev()))
    assert y.requires_grad and y.shape == (1, 3, 384, 384)
    (y * R).sum().backward()
    return y.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}


@pytest.fixture(scope="module")
def grads_case():
    from oracle import make_golden, weights
    sd = weights.make_state_dict(0, 3)
    x = make_golden.golden_input(1, seed=0)
    g = torch.Generator(device="cpu").manual_seed(123)
    R = torch.randn(1, 3, 384, 384, generator=g).to(dev())
    y_ref, g_ref = _oracle_grads(sd, x, R)
    return sd, x, R, y_ref, g_ref


_HEAD = ["scratch.output_conv.0.weight", "scratch.output_conv.0.bias", "scratch.output_conv.2.weight",
         "scratch.output_conv.2.bias", "scratch.output_conv.4.weight", "scratch.output_conv.4.bias"]


def _head(sd, path_1, m2=None, m4=None):
    """float64 head (dpt_depth.py:91-99) from path_1: its two ReLUs, or the given 0/1 masks in their place.
    -> (output, inner pre-activation, leaves)."""
    p = {k: sd[k].to(dev()).double().requires_grad_(True) for k in _HEAD}
    o = F.conv2d(path_1, p[_HEAD[0]], p[_HEAD[1]], padding=1)
    o = F.interpolate(o, scale_factor=2, mode="bilinear", align_corners=True)
    pre2 = F.conv2d(o, p[_HEAD[2]], p[_HEAD[3]], padding=1)
    o = pre2 * m2 if m2 is not None else F.relu(pre2)
    o = F.conv2d(o, p[_HEAD[4]], p[_HEAD[5]])
    o = o * m4 if m4 is not None else F.relu(o)
    return o, pre2.detach(), p


def _group_rel(g, g_ref, keys):
    num = sum(float((g[k].double() - g_ref[k].double()).pow(2).sum()) for k in keys)
    return (num / sum(float(g_ref[k].double().pow(2).sum()) for k in keys)) ** 0.5


def test_network_backward_3ch_fp32_mode(grads_case):
    """Output <= 1e-5, per tensor <= 5e-3 and cosine >= 0.999999 as for the depth model; global <= 1e-3, the bound of
    the depth model off the 384x384 grid (test_train_sizes_gpu.py), for the reason given there: the global error is set by
    the few ReLU threshold flips an fp32 forward makes, each of which moves the exact gradient by O(1) at one element.
    The head shows the mechanism, so its backward is also held to float64 on the branch of the ReLUs the engine's forward
    took (<= 1e-5), and a defect in a backward kernel cannot hide behind the flips."""
    from oracle import dpt_oracle
    sd, x, R, y_ref, g_ref = grads_case
    model = _model_c3(sd, "fp32")
    y, g = _engine_grads(model, x, R)
    err_y = rel(y, y_ref)
    print(f"3-channel fp32 mode: output rel-L2 {err_y:.2e}; final ReLU clamps {float((y_ref == 0).double().mean()):.2%}")
    assert err_y <= 1e-5
    glob, cos, worst, name = _compare(g_ref, g)
    assert glob <= 1e-3 and cos >= 0.999999, (glob, cos)
    assert worst <= 5e-3, (worst, name)
    hd = model._train_engine.saved["head"]
    m2 = (hd["a"][..., :32] > 0).permute(0, 3, 1, 2).double()
    m4 = (hd["out"] > 0).double()
    taps = {}
    with torch.no_grad():
        dpt_oracle.forward_fp32({k: v.to(dev()).double() for k, v in sd.items()}, x.to(dev()).double(), taps=taps,
                                dtype=torch.float64)
    y64, pre2, _ = _head(sd, taps["path_1"])
    flips2, flips4 = int(((pre2 > 0).double() != m2).sum()), int(((y64 > 0).double() != m4).sum())
    o, _, p = _head(sd, taps["path_1"], m2, m4)
    g_msk = dict(zip(_HEAD, torch.autograd.grad((o * R.double()).sum(), [p[k] for k in _HEAD])))
    e_nat, e_msk = _group_rel(g, g_ref, _HEAD), _group_rel(g, g_msk, _HEAD)
    rest = [k for k in g_ref if k not in _HEAD]
    print(f"  head: rel-L2 {e_nat:.2e} against float64, {e_msk:.2e} with the engine's ReLU masks; flipped elements: "
          f"{flips2} of {m2.numel()} (inner ReLU), {flips4} of {m4.numel()} (final ReLU); the other 362 tensors "
          f"{_group_rel(g, g_ref, rest):.2e}")
    assert e_msk <= 1e-5


def test_network_backward_3ch_bf16_mode(grads_case):
    sd, x, R, y_ref, g_ref = grads_case
    y, g = _engine_grads(_model_c3(sd, "bf16"), x, R)
    mine, *_ = _compare(g_ref, g)
    _, g_ac = _oracle_grads(sd, x, R, torch.float32, autocast=True)   # stock torch.autocast(bfloat16) training
    stock, *_ = _compare(g_ref, g_ac)
    print(f"bf16 engine {mine:.3e} vs stock autocast {stock:.3e} (ratio {mine / stock:.2f})")
    assert mine <= 1.6 * stock, (mine, stock)
    _, g2 = _engine_grads(_model_c3(sd, "bf16"), x, R)
    assert all(torch.equal(g[k], g2[k]) for k in g)


# ------------------------------------------------------------------------------------------ train step
def _batch(size=(384, 384), seed=9):
    h, w = size
    g = torch.Generator(device="cpu").manual_seed(seed)
    rgb = (torch.rand(2, 3, h, w, generator=g) * 2 - 1).to(dev())
    gt = torch.rand(2, 3, h, w, generator=g).to(dev())
    mask = (torch.rand(2, 1, h, w, generator=g) > 0.1).float().to(dev())
    return rgb, gt, mask


def _model(sd=None, trainable=lambda n: True):
    from omnidata_b200 import synthetic
    from omnidata_b200.model import DPTDepthModel
    model = DPTDepthModel(num_channels=3)
    model.load_state_dict(synthetic.make_state_dict(0, 3) if sd is None else sd, strict=True)
    model = model.to(dev()).train()
    for n, p in model.named_parameters():
        p.requires_grad_(trainable(n))
    return model


def _step(size=(384, 384), graph=False, clip=10.0, trainable=lambda n: True, sd=None, lr=LR):
    from omnidata_b200.train import NormalTrainStep
    step = NormalTrainStep(_model(sd, trainable), lr=lr, clip=clip, precision="bf16", input_size=size)
    step.use_cuda_graph = graph
    return step


def test_step_gradient_is_the_autograd_gradient():
    from omnidata_b200 import losses
    from oracle import weights
    sd = weights.make_state_dict(0, 3)
    rgb, gt, mask = _batch()
    # autograd: model(x) -> normal_step_losses -> backward (the same kernels with w_l1 = 10, w_cos = 1)
    ref = _model(sd)
    out = ref(rgb)
    lv = losses.normal_step_losses(out, gt, mask)
    lv["normal_loss"].backward()
    g_ref = {n: p.grad.detach().clone() for n, p in ref.named_parameters()}
    step = _step(clip=None, sd=sd)
    res = step.step(rgb, gt, mask)
    torch.cuda.synchronize()
    assert res.shape == (4,) and float(res[3]) == 0.0                  # no clip: no norm
    assert torch.equal(res[0], lv["normal_loss"].detach()) and torch.equal(res[1], lv["l1_loss"].detach())
    assert torch.equal(res[2], lv["cos_loss"].detach())
    eng = step.engine
    for n, gr in g_ref.items():
        assert torch.equal(eng.G[n], gr), n
    # clip 10 + Adam against torch.nn.utils.clip_grad_norm_ + torch.optim.Adam applied to those gradients
    # (tolerances of test_optim_gpu.py: torch's fp32 norm carries ~1e-5, the update one rounding of p)
    step = _step(clip=10.0, sd=sd, lr=1e-5)
    res = step.step(rgb, gt, mask)
    ps = {n: torch.nn.Parameter(v.to(dev()).clone()) for n, v in sd.items()}
    for n, p in ps.items():
        p.grad = g_ref[n].clone()
    ref_norm = torch.nn.utils.clip_grad_norm_(list(ps.values()), 10.0)
    adam = torch.optim.Adam(list(ps.values()), lr=1e-5)
    adam.step()
    torch.cuda.synchronize()
    exact = float(torch.cat([g.reshape(-1) for g in g_ref.values()]).double().norm())
    print(f"gradient norm {exact:.4e} (clip 10): step {float(res[3]):.6e}, torch {float(ref_norm):.6e}")
    assert abs(float(res[3]) - exact) <= 1e-6 * exact
    for n, p in ps.items():
        off, k = eng.G[n].storage_offset(), p.numel()
        st = adam.state[p]
        m, v = step.opt.exp_avg[off:off + k].view_as(p), step.opt.exp_avg_sq[off:off + k].view_as(p)
        assert torch.allclose(m, st["exp_avg"], rtol=1e-4, atol=1e-4 * float(st["exp_avg"].abs().max())), n
        assert torch.allclose(v, st["exp_avg_sq"], rtol=2e-4, atol=1e-20), n
        err = (step.engine.P[n] - p.detach()).abs()
        assert bool((err <= torch.clamp(p.detach().abs() * 2.0 ** -23, min=5e-7)).all()), n


def test_train_step_learns_and_is_deterministic():
    rgb, gt, mask = _batch()
    runs = []
    for graph in (False, False, True):
        step = _step(graph=graph)
        w0 = step.engine.flat.clone()
        hist = [step.step(rgb, gt, mask).cpu() for _ in range(3)]
        torch.cuda.synchronize()
        print("losses / norms:", [[round(float(v), 6) for v in h] for h in hist])
        assert all(torch.isfinite(h).all() for h in hist) and torch.isfinite(step.engine.flat).all()
        assert float(hist[-1][0]) < float(hist[0][0])                   # the loss goes down on the fixed batch
        assert float((step.engine.flat - w0).abs().max()) > 0 and float(hist[0][3]) > 0
        assert step.opt.step_count == 3 and step.global_step == 3
        runs.append((hist, step.engine.flat.clone(), step.opt.exp_avg.clone(), step.opt.exp_avg_sq.clone()))
    # a second eager run, then the three steps replayed as one CUDA graph (its warm-up step undone): the same bits
    for hist, *state in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(hist, runs[0][0]))
        assert all(torch.equal(a, b) for a, b in zip(state, runs[0][1:]))
    assert len(step._graphs) == 1
    # new inputs through the captured step's static copies == an eager step from the same state
    ref = _step()
    ref.engine.flat.copy_(step.engine.flat); ref.opt.exp_avg.copy_(step.opt.exp_avg)
    ref.opt.exp_avg_sq.copy_(step.opt.exp_avg_sq)
    ref.opt.step_count = 3
    rgb2, gt2, mask2 = _batch(seed=10)
    a = [step.step(rgb2, gt2, mask2).cpu(), step.step(rgb, gt, mask).cpu()]
    b = [ref.step(rgb2, gt2, mask2).cpu(), ref.step(rgb, gt, mask).cpu()]
    torch.cuda.synchronize()
    assert len(step._graphs) == 1 and step.global_step == 5 and step.opt.step_count == 5
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and torch.equal(step.engine.flat, ref.engine.flat)
    assert torch.equal(step.opt.exp_avg, ref.opt.exp_avg) and torch.equal(step.opt.exp_avg_sq, ref.opt.exp_avg_sq)


def test_train_step_with_a_frozen_encoder():
    decoder = lambda n: n.startswith("scratch.")                        # noqa: E731
    rgb, gt, mask = _batch()
    full, part = _step(clip=None), _step(clip=None, trainable=decoder)
    full.step(rgb, gt, mask)
    part.step(rgb, gt, mask)
    torch.cuda.synchronize()
    for n in part.engine.param_names:
        if decoder(n):
            assert torch.equal(part.engine.G[n], full.engine.G[n]), n
    assert [t for *_, t in part.buckets] == ["decoder"]
    runs = []
    for graph in (False, True):
        step = _step(graph=graph, trainable=decoder)
        eng = step.engine
        w0 = eng.flat.clone()
        frozen = torch.ones_like(eng.flat, dtype=torch.bool)
        for s, e in step.opt.segments:
            frozen[s:e] = False
        hist = [step.step(rgb, gt, mask).cpu() for _ in range(3)]
        torch.cuda.synchronize()
        assert torch.equal(eng.flat[frozen], w0[frozen])
        assert not step.opt.exp_avg[frozen].any() and not step.opt.exp_avg_sq[frozen].any()
        assert all(torch.isfinite(h).all() for h in hist) and float(hist[-1][0]) < float(hist[0][0])
        runs.append((hist, eng.flat.clone(), step.opt.exp_avg.clone()))
        step._flag_params[0].requires_grad_(not step._flag_params[0].requires_grad)
        with pytest.raises(ValueError):
            step.step(rgb, gt, mask)
    (h0, f0, m0), (h1, f1, m1) = runs
    assert all(torch.equal(a, b) for a, b in zip(h0, h1)) and torch.equal(f0, f1) and torch.equal(m0, m1)


def test_train_step_at_320x480_learns_and_is_deterministic():
    size = SIZES[1]
    rgb, gt, mask = _batch(size)
    runs = []
    for graph in (False, False, True):
        step = _step(size, graph)
        hist = [step.step(rgb, gt, mask).cpu() for _ in range(3)]
        torch.cuda.synchronize()
        assert all(torch.isfinite(h).all() for h in hist) and torch.isfinite(step.engine.flat).all()
        assert float(hist[-1][0]) < float(hist[0][0]) and float(hist[0][3]) > 0
        runs.append((hist, step.engine.flat.clone()))
    for hist, flat in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(hist, runs[0][0])) and torch.equal(flat, runs[0][1])


def test_step_inputs_are_validated_before_any_launch():
    from omnidata_b200 import _capi
    size = SIZES[1]
    rgb, gt, mask = _batch(size)
    sq = _batch((384, 384))
    step = _step(size)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    bad = [sq, (rgb, sq[1], mask), (rgb, gt, sq[2]),                    # another input size
           (rgb, gt[:, :1], mask), (rgb, gt, mask.expand(-1, 3, -1, -1)),  # depth-shaped target, repeated mask
           (rgb[:1], gt, mask), (rgb, gt[:1], mask), (rgb, gt, mask[:1]),  # batch mismatch
           (rgb[:, :1], gt, mask)]
    for graph in (False, True):
        step.use_cuda_graph = graph
        for args in bad:
            with pytest.raises(ValueError):
                step.step(*args)
    assert _capi.launch_count() == n0
    assert step.global_step == 0 and not step._graphs
