"""requires_grad in the DPT-Hybrid backward and train step: a partly or fully frozen model forms only the gradients
autograd or the train step needs, and those are the bits of the full backward.

Setup as test_input_grad_gpu.py: seeded weights, the golden input (384 x 384) or a seeded image (320 x 480), and the
R-weighted loss sum(model(x) * R)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BB = "pretrained.model.patch_embed.backbone."
PATTERNS = {
    "encoder": (lambda n: n.startswith("scratch."), False),
    "top_blocks": (lambda n: n.startswith(("scratch.",) + tuple(f"pretrained.model.blocks.{i}." for i in (8, 9, 10, 11))),
                   False),
    "resnet": (lambda n: not n.startswith(BB), False),
    "all_frozen_dx": (lambda n: False, True),
}


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def sd():
    from oracle import weights
    return weights.make_state_dict(0, 1)


def _inputs(size):
    from oracle import make_golden
    g = torch.Generator(device="cpu").manual_seed(123)
    if size == (384, 384):
        x = make_golden.golden_input(1, seed=0)
    else:
        x = torch.rand(1, 3, *size, generator=g) * 2 - 1
    R = torch.randn(1, *size, generator=g).to(dev())
    return x.to(dev()), R


def _model(sd, precision):
    from omnidata_b200.model import DPTDepthModel
    m = DPTDepthModel(backbone="vitb_rn50_384")
    m.load_state_dict(sd, strict=True)
    m = m.to(dev()).train()
    m.precision = precision
    return m


def _grads(model, x, R, trainable, want_dx):
    """-> (x.grad or None, {name: p.grad or None}) of sum(model(x) * R) with requires_grad = trainable(name)."""
    for n, p in model.named_parameters():
        p.requires_grad_(trainable(n))
        p.grad = None
    xi = x.clone().requires_grad_(want_dx)
    (model(xi) * R).sum().backward()
    return (xi.grad.clone() if want_dx else None), {n: (None if p.grad is None else p.grad.clone())
                                                    for n, p in model.named_parameters()}


@pytest.fixture(scope="module", params=[("bf16", (384, 384)), ("fp32", (384, 384)), ("bf16", (320, 480)),
                                        ("fp32", (320, 480))], ids=lambda p: f"{p[0]}-{p[1][0]}x{p[1][1]}")
def case(request, sd):
    precision, size = request.param
    x, R = _inputs(size)
    model = _model(sd, precision)
    full = _grads(model, x, R, lambda n: True, True)
    return model, x, R, full


@pytest.mark.parametrize("pattern", list(PATTERNS))
def test_frozen_backward_is_the_full_backwards_bits(case, pattern):
    model, x, R, (dx_full, g_full) = case
    trainable, want_dx = PATTERNS[pattern]
    if pattern == "all_frozen_dx":
        model.eval()
    try:
        dx, g = _grads(model, x, R, trainable, want_dx)
    finally:
        model.train()
    for n, gr in g.items():
        if trainable(n):
            assert gr is not None and torch.equal(gr, g_full[n]), n
        else:
            assert gr is None, n
    assert (dx is None) == (not want_dx)
    if want_dx:
        assert torch.equal(dx, dx_full)


def _wgrad_count(eng, trainable):
    """conv_wgrad calls of a backward: one per trainable GEMM weight (engine layer table and the stem), two per
    trainable readout projection (its token and cls halves)."""
    gemm = {L.weight for L in eng.layers} | {BB + "stem.conv.weight"}
    ro = {f"pretrained.act_postprocess{n}.0.project.0.weight" for n in (3, 4)}
    return sum(1 for n in trainable if n in gemm) + 2 * sum(1 for n in trainable if n in ro)


@pytest.mark.parametrize("pattern", list(PATTERNS))
def test_frozen_slices_are_not_written(sd, pattern, monkeypatch):
    from omnidata_b200 import _capi, bwd
    from omnidata_b200.train import TrainEngine
    x, R = _inputs((384, 384))
    model = _model(sd, "bf16")
    eng = TrainEngine(model)
    pred, want_dx = PATTERNS[pattern]
    trainable = frozenset(n for n in eng.param_names if pred(n))
    calls = []
    real = bwd.conv_wgrad
    monkeypatch.setattr(bwd, "conv_wgrad", lambda *a, **k: (calls.append(1), real(*a, **k)))
    dout = R.view(1, 1, *R.shape[1:]).contiguous()
    dx = torch.empty_like(x) if want_dx else None
    eng.forward(x)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    eng.backward(dout, dx=dx)
    torch.cuda.synchronize()
    n_full = _capi.launch_count() - n0
    calls.clear()
    eng.forward(x, trainable=trainable)
    eng.flat_grad.fill_(float("nan"))
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    eng.backward(dout, dx=dx, trainable=trainable)
    torch.cuda.synchronize()
    n_frozen = _capi.launch_count() - n0
    print(f"{pattern}: backward launches {n_frozen} (full backward {n_full}); conv_wgrad calls {len(calls)}")
    for n in eng.param_names:
        if n not in trainable:
            assert torch.isnan(eng.G[n]).all(), n
    assert len(calls) == _wgrad_count(eng, trainable)
    assert n_frozen < n_full


def test_frozen_layer_operands_are_packed_only_when_they_change(sd, monkeypatch):
    from omnidata_b200 import bwd
    from oracle import weights
    x, R = _inputs((384, 384))
    model = _model(sd, "bf16").eval().requires_grad_(False)
    xi = x.clone().requires_grad_(True)
    (model(xi) * R).sum().backward()
    eng = model._train_engine
    runs = []
    real = bwd.PackTable.run
    monkeypatch.setattr(bwd.PackTable, "run", lambda self, *a, **k: (runs.append(1), real(self, *a, **k)))
    derived = [eng.pk["gemm"]["stem"], eng.pk["vec"]["scratch.output_conv.2.bias"], eng.pk["gemm"]["ro3.full"],
               eng.bufs["w.ro4.tokT"]]
    versions = [t._version for t in derived]
    xi = x.clone().requires_grad_(True)
    out = model(xi)
    (out * R).sum().backward()
    assert runs == [] and [t._version for t in derived] == versions      # no packing launch, no torch-op packing
    # a changed frozen weight is re-packed by the next forward: output and x.grad are a fresh model's bits
    sd2 = weights.make_state_dict(1, 1)
    for change in ("load_state_dict", "copy_"):
        if change == "load_state_dict":
            model.load_state_dict(sd2, strict=True)
        else:
            w = dict(model.named_parameters())["scratch.layer1_rn.weight"]
            with torch.no_grad():
                w.copy_(sd["scratch.layer1_rn.weight"].to(dev()))
            sd2 = {k: (sd[k] if k == "scratch.layer1_rn.weight" else v) for k, v in sd2.items()}
        xi = x.clone().requires_grad_(True)
        out = model(xi)
        (out * R).sum().backward()
        assert runs, change
        runs.clear()
        fresh = _model(sd2, "bf16").eval().requires_grad_(False)
        xf = x.clone().requires_grad_(True)
        out_f = fresh(xf)
        (out_f * R).sum().backward()
        assert torch.equal(out, out_f) and torch.equal(xi.grad, xf.grad), change


# ------------------------------------------------------------------------------------------ segment clip / Adam
SEGMENTS = [(0, 4096), (8192, 100000), (131072, 500004), (600000, 600003)]


@pytest.mark.parametrize("max_norm", [10.0, 0.5, None])
def test_segment_clip_and_adam_match_torch(lib_built, max_norm):
    from omnidata_b200.optim import FlatAdam
    n = 1000003
    g = torch.Generator().manual_seed(5)
    p0 = torch.randn(n, generator=g)
    ref_ps = [torch.nn.Parameter(p0[s:e].clone()) for s, e in SEGMENTS]
    ref = torch.optim.Adam(ref_ps, lr=1e-5)
    mine = p0.clone().cuda()
    opt = FlatAdam(mine, lr=1e-5, segments=SEGMENTS)
    outside = torch.ones(n, dtype=torch.bool)
    for s, e in SEGMENTS:
        outside[s:e] = False
    outside = outside.cuda()
    for step in range(4):
        grad = torch.randn(n, generator=g) * (3.0 if step % 2 else 0.01)
        for rp, (s, e) in zip(ref_ps, SEGMENTS):
            rp.grad = grad[s:e].clone()
        if max_norm is not None:
            torch.nn.utils.clip_grad_norm_(ref_ps, max_norm)
        ref.step()
        gd = grad.cuda()
        gd[outside] = float("nan")                                   # never read
        norm = opt.step(gd, max_norm=max_norm)
        torch.cuda.synchronize()
        if max_norm is not None:
            exact = float(torch.cat([grad[s:e] for s, e in SEGMENTS]).double().norm())
            assert abs(float(norm) - exact) <= 1e-6 * exact
        rt = 1e-5 if max_norm is None else 1e-4
        for rp, (s, e) in zip(ref_ps, SEGMENTS):
            st = ref.state[rp]
            assert torch.allclose(opt.exp_avg[s:e].cpu(), st["exp_avg"], rtol=rt, atol=rt * float(st["exp_avg"].abs().max()))
            assert torch.allclose(opt.exp_avg_sq[s:e].cpu(), st["exp_avg_sq"], rtol=2 * rt, atol=1e-20)
            assert float((mine[s:e].cpu() - rp.detach()).abs().max()) <= 5e-7 * (step + 1)
        assert torch.equal(mine[outside], p0.cuda()[outside])        # bit-unchanged outside the segments
        assert not opt.exp_avg[outside].any() and not opt.exp_avg_sq[outside].any()


def test_one_segment_is_the_whole_buffer_step(lib_built):
    from omnidata_b200.optim import FlatAdam
    n = 123147 * 10 + 1
    g = torch.Generator().manual_seed(3)
    p0 = torch.randn(n, generator=g).cuda()
    a, b = p0.clone(), p0.clone()
    oa, ob = FlatAdam(a, lr=1e-4), FlatAdam(b, lr=1e-4, segments=[(0, n)])
    for _ in range(3):
        grad = torch.randn(n, generator=g).cuda() * 2
        na, nb = oa.step(grad, max_norm=10.0), ob.step(grad, max_norm=10.0)
        assert torch.equal(na, nb)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(oa.exp_avg, ob.exp_avg) and torch.equal(oa.exp_avg_sq, ob.exp_avg_sq)


def test_segment_entry_points_reject_bad_arguments(lib_built):
    from omnidata_b200 import _capi
    lib = _capi.lib()
    stream = torch.cuda.current_stream().cuda_stream
    buf = torch.zeros(4096, device=dev())
    tab = torch.tensor([[0, 1024]], dtype=torch.int64, device=dev())
    ws = torch.zeros(int(lib.odb_grad_norm_workspace_bytes()), dtype=torch.uint8, device=dev())
    out2 = torch.zeros(2, device=dev())
    p, t, w, o = buf.data_ptr(), tab.data_ptr(), ws.data_ptr(), out2.data_ptr()
    for args in [(None, t, 1, 1024), (p, None, 1, 1024), (p, t, 0, 1024), (p, t, 1025, 1024), (p, t, 1, 0),
                 (p + 4, t, 1, 1024), (p, t + 8, 1, 1024)]:
        with pytest.raises(_capi.OdbError):
            _capi.check(lib.odb_clip_grad_norm_segments(*args, 10.0, w, o, stream), "clip_grad_norm_segments")
    with pytest.raises(_capi.OdbError):
        _capi.check(lib.odb_clip_grad_norm_segments(p, t, 1, 1024, 10.0, None, o, stream), "clip_grad_norm_segments")
    for args in [(None, p, p, p, t, 1, 1024), (p, p, p, p, None, 1, 1024), (p, p, p, p, t, 0, 1024),
                 (p, p, p, p, t, 1, 0), (p, p + 4, p, p, t, 1, 1024), (p, p, p, p, t + 8, 1, 1024)]:
        with pytest.raises(_capi.OdbError):
            _capi.check(lib.odb_adam_step_segments(*args, None, 1e-5, 0.9, 0.999, 1e-8, 1, None, stream),
                        "adam_step_segments")
    with pytest.raises(_capi.OdbError):
        _capi.check(lib.odb_adam_step_segments(p, p, p, p, t, 1, 1024, None, 1e-5, 0.9, 0.999, 1e-8, 0, None, stream),
                    "adam_step_segments")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ train step
def _batch():
    g = torch.Generator(device="cpu").manual_seed(9)
    rgb = (torch.rand(2, 3, 384, 384, generator=g) * 2 - 1).to(dev())
    gt = torch.rand(2, 1, 384, 384, generator=g).to(dev())
    mask = (torch.rand(2, 1, 384, 384, generator=g) > 0.1).float().to(dev())
    return rgb, gt, mask


def _train_model(freeze_encoder: bool):
    from omnidata_b200 import synthetic
    from omnidata_b200.model import DPTDepthModel
    model = DPTDepthModel()
    model.load_state_dict(synthetic.make_state_dict(0, 1), strict=True)
    model = model.to(dev()).train()
    if freeze_encoder:
        for n, p in model.named_parameters():
            p.requires_grad_(n.startswith("scratch."))
    return model


def test_train_step_with_a_frozen_encoder():
    from omnidata_b200.train import DepthTrainStep
    LR = 1e-6
    rgb, gt, mask = _batch()
    # one step without clipping: the decoder weights are those of a fully trainable step's (same forward, same decoder
    # gradients, elementwise Adam)
    full = DepthTrainStep(_train_model(False), lr=LR, clip=None)
    part = DepthTrainStep(_train_model(True), lr=LR, clip=None)
    np.random.seed(11)
    full.step(rgb, gt, mask, full_mix=True)
    np.random.seed(11)
    part.step(rgb, gt, mask, full_mix=True)
    torch.cuda.synchronize()
    eng_f, eng_p = full.engine, part.engine
    for n in eng_p.param_names:
        if n.startswith("scratch."):
            assert torch.equal(eng_p.P[n], eng_f.P[n]), n
    assert [t for *_, t in part.buckets] == ["decoder"]
    # three clipped steps, eager and as a CUDA graph: frozen weights and moments bit-unchanged, the loss goes down,
    # the two paths bit-identical, the norm the float64 norm of the trainable gradients
    runs = []
    for graph in (False, True):
        step = DepthTrainStep(_train_model(True), lr=LR, clip=10.0)
        step.use_cuda_graph = graph
        eng = step.engine
        w0 = eng.flat.clone()
        frozen = torch.ones_like(eng.flat, dtype=torch.bool)
        for s, e in step.opt.segments:
            frozen[s:e] = False
        np.random.seed(11)
        hist = [step.step(rgb, gt, mask, full_mix=True).cpu() for _ in range(3)]
        torch.cuda.synchronize()
        assert torch.equal(eng.flat[frozen], w0[frozen])
        assert not step.opt.exp_avg[frozen].any() and not step.opt.exp_avg_sq[frozen].any()
        assert all(torch.isfinite(h).all() for h in hist) and float(hist[-1][0]) < float(hist[0][0])
        runs.append((hist, eng.flat.clone(), step.opt.exp_avg.clone()))
        if not graph:
            exact = float(torch.cat([eng.flat_grad[s:e] for s, e in step.opt.segments]).double().norm())
            assert abs(float(hist[-1][4]) - exact) <= 1e-6 * exact
            for p in step._flag_params[:1]:
                p.requires_grad_(not p.requires_grad)
            with pytest.raises(ValueError):
                step.step(rgb, gt, mask, full_mix=True)
    (h0, f0, m0), (h1, f1, m1) = runs
    assert all(torch.equal(a, b) for a, b in zip(h0, h1)) and torch.equal(f0, f1) and torch.equal(m0, m1)
