"""Training and differentiating the DPT-Hybrid at input sizes other than 384x384 (H, W multiples of 32, <= 639 patches).

Off the 24 x 24 patch grid the forward resizes pos_embed's patch rows bilinearly (vit.py:102-116); the backward takes their
gradient through odb_pos_embed_resize_bwd, the adjoint of that resize.  Checkers:
  * the kernel: float64 torch.autograd of F.interpolate(mode="bilinear", align_corners=False) on the identical input;
  * the network: float64 torch.autograd of oracle/dpt_oracle.py::forward_fp32 (which resizes pos_embed the same way),
    with the seeded weights and R-weighted loss of test_train_gpu.py, at the bounds that file holds 384x384 to;
  * bf16: stock torch.autocast(bfloat16) autograd of the same oracle, measured live.
Sizes are (H, W)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SIZES = [(320, 480), (384, 416)]


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


# ------------------------------------------------------------------------------------------ the kernel
def _resize_reference(dgrid, gh, gw):
    """float64 autograd of F.interpolate(bilinear) of a 24 x 24 grid to gh x gw -> [24*24, D].  In float64, torch also
    computes the interpolation weights in float64."""
    d = dgrid.shape[-1]
    src = torch.zeros(1, d, 24, 24, dtype=torch.float64, device=dev(), requires_grad=True)
    y = F.interpolate(src, size=(gh, gw), mode="bilinear", align_corners=False)
    g, = torch.autograd.grad(y, src, dgrid.double().view(gh, gw, d).permute(2, 0, 1).unsqueeze(0))
    return g[0].permute(1, 2, 0).reshape(24 * 24, d)


def _fp32_map_transpose(dgrid, gh, gw):
    """The transpose of the map the fp32 forward applies, evaluated in float64: the per-axis weight matrices are read off
    fp32 F.interpolate of one-hot rows (resized along one axis only, where every product is exact)."""
    d = dgrid.shape[-1]
    eye = torch.eye(24, device=dev()).view(1, 24, 24, 1).expand(1, 24, 24, 24).contiguous()     # [1][i][y][x] = (y == i)
    my = F.interpolate(eye, size=(gh, 24), mode="bilinear")[0, :, :, 0].double()               # [i][jy]
    mx = F.interpolate(eye.transpose(2, 3), size=(24, gw), mode="bilinear")[0, :, 0, :].double()  # [i][jx]
    return torch.einsum("ij,kl,jld->ikd", my, mx, dgrid.double().view(gh, gw, d)).reshape(24 * 24, d)


@pytest.mark.parametrize("gh,gw", [(16, 16), (20, 30), (24, 26), (26, 24), (38, 16)])
def test_pos_embed_resize_bwd_kernel(gh, gw):
    """Against the float64 transpose of the fp32 map: <= 1e-6 (fp32 accumulation only).  Against float64 autograd of
    F.interpolate the fp32 interpolation weights the forward uses (torch's float index arithmetic) add up to ~1.5e-6
    of their own, so that comparison is held to 2e-6."""
    from omnidata_b200 import bwd
    g = torch.Generator(device="cpu").manual_seed(gh * 100 + gw)
    dgrid = torch.randn(gh * gw, 768, generator=g).to(dev())
    dpos = torch.full((24 * 24, 768), float("nan"), device=dev())
    bwd.pos_embed_resize_bwd(dgrid, gh, gw, dpos)
    torch.cuda.synchronize()
    err = rel(dpos, _fp32_map_transpose(dgrid, gh, gw))
    err64 = rel(dpos, _resize_reference(dgrid, gh, gw))
    print(f"pos_embed_resize_bwd 24x24 <- {gh}x{gw}: rel-L2 {err:.2e} against the float64 transpose of the fp32 map, "
          f"{err64:.2e} against float64 autograd of F.interpolate")
    assert err <= 1e-6 and err64 <= 2e-6
    dpos2 = torch.full_like(dpos, float("nan"))
    bwd.pos_embed_resize_bwd(dgrid, gh, gw, dpos2)
    assert torch.equal(dpos, dpos2)


def test_pos_embed_resize_bwd_rejects_bad_arguments():
    from omnidata_b200 import _capi, bwd
    dgrid = torch.zeros(20 * 30, 768, device=dev())
    dpos = torch.empty(24 * 24, 768, device=dev())
    lib = _capi.lib()
    stream = torch.cuda.current_stream().cuda_stream
    p, o = dgrid.data_ptr(), dpos.data_ptr()
    bad = [
        (None, o, 20, 30, 768),            # null pointers
        (p, None, 20, 30, 768),
        (p, o, 0, 30, 768),                # non-positive sizes
        (p, o, 20, -1, 768),
        (p, o, 20, 30, 0),
        (p, o, 20, 30, 766),               # D not a multiple of 4
        (p + 4, o, 20, 30, 768),           # misaligned
    ]
    for args in bad:
        with pytest.raises(_capi.OdbError):
            _capi.check(lib.odb_pos_embed_resize_bwd(*args, stream), "pos_embed_resize_bwd")
    with pytest.raises(_capi.OdbError):
        bwd.pos_embed_resize_bwd(dgrid, 20, 31, dpos)                              # dgrid is not gh*gw rows
    with pytest.raises(_capi.OdbError):
        bwd.pos_embed_resize_bwd(dgrid, 20, 30, dpos[:-1])                         # dpos is not 24*24 rows
    with pytest.raises(_capi.OdbError):
        bwd.pos_embed_resize_bwd(dgrid.bfloat16(), 20, 30, dpos)                   # fp32 only
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ whole network
def _inputs(h, w, batch=1, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.rand(batch, 3, h, w, generator=g) * 2 - 1
    R = torch.randn(batch, h, w, generator=torch.Generator(device="cpu").manual_seed(123 + seed)).to(dev())
    return x, R


def _model(sd, precision, mode="train"):
    from omnidata_b200.model import DPTDepthModel
    m = DPTDepthModel(backbone="vitb_rn50_384")
    m.load_state_dict(sd, strict=True)
    m = m.to(dev())
    m.train(mode == "train")
    m.precision = precision
    return m


def _engine_grads(model, x, R, need_x_grad=False):
    """-> (output, {name: p.grad}, x.grad or None) of sum(model(x) * R)."""
    for p in model.parameters():
        p.grad = None
    xi = x.to(dev()).clone().requires_grad_(need_x_grad)
    y = model(xi)
    assert y.requires_grad
    (y * R).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    return y.detach(), grads, (xi.grad.detach().clone() if need_x_grad else None)


def _reference_grads(sd, x, R, dtype=torch.float64, autocast=False):
    from oracle import dpt_oracle
    leaves = {k: v.to(dev()).to(dtype).requires_grad_(True) for k, v in sd.items()}
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        y = dpt_oracle.forward_fp32(leaves, x.to(dev()).to(dtype), dtype=dtype)
    grads = torch.autograd.grad((y.to(dtype) * R.to(dtype)).sum(), list(leaves.values()), allow_unused=True)
    return y.detach(), {k: (g if g is not None else torch.zeros_like(leaves[k])) for k, g in zip(leaves, grads)}


def _compare(g_ref, g_mine, per_tensor_tol, global_tol, min_cos):
    worst, num, dot, n1, n2 = [], 0.0, 0.0, 0.0, 0.0
    assert set(g_ref) == set(g_mine) and len(g_ref) == 368
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


@pytest.fixture(scope="module")
def sd():
    from oracle import weights
    return weights.make_state_dict(0, 1)


_HEAD = ["scratch.output_conv.0.weight", "scratch.output_conv.0.bias", "scratch.output_conv.2.weight",
         "scratch.output_conv.2.bias", "scratch.output_conv.4.weight", "scratch.output_conv.4.bias"]


def _head_grads_with_masks(sd, path_1, R, m2, m4):
    """float64 autograd of the head (dpt_depth.py:91-99) from path_1, with its two ReLUs replaced by the given 0/1 masks."""
    p = {k: sd[k].to(dev()).double().requires_grad_(True) for k in _HEAD}
    o = F.conv2d(path_1, p[_HEAD[0]], p[_HEAD[1]], padding=1)
    o = F.interpolate(o, scale_factor=2, mode="bilinear", align_corners=True)
    o = F.conv2d(o, p[_HEAD[2]], p[_HEAD[3]], padding=1) * m2
    o = F.conv2d(o, p[_HEAD[4]], p[_HEAD[5]]) * m4
    return dict(zip(_HEAD, torch.autograd.grad((o.squeeze(1) * R.double()).sum(), [p[k] for k in _HEAD])))


def _group_rel(g, g_ref, keys):
    num = sum(float((g[k].double() - g_ref[k].double()).pow(2).sum()) for k in keys)
    return (num / sum(float(g_ref[k].double().pow(2).sum()) for k in keys)) ** 0.5


@pytest.mark.parametrize("h,w", SIZES)
def test_network_backward_fp32_mode(sd, h, w):
    """Output <= 1e-5, per tensor <= 5e-3 and cosine >= 0.999999 as at 384x384; global <= 1e-3 on these seeded inputs
    (H100: 8.3e-4 at 320x480, 6.6e-4 at 384x416; bit-reproducible, so the numbers do not move between runs).

    The global error is set by ReLU threshold flips, not by the input size: an fp32 forward puts a handful of the
    millions of pre-activations on the other side of zero, and each flip moves the exact gradient by O(1) at one element.
    Measured with this recipe on an H100: at 384x384, seeds 0 / 1 / 2 give 1.6e-4 / 3.6e-4 / 4.5e-4; at other sizes,
    256x256 2.6e-4 up to 448x320 3.6e-3.  The float64 gradient itself moves by 1.3e-3 to 7.9e-3 when the input gets
    1e-6 of noise, at every size including 384x384.  The head shows the mechanism: its gradients here are 2.8e-4 from
    float64 at 320x480 and 3.8e-3 at 448x320, from 1 and 2 flipped elements of its 4.9M / 4.6M-element inner ReLU.  With
    the engine's own ReLU masks put into the float64 head they are 1.0e-6 to 3.6e-6 from it at every size.  The same
    check is asserted below, so a defect in a backward kernel at these shapes cannot hide behind the flips."""
    from oracle import dpt_oracle
    x, R = _inputs(h, w)
    model = _model(sd, "fp32")
    y, g, _ = _engine_grads(model, x, R)
    y_ref, g_ref = _reference_grads(sd, x, R)
    assert y.shape == (1, h, w)
    err_y = rel(y, y_ref)
    print(f"{h}x{w} fp32 mode: output rel-L2 {err_y:.2e}")
    assert err_y <= 1e-5
    _compare(g_ref, g, per_tensor_tol=5e-3, global_tol=1e-3, min_cos=0.999999)
    pm = "pretrained.model."
    for k in (pm + "pos_embed", pm + "cls_token"):
        e = rel(g[k], g_ref[k])
        print(f"  {k}: rel-L2 {e:.2e}")
        assert float(g_ref[k].norm()) > 0 and e <= 5e-3
    # the head's backward against float64 on the branch of the ReLUs the engine's forward took
    hd = model._train_engine.saved["head"]
    m2 = (hd["a"][..., :32] > 0).permute(0, 3, 1, 2).double()
    m4 = (hd["out"] > 0).double()
    taps = {}
    with torch.no_grad():
        dpt_oracle.forward_fp32({k: v.to(dev()).double() for k, v in sd.items()}, x.to(dev()).double(), taps=taps,
                                dtype=torch.float64)
    g_head = _head_grads_with_masks(sd, taps["path_1"], R, m2, m4)
    e_nat, e_msk = _group_rel(g, g_ref, _HEAD), _group_rel(g, g_head, _HEAD)
    print(f"  head: rel-L2 {e_nat:.2e} against float64, {e_msk:.2e} with the engine's ReLU masks")
    assert e_msk <= 1e-5


def test_network_backward_bf16_mode(sd):
    h, w = SIZES[0]
    x, R = _inputs(h, w)
    model = _model(sd, "bf16")
    _, g, _ = _engine_grads(model, x, R)
    _, g_ref = _reference_grads(sd, x, R)
    mine = _compare(g_ref, g, per_tensor_tol=10.0, global_tol=10.0, min_cos=0.0)
    _, g_ac = _reference_grads(sd, x, R, torch.float32, autocast=True)
    stock = _compare(g_ref, g_ac, per_tensor_tol=10.0, global_tol=10.0, min_cos=0.0)
    print(f"{h}x{w} bf16 mode: global rel-L2 {mine:.3e}; stock autocast(bf16) autograd {stock:.3e}")
    assert mine <= 1.6 * stock, (mine, stock)
    _, g2, _ = _engine_grads(model, x, R)
    assert all(torch.equal(g[k], g2[k]) for k in g)


def _train_and_eval(sd, precision, h, w):
    """-> (train-mode output, eval-mode output, train engine's pos rows, inference's pos rows) on one batch of 2."""
    x, _ = _inputs(h, w, batch=2)
    model = _model(sd, precision)
    y_train = model(x.to(dev()))
    assert y_train.requires_grad
    pos_train = model._train_engine.pk["pos_cache"][(h // 16, w // 16, 2)].clone()
    model.eval()
    y_eval = model(x.to(dev()))
    assert not y_eval.requires_grad
    return y_train.detach(), y_eval, pos_train, model._packed["pos_cache"][(h // 16, w // 16, 2)]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("h,w", SIZES)
def test_train_forward_matches_eval_forward(sd, precision, h, w):
    """The training forward resizes pos_embed exactly as inference does: the patch GEMM's pos rows are the same bits.
    The two outputs are not bit-identical at any size, 384x384 included: the training sequence stores and rounds at
    the points its backward needs (DESIGN §1).  So the difference at (h, w) is held to the one at 384x384, measured live
    (H100: fp32 1.7e-6 / 1.8e-6, bf16 2.4e-2 / 2.5e-2 at 384x384 / 320x480)."""
    y_train, y_eval, pos_train, pos_eval = _train_and_eval(sd, precision, h, w)
    assert torch.equal(pos_train, pos_eval)
    d = rel(y_train, y_eval)
    y_train, y_eval, _, _ = _train_and_eval(sd, precision, 384, 384)
    d384 = rel(y_train, y_eval)
    print(f"{h}x{w} {precision}: train vs eval forward rel-L2 {d:.2e} (384x384: {d384:.2e})")
    assert d <= 1.5 * d384 + 1e-7


def test_input_grad_at_320x480(sd):
    from oracle import dpt_oracle
    h, w = SIZES[0]
    x, R = _inputs(h, w)
    _, _, dx = _engine_grads(_model(sd, "fp32"), x, R, need_x_grad=True)
    xi = x.to(dev()).double().requires_grad_(True)
    leaves = {k: v.to(dev()).double() for k, v in sd.items()}
    dx64, = torch.autograd.grad((dpt_oracle.forward_fp32(leaves, xi, dtype=torch.float64) * R.double()).sum(), xi)
    err = rel(dx, dx64)
    print(f"{h}x{w} fp32 mode x.grad rel-L2 {err:.3e} against float64 autograd")
    assert err <= 5e-3
    # bf16: one image alone and inside a batch of 2; eval() and train() give the same x.grad
    model = _model(sd, "bf16")
    x2, R2 = _inputs(h, w, batch=2, seed=5)
    x2[0], R2[0] = x[0], R[0]
    _, _, dx1 = _engine_grads(model, x, R, need_x_grad=True)
    _, _, dx2 = _engine_grads(model, x2, R2, need_x_grad=True)
    assert torch.equal(dx1[0], dx2[0])
    model.eval()
    _, _, dx_eval = _engine_grads(model, x, R, need_x_grad=True)
    assert torch.equal(dx_eval, dx1)


def test_one_engine_switching_sizes_equals_fresh_engines(sd):
    cases = [(384, 384), (320, 480), (384, 384)]
    model = _model(sd, "bf16")
    switched = [_engine_grads(model, *_inputs(h, w), need_x_grad=True) for h, w in cases]
    for (h, w), (y, g, dx) in zip(cases, switched):
        y0, g0, dx0 = _engine_grads(_model(sd, "bf16"), *_inputs(h, w), need_x_grad=True)
        assert torch.equal(y, y0) and torch.equal(dx, dx0), (h, w)
        assert all(torch.equal(g[k], g0[k]) for k in g), (h, w)


# ------------------------------------------------------------------------------------------ the train step
def _step_batch(h, w, batch=2):
    g = torch.Generator(device="cpu").manual_seed(9)
    rgb = (torch.rand(batch, 3, h, w, generator=g) * 2 - 1).to(dev())
    gt = torch.rand(batch, 1, h, w, generator=g).to(dev())
    mask = (torch.rand(batch, 1, h, w, generator=g) > 0.1).float().to(dev())
    return rgb, gt, mask


def _train_step(size, graph=False):
    from omnidata_b200 import synthetic
    from omnidata_b200.model import DPTDepthModel
    from omnidata_b200.train import DepthTrainStep
    model = DPTDepthModel()
    model.load_state_dict(synthetic.make_state_dict(0, 1), strict=True)
    step = DepthTrainStep(model.to(dev()).train(), lr=1e-6, clip=10.0, precision="bf16", input_size=size)
    step.use_cuda_graph = graph
    return step


def test_train_step_at_320x480_learns_and_is_deterministic():
    size = SIZES[0]
    batch = _step_batch(*size)
    runs = []
    for graph in (False, False, True):
        step = _train_step(size, graph)
        np.random.seed(11)
        hist = [step.step(*batch, full_mix=True).cpu() for _ in range(3)]
        torch.cuda.synchronize()
        assert all(torch.isfinite(hh).all() for hh in hist) and torch.isfinite(step.engine.flat).all()
        assert float(hist[-1][0]) < float(hist[0][0])               # the loss goes down on the fixed batch
        assert float(hist[0][4]) > 0
        runs.append((hist, step.engine.flat.clone()))
    for hist, flat in runs[1:]:                                      # a second eager run, then the CUDA-graph replay
        assert all(torch.equal(a, b) for a, b in zip(hist, runs[0][0])) and torch.equal(flat, runs[0][1])


def test_step_inputs_are_validated_before_any_launch():
    from omnidata_b200 import _capi, losses
    size = SIZES[0]
    h, w = size
    rgb, gt, mask = _step_batch(h, w)
    step = _train_step(size)
    fn = losses.DepthStepLoss(size)
    pred = torch.rand(2, 1, h, w, device=dev())
    np.random.seed(3)
    good = fn.vnl.select_index()
    over = [good[0], good[1].copy(), good[2]]
    over[1][7] = h * w
    under = [good[0].copy(), good[1], good[2]]
    under[0][0] = -1
    short = [good[0], good[1][:-1], good[2]]
    sq = _step_batch(384, 384)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    for args, kw in [((torch.rand(2, 1, 384, 384, device=dev()), sq[1], sq[2]), {}),      # size mismatch
                     ((pred, gt, mask), {"points": over}), ((pred, gt, mask), {"points": under}),
                     ((pred, gt, mask), {"points": short})]:
        with pytest.raises(ValueError):
            fn(*args, full_mix=True, **kw)
    for args, kw in [(sq, {}), ((rgb, sq[1], mask), {}), ((rgb, gt, sq[2]), {}),          # size mismatch
                     ((rgb, gt, mask), {"points": over}), ((rgb, gt, mask), {"points": under}),
                     ((rgb, gt, mask), {"points": short})]:
        with pytest.raises(ValueError):
            step.step(*args, full_mix=True, **kw)
    step.use_cuda_graph = True
    with pytest.raises(ValueError):
        step.step(rgb, gt, mask, full_mix=True, points=over)
    assert _capi.launch_count() == n0
    assert step.global_step == 0 and not step._graphs
