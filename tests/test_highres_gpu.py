"""Inference beyond 639 patches (up to 4 096 patches, 4 097 tokens): the streaming instances of the bf16 and fp32
attention kernels, the whole DPTs at high-resolution and non-square inputs, and the input sizes that stay refused.

- Kernels: odb_attention above 640 tokens against the kernel's own rounding definition (oracle/gemm_oracle.py
  attention_bf16, rounded to bf16) at the bound of test_kernels_gpu.py::test_attention (rel-L2 1e-3), lse against float64 log2-sum-exp,
  every output element written, bit-reproducible, batch-independent; odb_attention_f32 against float64 (2e-6).
- Whole model, fp32 mode: rel-L2 <= 1e-5 at every tap, pre-ReLU head included, against the fp32 oracles evaluated in
  float64 (their dtype argument).
- Whole model, bf16: at every tap no further from the fp32 oracle than 1.10 x stock torch.autocast(bfloat16) of the
  oracle, measured live (the rule of test_model_gpu.py::test_not_worse_than_stock_autocast).
- CUDA-graph replay equals eager; batch 17 at 1024 x 1024 (where the head's upsampled map passes 2^31 elements) equals
  17 batch-1 runs bit for bit.
- Refusals (ValueError / OdbError before any launch): more than 4 097 tokens or 4 096 patches, the hybrid's stem width,
  and training / x.grad beyond 639 patches."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TOKENS = [641, 705, 767, 768, 769, 1025, 1201, 2305, 3073, 4097]
TAPS_HYBRID = ["layer_1", "layer_2", "tokens_8", "tokens_11", "layer_3", "layer_4", "layer_1_rn", "layer_2_rn",
               "layer_3_rn", "layer_4_rn", "path_4", "path_3", "path_2", "path_1"]


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


def _qkv(b, t, heads, dtype, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    qkv = torch.randn(b, t, 3, heads * 64, generator=g)
    qkv[:, :, :2] *= 1.5                                    # wider logits: a peaked softmax
    return qkv.reshape(b, t, 3 * heads * 64).to(dev(), dtype)


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("b", [1, 3])
@pytest.mark.parametrize("heads", [12, 16])
@pytest.mark.parametrize("t", TOKENS)
def test_attention_streaming_bf16(t, heads, b):
    from omnidata_b200 import ops
    from oracle import gemm_oracle as G
    qkv = _qkv(b, t, heads, torch.bfloat16, 100 * t + heads + b)
    out = torch.full((b, t, heads * 64), float("nan"), device=dev(), dtype=torch.bfloat16)
    lse = torch.full((b, heads, t), float("nan"), device=dev())
    ops.attention(qkv, out, heads=heads, lse=lse)
    out2 = torch.full_like(out, float("nan"))
    ops.attention(qkv, out2, heads=heads)
    torch.cuda.synchronize()
    assert not out.isnan().any() and not lse.isnan().any()
    assert torch.equal(out, out2)                           # bit-reproducible, lse or not
    errs, lerrs = [], []
    for i in range(b):                                      # one image at a time: S is T x T per head
        q, k, v = qkv[i:i + 1].float().view(1, t, 3, heads, 64).permute(2, 0, 3, 1, 4)
        ref = G.attention_bf16(q, k, v).transpose(1, 2).reshape(1, t, heads * 64)
        errs.append(rel(out[i:i + 1].float(), ref.to(torch.bfloat16).float()))   # as test_kernels_gpu.py::check
        lref = G.lse_ref(qkv[i:i + 1], heads)
        lerrs.append(rel(lse[i:i + 1], lref))
        del q, k, v, ref, lref
    print(f"attention T={t} heads={heads} b={b}: rel-L2 {max(errs):.2e}, lse rel-L2 {max(lerrs):.2e}")
    assert max(errs) <= 1e-3 and max(lerrs) <= 1e-6
    if b > 1:
        for i in range(b):                                  # b images == b single-image calls, bit for bit
            o1 = torch.empty_like(out[:1])
            ops.attention(qkv[i:i + 1].contiguous(), o1, heads=heads)
            torch.cuda.synchronize()
            assert torch.equal(o1[0], out[i])


@pytest.mark.parametrize("heads", [12, 16])
@pytest.mark.parametrize("t", TOKENS)
def test_attention_streaming_fp32(t, heads):
    from omnidata_b200 import ops
    from oracle import gemm_oracle as G
    b = 2
    qkv = _qkv(b, t, heads, torch.float32, 7 * t + heads)
    out = torch.full((b, t, heads * 64), float("nan"), device=dev())
    ops.attention(qkv, out, heads=heads)
    torch.cuda.synchronize()
    assert not out.isnan().any()
    err = max(rel(out[i:i + 1], G.attention_ref(qkv[i:i + 1], heads)) for i in range(b))
    print(f"attention fp32 T={t} heads={heads}: rel-L2 {err:.2e}")
    assert err <= 2e-6


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_attention_refuses_more_than_4097_tokens(dtype):
    from omnidata_b200 import _capi, ops
    qkv = torch.zeros(1, 4098, 3 * 768, device=dev(), dtype=dtype)
    out = torch.zeros(1, 4098, 768, device=dev(), dtype=dtype)
    n0 = _capi.launch_count()
    with pytest.raises(_capi.OdbError):
        ops.attention(qkv, out)
    assert _capi.launch_count() == n0


# ------------------------------------------------------------------------------------------ models
def _model(backbone, c=1, seed=0):
    from omnidata_b200 import synthetic
    from omnidata_b200.model import DPTDepthModel, state_dict_spec
    from oracle import weights
    if backbone == "vitb_rn50_384":
        sd = weights.make_state_dict(seed, c)
    else:
        sd = synthetic.make_state_dict(seed, c, spec=state_dict_spec(c, backbone=backbone))
    m = DPTDepthModel(backbone=backbone, num_channels=c)
    m.load_state_dict(sd, strict=True)
    return m.to(dev()).eval(), sd


def _input(b, h, w, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed + h + 7 * w)
    return (torch.rand(b, 3, h, w, generator=g) * 2 - 1).to(dev())


def _oracle(backbone, sd, x, taps, autocast=False, dtype=torch.float32):
    from oracle import dpt_oracle, plain_vit_oracle
    fwd = dpt_oracle.forward_fp32 if backbone == "vitb_rn50_384" else plain_vit_oracle.forward_fp32
    sdg = {k: v.to(dev()) for k, v in sd.items()}
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        y = fwd(sdg, x, taps, dtype=dtype)
    return y


def _run(model, x, precision):
    model.precision = precision
    model.keep_taps = True
    try:
        with torch.no_grad():
            y = model(x).float()
        # channels-last -> NCHW; vitb16_384 carries layer_1's 96 channels zero-padded to 128
        taps = {k: (v.float() if k.startswith("tokens") or v.dim() != 4 or k == "head_pre_relu"
                    else v.float().permute(0, 3, 1, 2)) for k, v in model.taps.items()}
    finally:
        model.keep_taps = False
        model.precision = "bf16"
    return y, taps


MODEL_CASES = [("vitb_rn50_384", 1, 512, 512), ("vitb_rn50_384", 1, 480, 640), ("vitb_rn50_384", 1, 1024, 1024),
               ("vitb_rn50_384", 3, 512, 512), ("vitl16_384", 1, 512, 512), ("vitl16_384", 1, 768, 1024),
               ("vitb16_384", 1, 512, 512), ("vitb16_384", 1, 768, 1024)]


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(backbone, c):
        if (backbone, c) not in cache:
            cache.clear()                                   # one model resident at a time
            torch.cuda.empty_cache()
            cache[(backbone, c)] = _model(backbone, c)
        return cache[(backbone, c)]
    return get


@pytest.mark.parametrize("backbone,c,h,w", MODEL_CASES, ids=[f"{b}-c{c}-{h}x{w}" for b, c, h, w in MODEL_CASES])
def test_model_highres(models, backbone, c, h, w):
    model, sd = models(backbone, c)
    x = _input(1, h, w)
    # fp32 mode: 1e-5 at every tap against the oracle's arithmetic evaluated in float64.  (At these sizes the fp32
    # evaluation of the oracle itself is about 1e-5 from it at the ReLU output: 480x640 measured 1.1e-5 fp32 mode vs
    # fp32 oracle, every other tap <= 7.2e-6.)
    t64 = {}
    y64 = _oracle(backbone, sd, x, t64, dtype=torch.float64)
    y, taps = _run(model, x, "fp32")
    keys = [k for k in taps if k in t64]
    assert len(keys) >= 12 and "head_pre_relu" in keys
    for k in keys:
        if taps[k].dim() == 4 and taps[k].shape[1] > t64[k].shape[1]:
            assert float(taps[k][:, t64[k].shape[1]:].abs().max()) == 0.0, k
            taps[k] = taps[k][:, :t64[k].shape[1]]
    report = {k: rel(taps[k], t64[k]) for k in keys}
    report["output"] = rel(y, y64)
    del t64, y64
    t32 = {}
    y32 = _oracle(backbone, sd, x, t32).float()
    print(f"\n{backbone} c{c} {h}x{w} fp32 mode: " + ", ".join(f"{k} {v:.2e}" for k, v in report.items()))
    assert max(report.values()) <= 1e-5, report
    # bf16: no further from fp32 than stock autocast
    tac = {}
    yac = _oracle(backbone, sd, x, tac, autocast=True).float()
    y16, taps16 = _run(model, x, "bf16")
    assert tuple(y16.shape) == ((1, h, w) if c == 1 else (1, 3, h, w))
    rows = []
    for k in [k for k in keys if k != "head_pre_relu" and k in tac]:
        mine, stock = rel(taps16[k][:, :t32[k].shape[1]], t32[k]), rel(tac[k].float(), t32[k])
        rows.append((k, mine, stock))
    rows.append(("output", rel(y16, y32), rel(yac, y32)))
    if backbone == "vitb_rn50_384":
        from oracle import dpt_oracle
        t16 = {}
        with torch.no_grad():
            y16o = dpt_oracle.forward_bf16({k: v.to(dev()) for k, v in sd.items()}, x, t16)
        print(f"{backbone} c{c} {h}x{w} bf16 vs forward_bf16: output {rel(y16, y16o.float()):.2e}, " +
              ", ".join(f"{k} {rel(taps16[k], t16[k].float()):.2e}" for k in TAPS_HYBRID if k in t16))
    print(f"{backbone} c{c} {h}x{w} bf16 vs fp32 (stock autocast): " +
          ", ".join(f"{k} {m:.2e} ({s:.2e})" for k, m, s in rows))
    for k, mine, stock in rows:
        assert mine <= 1.10 * stock, (k, mine, stock)


def test_graph_replay_equals_eager_768(models):
    model, _ = models("vitb_rn50_384", 1)
    x = _input(2, 768, 768, seed=3)
    with torch.no_grad():
        e = model(x).clone()
        model.use_cuda_graph = True
        try:
            g1 = model(x).clone()
            g2 = model(x.flip(0)).clone()
        finally:
            model.use_cuda_graph = False
    assert torch.equal(e, g1) and torch.equal(g2, e.flip(0))


@pytest.mark.parametrize("backbone,precision", [("vitb_rn50_384", "bf16"), ("vitb_rn50_384", "fp32"),
                                                ("vitb16_384", "bf16")])
def test_batch17_at_1024_equals_batch1(models, backbone, precision):
    """B = 17 at 1024 x 1024: the head's upsampled map [17, 1024, 1024, 128] has more than 2^31 elements."""
    model, _ = models(backbone, 1)
    x = _input(17, 1024, 1024, seed=5)
    model.precision = precision
    try:
        with torch.no_grad():
            y = model(x)
            for i in range(17):
                assert torch.equal(model(x[i:i + 1])[0], y[i]), i
    finally:
        model.precision = "bf16"
        model._graphs.clear()                               # graphs replay into the workspaces dropped here
        model._workspaces.clear()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ refusals
def test_size_refusals_before_any_launch(models):
    from omnidata_b200 import _capi
    from omnidata_b200.train import DepthTrainStep
    model, _ = models("vitb_rn50_384", 1)
    n0 = _capi.launch_count()
    with torch.no_grad():
        for h, w in [(1056, 1024), (384, 1824), (512, 500)]:   # 4 224 patches; hybrid stem width; not a multiple of 32
            with pytest.raises(ValueError):
                model(torch.zeros(1, 3, h, w, device=dev()))
    with pytest.raises(ValueError):                          # x.grad beyond 639 patches
        model(torch.zeros(1, 3, 512, 512, device=dev(), requires_grad=True))
    model.train()
    try:
        with pytest.raises(ValueError):                      # training beyond 639 patches
            model(torch.zeros(1, 3, 512, 512, device=dev()))
        with pytest.raises(ValueError):
            DepthTrainStep(model, input_size=(512, 512))
    finally:
        model.eval()
    assert _capi.launch_count() == n0
    plain, _ = _model("vitb16_384")
    with torch.no_grad(), pytest.raises(ValueError):
        plain(torch.zeros(1, 3, 1056, 1024, device=dev()))
    assert _capi.launch_count() == n0
