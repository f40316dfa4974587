"""Drop-in boundary without a GPU: state_dict layout, constructor / error behaviour, the C-ABI
library loads and exports every symbol that include/omnidata_b200.h declares."""
import ctypes
import json
import re
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = Path(__file__).parent / "golden"


def test_c_abi_exports_every_declared_symbol(lib_built):
    header = (ROOT / "include" / "omnidata_b200.h").read_text()
    declared = sorted(set(re.findall(r"\b(odb_[a-z0-9_]+)\s*\(", header)))
    assert len(declared) >= 12
    lib = ctypes.CDLL(str(lib_built))
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    from omnidata_b200 import _capi
    assert sorted(_capi.exported_symbols()) == declared
    assert _capi.lib().odb_abi_version() == _capi.ABI_VERSION == 4
    assert _capi.launch_count() == 0


def test_compute_entry_fails_loudly_without_gpu(lib_built):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from omnidata_b200 import _capi, ops
    with pytest.raises(_capi.OdbError):
        ops.layernorm(torch.zeros(2, 768, dtype=torch.bfloat16), torch.ones(768), torch.zeros(768),
                      torch.zeros(2, 768, dtype=torch.bfloat16))
    # a raw C call on host pointers must return an error code, not crash or silently compute
    d = _capi.ConvGemmDesc()
    rc = _capi.lib().odb_conv_gemm(ctypes.byref(d), None)
    assert rc != 0 and len(_capi.lib().odb_last_error()) > 0


@pytest.mark.parametrize("c", [1, 3])
def test_state_dict_layout_is_the_reference_layout(c):
    from omnidata_b200.model import DPTDepthModel, state_dict_spec
    keys = json.loads((GOLDEN / "state_dict_keys.json").read_text())
    if c == 3:
        keys = [[k, ([3] + s[1:] if k.startswith("scratch.output_conv.4.") else s)] for k, s in keys]
    model = DPTDepthModel(backbone="vitb_rn50_384", num_channels=c)
    got = [[k, list(v.shape)] for k, v in model.state_dict().items()]
    assert got == keys
    assert [[k, list(s)] for k, s in state_dict_spec(c)] == keys
    # strict load of a reference-layout checkpoint, incl. the PL 'model.' prefix handling of demo.py:65-68
    from oracle import weights
    sd = weights.make_state_dict(0, c)
    model.load_state_dict(sd, strict=True)
    assert torch.equal(model.state_dict()["scratch.refinenet4.resConfUnit1.conv1.weight"],
                       sd["scratch.refinenet4.resConfUnit1.conv1.weight"])
    with pytest.raises(RuntimeError):
        bad = dict(sd)
        bad.pop("pretrained.model.norm.weight")
        model.load_state_dict(bad, strict=True)


def test_constructor_and_forward_errors():
    from omnidata_b200._capi import OdbError
    from omnidata_b200.model import DPTDepthModel
    with pytest.raises(AssertionError):
        DPTDepthModel(backbone="resnext101_wsl")   # reference: print + assert False for backbones it does not build
    m = DPTDepthModel()
    assert m.num_channels == 1 and m.non_negative
    if not torch.cuda.is_available():
        with pytest.raises(OdbError):
            m(torch.zeros(1, 3, 384, 384))


def test_hub_entry_points_exist():
    import importlib.util
    spec = importlib.util.spec_from_file_location("hubconf", ROOT / "hubconf.py")
    hub = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(hub)
    for name in ("depth_dpt_hybrid_384", "surface_normal_dpt_hybrid_384", "dpt_hybrid_384"):
        assert callable(getattr(hub, name))
    m = hub.dpt_hybrid_384(pretrained=False, task="normal")
    assert m.num_channels == 3
    m = hub.dpt_hybrid_384(pretrained=False, task="depth")
    assert m.num_channels == 1


@pytest.mark.parametrize("backbone,golden", [("vitl16_384", "dpt_large_fp32_seed0_c1.pt"),
                                             ("vitb16_384", "dpt_vitb16_fp32_seed0_c1.pt")])
def test_plain_vit_state_dict_layout_is_the_reference_layout(backbone, golden):
    """backbones 'vitl16_384' (demo.py:81) / 'vitb16_384': key / shape / order of the reference class, from the golden
    file (any box) and from the unmodified reference class itself (build container)."""
    from omnidata_b200.model import DPTDepthModel, state_dict_spec
    from oracle import reference_loader
    rec = torch.load(GOLDEN / golden)
    spec = [[k, list(s)] for k, s in state_dict_spec(1, backbone=backbone)]
    assert spec == rec["spec"]
    model = DPTDepthModel(backbone=backbone)
    assert [[k, list(v.shape)] for k, v in model.state_dict().items()] == spec
    if reference_loader.reference_available():
        ref = reference_loader.load_reference_dpt(1, backbone)
        assert [[k, list(v.shape)] for k, v in ref.state_dict().items()] == spec


@pytest.mark.parametrize("backbone", ["vitb_rn50_384", "vitl16_384", "vitb16_384"])
def test_gemm_layer_table_matches_the_state_dict(backbone):
    """Every GEMM layer reads its whole weight as [n][c][taps], pads without truncating and names a bias of the
    model."""
    import math
    from omnidata_b200.model import _ARCH, gemm_layers, state_dict_spec
    spec = dict(state_dict_spec(1, backbone=backbone))
    layers = gemm_layers(_ARCH[backbone])
    assert len({L.key for L in layers}) == len(layers)
    for L in layers:
        assert L.n * L.c * L.taps == math.prod(spec[L.weight]), L.key
        assert L.n_pad >= L.n and L.c_pad >= L.c, L.key
        assert L.bias is None or spec.get(L.bias) == (L.n,), L.key


def test_every_host_module_refuses_cpu_tensors():
    """No CPU / eager fallback anywhere: the host mirrors raise instead of computing on the CPU."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import numpy as np
    from omnidata_b200 import imageproc, losses, optim, refocus
    from omnidata_b200._capi import OdbError
    with pytest.raises(OdbError):
        optim.FlatAdam(torch.zeros(8))
    with pytest.raises(OdbError):
        imageproc.bicubic_resize(torch.zeros(1, 4, 4), (8, 8))
    with pytest.raises(OdbError):
        imageproc.to_uint8_hwc(torch.zeros(3, 4, 4))
    with pytest.raises(OdbError):
        losses.MidasLoss()(torch.zeros(1, 1, 8, 8), torch.zeros(1, 1, 8, 8), torch.ones(1, 1, 8, 8, dtype=torch.bool))
    with pytest.raises(OdbError):
        losses.VNL_Loss(1.0, 1.0, (8, 8))(torch.zeros(1, 1, 8, 8), torch.zeros(1, 1, 8, 8))
    with pytest.raises(OdbError):
        losses.normal_losses(torch.zeros(1, 3, 8, 8), torch.zeros(1, 3, 8, 8), torch.ones(1, 1, 8, 8, dtype=torch.bool))
    with pytest.raises(OdbError):
        refocus.compute_quantiles(torch.zeros(1, 1, 8, 8), 4)
    with pytest.raises((OdbError, RuntimeError, AssertionError)):
        imageproc.DevicePreprocessor("depth")(np.zeros((8, 8, 3), dtype=np.uint8))


def test_adam_step_scalars_are_torchs_host_arithmetic(lib_built):
    """odb_adam_step_scalars (host function; what a captured train step stages before each replay) reproduces
    torch.optim.Adam's scalar preparation: python floats (doubles) for bias_correction1/2, step_size = lr / bc1 and
    sqrt(bc2), then one rounding to fp32 — and refuses step < 1 / a null pointer."""
    import ctypes as C
    import math
    import numpy as np
    from omnidata_b200 import _capi
    lib = _capi.lib()
    out = (C.c_float * 2)()
    for lr, b1, b2 in ((1e-5, 0.9, 0.999), (3e-4, 0.8, 0.99)):
        lr32, b132, b232 = (float(np.float32(v)) for v in (lr, b1, b2))     # the C ABI takes fp32 scalars
        for step in (1, 2, 10, 1000, 15000):
            assert lib.odb_adam_step_scalars(lr, b1, b2, step, out) == 0
            bc1, bc2 = 1.0 - b132 ** step, 1.0 - b232 ** step
            assert out[0] == np.float32(lr32 / bc1) and out[1] == np.float32(math.sqrt(bc2))
    assert lib.odb_adam_step_scalars(1e-5, 0.9, 0.999, 0, out) != 0
    assert lib.odb_adam_step_scalars(1e-5, 0.9, 0.999, 1, None) != 0
