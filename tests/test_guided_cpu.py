"""Guided upsampling without a GPU: the float64 oracle's properties (oracle/guided_oracle.py), the refusals that need
no device, and the compiler report of the guided kernels (csrc/guided.cu)."""
import math
import re
import subprocess

import pytest
import torch

from oracle import guided_oracle as G


def _rand(*shape, seed=0):
    return torch.rand(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


@pytest.mark.parametrize("h,w", [(5, 7), (1, 9), (9, 1)])
@pytest.mark.parametrize("r", [1, 2, 4, 9, 32])
def test_box_mean_is_the_mean_over_clipped_windows(h, w, r):
    """Against a direct loop over every window, including windows larger than the image (r >= h, r >= w)."""
    f = _rand(2, h, w, seed=h * 31 + w + r)
    got = G.box_mean(f, r)
    want = torch.empty_like(f)
    for y in range(h):
        for x in range(w):
            win = f[:, max(0, y - r):min(h, y + r + 1), max(0, x - r):min(w, x + r + 1)]
            want[:, y, x] = win.sum((1, 2)) / win[0].numel()
    assert float((got - want).abs().max()) <= 1e-15


def _scene(B, h, w, H, W, seed):
    """A full-resolution image x and its low-resolution guide g (as GuidedPredictor makes it: x resampled)."""
    x = _rand(B, 3, H, W, seed=seed) * 2 - 1
    return x, G.resample(x, h, w)


def test_affine_equivariance():
    x, g = _scene(2, 12, 16, 30, 41, seed=1)
    p = _rand(2, 1, 12, 16, seed=2)
    s, t = 2.75, -1.5
    q = G.guided(x, g, p, 2, 1e-3, round_fp32=False)
    qa = G.guided(x, g, s * p + t, 2, 1e-3, round_fp32=False)
    want = s * q + t
    assert float((qa - want).abs().max() / want.abs().max()) <= 1e-12


@pytest.mark.parametrize("C", [1, 3])
def test_edge_preservation(C):
    """p = c^T g + d exactly: at eps = 1e-10 the fit recovers (c, d) in every window, so the output at full resolution
    is c^T x + d, with the image's own edges, up to the fp32 rounding of the coefficients."""
    x, g = _scene(1, 16, 20, 61, 77, seed=3)
    gen = torch.Generator().manual_seed(4)
    c = torch.randn(C, 3, generator=gen, dtype=torch.float64)
    d = torch.randn(C, generator=gen, dtype=torch.float64)
    p = torch.einsum("ck,bkhw->bchw", c, g) + d[None, :, None, None]
    q = G.guided(x, g, p, 3, 1e-10)
    want = torch.einsum("ck,bkhw->bchw", c, x) + d[None, :, None, None]
    rng = float(want.max() - want.min())
    err = float((q - want).abs().max()) / rng
    print(f"C={C}: max |q - (c^T x + d)| {err:.2e} of its range")
    assert err <= 2e-6


def test_large_eps_tends_to_the_box_filtered_prediction():
    x, g = _scene(1, 10, 14, 23, 29, seed=5)
    p = _rand(1, 3, 10, 14, seed=6)
    q = G.guided(x, g, p, 2, 1e12, round_fp32=False)
    want = G.resample(G.box_mean(G.box_mean(p, 2), 2), 23, 29)
    assert float((q - want).abs().max()) <= 1e-9


def test_flat_guide_and_flat_prediction_stay_finite():
    x, _ = _scene(1, 8, 8, 20, 20, seed=7)
    g = torch.full((1, 3, 8, 8), 0.25, dtype=torch.float64)                 # Sigma = 0
    p = _rand(1, 1, 8, 8, seed=8)
    q = G.guided(x, g, p, 2, 1e-3)
    assert bool(torch.isfinite(q).all())
    flat = torch.full((1, 3, 8, 8), 0.7, dtype=torch.float64)               # flat prediction: a = 0, b = 0.7
    q = G.guided(x, _scene(1, 8, 8, 20, 20, seed=9)[1], flat, 2, 1e-3)
    assert bool(torch.isfinite(q).all()) and float((q - 0.7).abs().max()) <= 1e-6


class _Stub:
    num_channels = 1

    def __call__(self, x):
        return x[:, 0]


def test_refusals_without_a_device():
    from omnidata_b200 import _capi
    from omnidata_b200.guided import GuidedPredictor
    from omnidata_b200.model import DPTDepthModel
    from omnidata_b200.tiled import TiledPredictor

    class Two(_Stub):
        num_channels = 2
    with pytest.raises(ValueError):
        GuidedPredictor(Two(), size=(64, 64))
    for radius in (0, 33, -1, 2.5):
        with pytest.raises(ValueError):
            GuidedPredictor(_Stub(), size=(64, 64), radius=radius)
    for eps in (0.0, -1e-3, math.inf, math.nan):
        with pytest.raises(ValueError):
            GuidedPredictor(_Stub(), size=(64, 64), eps=eps)
    with pytest.raises(ValueError):
        GuidedPredictor(_Stub(), size=(64, 64), max_batch=0)
    with pytest.raises(ValueError):
        GuidedPredictor(_Stub(), size=(0, 64))
    model = DPTDepthModel().eval()
    for size in [(400, 384), (384, 200), (1056, 1024), (512, 1824)]:
        with pytest.raises(ValueError):
            GuidedPredictor(model, size=size)
    with pytest.raises(ValueError):                                         # beyond the 1 024-tile cap
        GuidedPredictor(TiledPredictor(model), size=(20000, 20000))
    gp = GuidedPredictor(model, size=(384, 512))
    assert gp.num_channels == 1
    with pytest.raises(ValueError):
        gp(torch.zeros(1, 3, 384, 384, requires_grad=True))
    with pytest.raises(_capi.OdbError):
        gp(torch.zeros(1, 3, 384, 384))
    model.train()
    with pytest.raises(ValueError):
        gp(torch.zeros(1, 3, 384, 384))


def test_evaluate_guided_flags():
    import evaluate
    base = ["--task", "depth", "--img_path", "x", "--gt_path", "y", "--synthetic_weights"]
    a = evaluate.parse_args([*base, "--mode", "guided", "--guided_size", "768x1024"])
    assert a.guided_size == (768, 1024) and a.radius == 4 and a.eps == 1e-3
    a = evaluate.parse_args([*base, "--mode", "guided", "--guided_size", "384x512", "--radius", "8", "--eps", "1e-2",
                             "--ensemble_sizes", "native", "--flip"])
    assert (a.radius, a.eps, a.ensemble_sizes, a.flip) == (8, 1e-2, [None], True)
    a = evaluate.parse_args(base)
    assert a.guided_size is None and a.radius is None and a.eps is None
    for bad in (["--mode", "guided"], ["--guided_size", "384x384"], ["--mode", "direct", "--guided_size", "384x384"],
                ["--radius", "3"], ["--eps", "0.1"], ["--mode", "guided", "--guided_size", "384"],
                ["--mode", "guided", "--guided_size", "384x384", "--anchor", "384x384"]):
        with pytest.raises(SystemExit):
            evaluate.parse_args([*base, *bad])


def _ptxas_report(src, tmp_path):
    from omnidata_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, *(["--use_fast_math"] if src in build.FAST_MATH_SOURCES else []),
           "-Xptxas", "-v", "-c", str(build.CSRC / src), "-o", str(tmp_path / (src + ".o"))]
    try:
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    except FileNotFoundError:
        pytest.skip("nvcc not found")
    assert r.returncode == 0, r.stdout
    found, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            found[cur] = tuple(int(x) for x in m.groups())
            cur = None
    return found


def test_guided_kernels_compile_without_spills(tmp_path):
    """The guided kernels, compiled as the build compiles them (without fast-math): no stack frame, no spills."""
    from omnidata_b200 import build
    assert "guided.cu" in build.SOURCES and "guided.cu" not in build.FAST_MATH_SOURCES
    found = _ptxas_report("guided.cu", tmp_path)
    kernels = {k: v for k, v in found.items() if "guided_" in k}
    assert len(kernels) == 8, sorted(found)         # products (C = 1, 3), solve (C = 1, 3), box_v, box_h, apply (C = 1, 3)
    assert all(v == (0, 0, 0) for v in kernels.values()), kernels
