"""Test-time ensembles without a GPU: the float64 oracle's properties (oracle/ensemble_oracle.py), the refusals that
need no device, and the compiler report of the ensemble kernels (csrc/ensemble.cu)."""
import math
import re
import subprocess

import pytest
import torch

from oracle import ensemble_oracle as E


def _smooth(B, H, W, seed=0):
    gen = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H, dtype=torch.float64), torch.linspace(0, 1, W, dtype=torch.float64),
                            indexing="ij")
    ph = torch.rand(B, 1, 1, generator=gen, dtype=torch.float64) * 3
    return 1.5 + torch.sin(3 * xx + 1 + ph) * torch.cos(2 * yy) + 0.5 * xx * yy


def _affine_members(g, K, flips, seed):
    """Members (g - t_k) / s_k of g [B, H, W], s_k in [0.5, 2], t_k ~ N(0, 1), member 0 = g, stored mirrored where
    bit k of flips is set: [K, B, 1, H, W] float32."""
    gen = torch.Generator().manual_seed(seed)
    B = g.shape[0]
    s = torch.rand(K, B, 1, 1, generator=gen, dtype=torch.float64) * 1.5 + 0.5
    t = torch.randn(K, B, 1, 1, generator=gen, dtype=torch.float64)
    s[0], t[0] = 1.0, 0.0
    a = ((g[None] - t) / s).float()
    return torch.stack([a[k].flip(-1) if (flips >> k) & 1 else a[k] for k in range(K)])[:, :, None]


def _merge(members, flips):
    K = members.shape[0]
    st = E.solve(E.gram(members, flips), K)
    return E.merge_depth(members, flips, st), st


@pytest.mark.parametrize("K,flips", [(2, 0b10), (3, 0b010), (6, 0b101010), (16, 0xAAAA)])
def test_exact_affine_members_merge_to_member_0(K, flips):
    """Members that are exact affine maps of member 0 align to it up to kappa's pull: kappa |(1 - s_k, t_k)| over the
    data's curvature (the variance of the member, ~0.2 here), ~1e-5 of member 0's range."""
    g = _smooth(2, 40, 56, seed=K)
    members = _affine_members(g, K, flips, seed=K)
    (out, spread), st = _merge(members, flips)
    a0 = members[0, :, 0].double()
    err = float((out.double() - a0).abs().max() / (a0.max() - a0.min()))
    print(f"K={K}: max |merge - member 0| {err:.2e} of its range, max spread {float(spread.max()):.2e}")
    assert err <= 5e-5
    assert float(spread.max()) <= 5e-5 * float(a0.max() - a0.min())


def test_permuting_members_1_to_k_does_not_change_the_merge():
    K, flips = 6, 0b101010
    g = _smooth(1, 33, 47, seed=1)
    gen = torch.Generator().manual_seed(2)
    members = _affine_members(g, K, flips, seed=3) + 0.01 * torch.randn(K, 1, 1, 33, 47, generator=gen)
    out, spread = _merge(members, flips)[0]
    perm = [0, 3, 5, 1, 4, 2]
    pflips = sum(1 << i for i, k in enumerate(perm) if (flips >> k) & 1)
    pout, pspread = _merge(members[perm], pflips)[0]
    assert float((pout - out).abs().max()) <= 1e-6 * float(out.abs().max())
    assert float((pspread - spread).abs().max()) <= 1e-6 * float(out.abs().max())


def test_one_member_is_the_identity():
    g = _smooth(2, 20, 30).float()[None, :, None]
    g[0, 1, 0, 3, 4] = math.nan
    (out, spread), st = _merge(g, 0)
    assert torch.equal(st, torch.tensor([[[1.0, 0.0]], [[1.0, 0.0]]], dtype=torch.float64))
    assert torch.equal(torch.isnan(out), torch.isnan(g[0, :, 0]))
    assert torch.equal(out.nan_to_num(), g[0, :, 0].nan_to_num())
    assert float(spread.nan_to_num().abs().max()) == 0.0 and bool(spread[1, 3, 4].isnan())


def test_flat_member_is_well_posed():
    """A constant member: its (s, t) is singular in the pair terms alone; kappa keeps the solve finite and pulls it to
    s = 1 only where the data leave it free."""
    K = 3
    g = _smooth(1, 30, 40)
    members = _affine_members(g, K, 0b010, seed=4)
    members[2] = 0.7
    (out, spread), st = _merge(members, 0b010)
    assert bool(torch.isfinite(st).all()) and bool(torch.isfinite(out).all())
    A, _ = E.normal_equations(E.gram(members, 0b010)[0], K)
    assert bool((torch.linalg.eigvalsh(A) > 0).all())


def test_solution_minimises_the_energy():
    K, flips = 4, 0b1010
    g = _smooth(1, 25, 31, seed=5)
    gen = torch.Generator().manual_seed(6)
    members = _affine_members(g, K, flips, seed=7) + 0.05 * torch.randn(K, 1, 1, 25, 31, generator=gen)
    st = E.solve(E.gram(members, flips), K)[0]
    a = E.unmirror(members, flips)[:, 0, 0]
    e0 = E.energy(a, st)
    for i in range(2, 2 * K):
        for h in (1e-4, -1e-4):
            p = st.clone().reshape(-1)
            p[i] += h
            assert E.energy(a, p.view(K, 2)) >= e0


def test_even_median_rule():
    """Even K: the float32 mean of the two middle values; spread: the same rule on |d_k - out|."""
    vals = torch.tensor([4.0, 1.0, 3.0, 10.0])
    members = vals.view(4, 1, 1, 1, 1).expand(4, 1, 1, 2, 2).contiguous()
    st = torch.tensor([[[1.0, 0.0]] * 4], dtype=torch.float64)
    out, spread = E.merge_depth(members, 0, st)
    assert torch.equal(out, torch.full((1, 2, 2), 3.5))                 # (3 + 4) / 2
    assert torch.equal(spread, torch.full((1, 2, 2), 1.5))              # |d - 3.5| = 0.5, 2.5, 0.5, 6.5 -> (0.5 + 2.5) / 2
    odd = E.merge_depth(members[:3], 0, st[:, :3])[0]
    assert torch.equal(odd, torch.full((1, 2, 2), 3.0))


def test_normal_flip_negates_x():
    """A mirrored member of a mirror-symmetric scene: un-mirroring and negating x gives back the unflipped member, so
    the merge is member 0's normalised vector and the spread is zero."""
    gen = torch.Generator().manual_seed(8)
    n = torch.randn(1, 3, 9, 13, generator=gen, dtype=torch.float64)
    n = n / n.norm(dim=1, keepdim=True)
    c = ((n + 1) / 2).float()
    mirrored = c.flip(-1).clone()
    mirrored[:, 0] = 1.0 - mirrored[:, 0]                               # x negated in the [0, 1] encoding
    out, spread = E.merge_normal(torch.stack([c, mirrored]), 0b10)
    ref, _ = E.merge_normal(c[None], 0)
    assert float((out - ref).abs().max()) <= 1e-7
    assert float(spread.max()) <= 1e-3


def test_refusals_without_a_device():
    from omnidata_b200 import _capi
    from omnidata_b200.ensemble import EnsemblePredictor
    from omnidata_b200.model import DPTDepthModel

    class Stub:
        num_channels = 1

        def __call__(self, x):
            return x[:, 0]
    with pytest.raises(ValueError):                         # 9 sizes x flip = 18 members
        EnsemblePredictor(Stub(), sizes=[None] * 9, flip=True)
    with pytest.raises(ValueError):
        EnsemblePredictor(Stub(), sizes=[(0, 10)])
    with pytest.raises(ValueError):
        EnsemblePredictor(Stub(), max_batch=0)
    model = DPTDepthModel().eval()
    for size in [(400, 384), (384, 200), (1056, 1024), (512, 1824)]:
        with pytest.raises(ValueError):
            EnsemblePredictor(model, sizes=[None, size])
    ens = EnsemblePredictor(model, sizes=[None, (384, 512)])
    with pytest.raises(ValueError):
        ens(torch.zeros(1, 3, 384, 384, requires_grad=True))
    with pytest.raises(_capi.OdbError):
        ens(torch.zeros(1, 3, 384, 384))
    model.train()
    with pytest.raises(ValueError):
        ens(torch.zeros(1, 3, 384, 384))


def test_evaluate_ensemble_flags():
    import evaluate
    base = ["--task", "depth", "--img_path", "x", "--gt_path", "y", "--synthetic_weights"]
    a = evaluate.parse_args([*base, "--ensemble_sizes", "384x512,768x1024", "--flip"])
    assert a.ensemble_sizes == [(384, 512), (768, 1024)] and a.flip
    a = evaluate.parse_args(base)
    assert a.ensemble_sizes is None and not a.flip
    with pytest.raises(SystemExit):
        evaluate.parse_args([*base, "--ensemble_sizes", "384"])


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


def test_ensemble_kernels_compile_without_spills(tmp_path):
    """The ensemble kernels, compiled as the build compiles them (without fast-math): no stack frame, no spills."""
    from omnidata_b200 import build
    assert "ensemble.cu" in build.SOURCES and "ensemble.cu" not in build.FAST_MATH_SOURCES
    found = _ptxas_report("ensemble.cu", tmp_path)
    kernels = {k: v for k, v in found.items() if "ensemble_" in k}
    assert len(kernels) == 8, sorted(found)                 # gram, reduce, solve, normal merge, 4 depth merges
    assert all(v == (0, 0, 0) for v in kernels.values()), kernels
