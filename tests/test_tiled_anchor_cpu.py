"""Anchored tiled inference without a GPU: the float64 oracle of the anchored alignment (oracle/tiled_anchor_oracle.py), the
resize coefficient tables against torch's antialiased bilinear rule, the evaluate.py refusal and the compiler report of
the new kernels (csrc/tiled.cu, csrc/imageproc.cu)."""
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from omnidata_b200 import build
from oracle import tiled_anchor_oracle as A
from oracle import tiled_oracle as O


def _smooth(H, W):
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H, dtype=torch.float64), torch.linspace(0, 1, W, dtype=torch.float64),
                            indexing="ij")
    return 1.5 + torch.sin(3 * xx + 1) * torch.cos(2 * yy) + 0.5 * xx * yy


def _tiles(g, tile, overlap, seed, ramp=0.0):
    """Tiles (g + n_i - t_i) / s_i of g: s_i in [0.5, 2], t_i ~ N(0, 1), n_i = ramp * (r_i x + q_i) an independent
    affine function of the tile's position (0: exact affine maps of g)."""
    H, W = g.shape
    gen = torch.Generator().manual_seed(seed)
    tiles = O.gather(g[None, None].expand(1, 3, H, W), tile, overlap)[:, :1].clone()
    T = tiles.shape[0]
    s = torch.rand(T, generator=gen, dtype=torch.float64) * 1.5 + 0.5
    t = torch.randn(T, generator=gen, dtype=torch.float64)
    if ramp:
        x = torch.linspace(-1, 1, tile[1], dtype=torch.float64)
        r, q = (torch.randn(T, 1, 1, 1, generator=gen, dtype=torch.float64) for _ in range(2))
        tiles = tiles + ramp * (r * x + q)
    return (tiles - t[:, None, None, None]) / s[:, None, None, None]


def _affine_residual(m, g):
    """max |m - (a g + b)| / range(m) for the least-squares a, b: how far m is from any one affine map of g."""
    A = torch.stack([g.flatten(), torch.ones(g.numel(), dtype=torch.float64)], 1)
    coef = torch.linalg.lstsq(A, m.flatten()[:, None]).solution
    return float(((A @ coef).flatten() - m.flatten()).abs().max() / (m.max() - m.min()))


def _rel(m, g):
    return float((m - g).abs().max() / (g.max() - g.min()))


def test_exact_affine_tiles_merge_to_the_anchor():
    """Tiles that are exact affine maps of g, anchored to g: E has a zero at s_i a + t_i = g, so the merge is g up to the
    kappa ridge's pull.  The ridge merge of the same tiles stays far from any one affine map of g."""
    H, W, tile, ov = 200, 300, (64, 96), 16
    g = _smooth(H, W)
    tiles = _tiles(g, tile, ov, seed=H + W)
    err = _rel(A.merge(tiles, g[None], 1, H, W, tile, ov)[0], g)
    ridge = _affine_residual(O.merge(tiles, 1, H, W, tile, ov)[0], g)
    print(f"anchored: {err:.2e} of g's range from g; ridge: {ridge:.2e} from the nearest affine map of g")
    assert err <= 1e-5
    assert 1e-2 <= ridge <= 2e-1


def test_anchor_removes_drift_along_a_strip():
    """A 1 x 30 strip whose tiles carry independent affine noise: the seams cannot agree exactly, and the ridge merge
    drifts along the chain of overlaps.  The anchored merge is closer to g than the ridge merge is to its best affine
    fit of g."""
    H, tile, ov = 64, (64, 64), 16
    W = 30 * (tile[1] - ov) + ov
    oy, ox = O.grid(H, W, tile, ov)
    assert (len(oy), len(ox)) == (1, 30)
    g = _smooth(H, W)
    tiles = _tiles(g, tile, ov, seed=5, ramp=0.01)
    anchored = _rel(A.merge(tiles, g[None], 1, H, W, tile, ov)[0], g)
    ridge = _affine_residual(O.merge(tiles, 1, H, W, tile, ov)[0], g)
    print(f"strip: anchored {anchored:.3e} of g's range from g; ridge {ridge:.3e} from its best affine fit of g")
    assert anchored < ridge


def test_blurred_anchor_does_not_fight_the_seams():
    """With a low-passed anchor, the seam part of E at the anchored solution is no more than 1 % above its value at the
    ridge solution (it is lower here: the ridge bends the tiles of really different scales)."""
    H, W, tile, ov = 200, 300, (64, 96), 16
    g = _smooth(H, W)
    gb = F.avg_pool2d(g[None, None], 31, stride=1, padding=15, count_include_pad=False)[0]
    tiles = _tiles(g, tile, ov, seed=H + W)
    oy, ox = O.grid(H, W, tile, ov)
    m = O.moments(tiles, 1, H, W, tile, ov)
    st_r = O.solve(m, len(oy), len(ox))
    st_a = A.solve(m, A.anchor_moments(tiles, gb, 1, H, W, tile, ov), len(oy), len(ox))
    e_r, e_a = (A.pair_energy(m[0], st[0], len(oy), len(ox)) for st in (st_r, st_a))
    print(f"seam energy: ridge {e_r:.3e}, anchored to a blurred g {e_a:.3e}")
    assert e_a <= 1.01 * e_r


def test_single_tile_is_compute_scale_and_shift():
    gen = torch.Generator().manual_seed(3)
    a = _smooth(64, 96) + 0.05 * torch.randn(64, 96, generator=gen, dtype=torch.float64)
    a = (a - a.mean()) / a.std()                       # well-conditioned: the kappa ridge's pull is ~kappa |(s-1, t)|
    g = _smooth(64, 96) ** 2
    am = A.anchor_moments(a.reshape(1, 1, 64, 96), g[None], 1, 64, 96, (64, 96), 0)
    st = A.solve(torch.zeros(1, 0, 6, dtype=torch.float64), am, 1, 1)
    # compute_scale_and_shift (L/midas_loss.py:10-30) of a against g, directly from the pixels
    n, sa, saa = float(a.numel()), float(a.sum()), float((a * a).sum())
    sg, sag = float(g.sum()), float((a * g).sum())
    det = n * saa - sa * sa
    s, t = (n * sag - sa * sg) / det, (saa * sg - sa * sag) / det
    assert abs(float(st[0, 0, 0]) - s) <= 1e-5 * abs(s) and abs(float(st[0, 0, 1]) - t) <= 1e-5 * max(abs(t), 1.0)


def test_flat_tile_is_finite():
    """All a equal: the anchor term alone is singular in (s, t); the kappa ridge keeps the solve well-posed."""
    g = _smooth(64, 96)
    flat = torch.full((1, 1, 64, 96), 0.5, dtype=torch.float64)
    st = A.solve(torch.zeros(1, 0, 6, dtype=torch.float64), A.anchor_moments(flat, g[None], 1, 64, 96, (64, 96), 0),
                 1, 1)
    assert bool(torch.isfinite(st).all())
    # a flat tile beside textured ones in a grid
    H, W, tile, ov = 100, 300, (64, 96), 16
    oy, ox = O.grid(H, W, tile, ov)
    gg = _smooth(H, W)
    tiles = _tiles(gg, tile, ov, seed=2)
    tiles[1] = 0.5
    out = A.merge(tiles, gg[None], 1, H, W, tile, ov)
    assert bool(torch.isfinite(out).all())


@pytest.mark.parametrize("n_in,n_out", [(200, 100), (370, 100), (590, 100), (37, 111), (64, 64), (4032, 1024),
                                        (3024, 768), (1, 7), (7, 1), (383, 97)])
def test_resize_tables_are_torchs_antialiased_bilinear(n_in, n_out):
    """imageproc.bilinear_aa_weights (Pillow's coefficients before the 8-bit step) applied as a matrix reproduces
    F.interpolate(mode="bilinear", align_corners=False, antialias=True) along one axis in float64."""
    from omnidata_b200.imageproc import bilinear_aa_weights
    bounds, w, ksize = bilinear_aa_weights(n_in, n_out)
    assert bounds.shape == (n_out, 2) and w.shape == (n_out, ksize)
    assert int(bounds[:, 1].max()) <= ksize and int(bounds[:, 0].min()) >= 0
    assert int((bounds[:, 0] + bounds[:, 1]).max()) <= n_in
    M = np.zeros((n_out, n_in))
    for o in range(n_out):
        M[o, bounds[o, 0]:bounds[o, 0] + bounds[o, 1]] = w[o, :bounds[o, 1]]
    x = torch.rand(3, 1, 5, n_in, generator=torch.Generator().manual_seed(n_in), dtype=torch.float64)
    want = F.interpolate(x, size=(5, n_out), mode="bilinear", align_corners=False, antialias=True)
    got = x @ torch.from_numpy(M).T
    assert float((got - want).abs().max()) <= 1e-14
    assert float((A.resize(x, (5, n_out)) - want).abs().max()) == 0.0


def test_evaluate_refuses_anchor_outside_tiled_depth():
    import evaluate
    base = ["--img_path", "x", "--gt_path", "y", "--synthetic_weights", "--anchor", "768x1024"]
    assert evaluate.parse_args(["--task", "depth", *base]).anchor == (768, 1024)
    for extra in (["--task", "depth", "--mode", "direct"], ["--task", "normal"]):
        with pytest.raises(SystemExit):
            evaluate.parse_args([*extra, *base])
    with pytest.raises(SystemExit):
        evaluate.parse_args(["--task", "depth", "--img_path", "x", "--gt_path", "y", "--synthetic_weights",
                             "--anchor", "768"])


def _ptxas_report(src, tmp_path):
    nvcc = build._nvcc()
    cmd = [nvcc, *build.NVCC_FLAGS, *(["--use_fast_math"] if src in build.FAST_MATH_SOURCES else []),
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


def test_anchor_kernels_compile_without_spills(tmp_path):
    """The anchor kernels, compiled as the build compiles their sources (neither with fast-math): no stack frame, no
    spills."""
    assert "tiled.cu" not in build.FAST_MATH_SOURCES and "imageproc.cu" not in build.FAST_MATH_SOURCES
    found = {**_ptxas_report("tiled.cu", tmp_path), **_ptxas_report("imageproc.cu", tmp_path)}
    names = ("tile_anchor_moments_kernel", "tile_align_solve_kernel", "resample_h_f32_kernel", "resample_v_f32_kernel")
    kernels = {k: v for k, v in found.items() if any(n in k for n in names)}
    assert len(kernels) == 4, sorted(found)
    assert all(v == (0, 0, 0) for v in kernels.values()), kernels
