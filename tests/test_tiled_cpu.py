"""Tiled inference without a GPU: the tile grid, the float64 merge oracle (oracle/tiled_oracle.py) and the compiler report
of the merge kernels (csrc/tiled.cu)."""
import re
import subprocess

import pytest
import torch

from omnidata_b200 import build
from omnidata_b200.tiled import tile_grid
from oracle import tiled_oracle as O

SIZES = [1, 31, 64, 299, 300, 383, 384, 385, 448, 500, 767, 1024, 1080, 1920, 3024, 4032, 9999]


@pytest.mark.parametrize("tile,overlap", [(384, 64), (384, 0), (512, 64), (64, 31), (96, 1)])
def test_tile_grid_covers_in_bounds_with_overlap(tile, overlap):
    for L in SIZES:
        o, _ = tile_grid(L, 1, (tile, 32), overlap)
        v = overlap
        assert o == O.axis_origins(L, tile, v), L                      # the oracle's exact-rational restatement
        if L <= tile:
            assert o == [0]
            continue
        assert o[0] == 0 and o[-1] == L - tile                          # in bounds, the last tile at the far edge
        assert all(0 <= a < b <= L - tile for a, b in zip(o, o[1:]))
        assert all(b - a <= tile - v for a, b in zip(o, o[1:]))         # neighbours overlap by at least v
        covered = torch.zeros(L, dtype=torch.bool)
        for a in o:
            covered[a:a + tile] = True
        assert bool(covered.all())


def test_tile_grid_counts():
    assert tuple(map(len, tile_grid(3024, 4032, (384, 384), 64))) == (10, 13)       # 130 tiles
    assert tuple(map(len, tile_grid(1080, 1920, (384, 384), 64))) == (4, 6)
    assert tuple(map(len, tile_grid(300, 500, (384, 384), 64))) == (1, 2)
    assert tile_grid(384, 384, (384, 384), 64) == ([0], [0])


def _smooth(H, W):
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H, dtype=torch.float64), torch.linspace(0, 1, W, dtype=torch.float64),
                            indexing="ij")
    return 1.5 + torch.sin(3 * xx + 1) * torch.cos(2 * yy) + 0.5 * xx * yy


def _affine_tiles(g, tile, overlap, seed):
    H, W = g.shape
    gen = torch.Generator().manual_seed(seed)
    tiles = O.gather(g[None, None].expand(1, 3, H, W), tile, overlap)[:, :1].clone()
    T = tiles.shape[0]
    s = torch.rand(T, generator=gen, dtype=torch.float64) * 1.5 + 0.5
    t = torch.randn(T, generator=gen, dtype=torch.float64)
    return (tiles - t[:, None, None, None]) / s[:, None, None, None]


def _affine_residual(m, g):
    A = torch.stack([g.flatten(), torch.ones(g.numel(), dtype=torch.float64)], 1)
    coef = torch.linalg.lstsq(A, m.flatten()[:, None]).solution
    return float(((A @ coef).flatten() - m.flatten()).abs().max() / (m.max() - m.min()))


@pytest.mark.parametrize("H,W,tile,overlap", [(200, 300, (64, 96), 16), (150, 97, (64, 64), 8), (64, 256, (64, 64), 20)])
def test_oracle_merge_of_affine_tiles_is_one_affine_map(H, W, tile, overlap):
    """Tiles (g - t_i) / s_i of one smooth map g merge into one affine map of g.  The ridge lam Nbar sum((s-1)^2 + t^2)
    pulls each tile towards s = 1, t = 0 and so bends the result by O(lam): in the limit of a small ridge the merge is
    affine in g to 1e-10 (and the residual shrinks in proportion to lam)."""
    g = _smooth(H, W)
    tiles = _affine_tiles(g, tile, overlap, seed=H + W)
    small = _affine_residual(O.merge(tiles, 1, H, W, tile, overlap, lam=1e-13)[0], g)
    assert small <= 1e-10, small
    r6, r9 = (_affine_residual(O.merge(tiles, 1, H, W, tile, overlap, lam=lam)[0], g) for lam in (1e-6, 1e-9))
    assert 300 < r6 / r9 < 3000, (r6, r9)


def test_oracle_constant_tiles_blend_to_the_constant():
    H, W, tile, ov = 150, 230, (64, 96), 20
    oy, ox = O.grid(H, W, tile, ov)
    pred = torch.full((2 * len(oy) * len(ox), 1, *tile), 0.375, dtype=torch.float64)
    assert torch.allclose(O.merge(pred, 2, H, W, tile, ov), torch.full((2, H, W), 0.375, dtype=torch.float64),
                          rtol=0, atol=1e-12)
    pred3 = torch.full((len(oy) * len(ox), 3, *tile), -1.25, dtype=torch.float64)
    assert torch.allclose(O.merge(pred3, 1, H, W, tile, ov), torch.full((1, 3, H, W), -1.25, dtype=torch.float64),
                          rtol=0, atol=1e-14)


def test_oracle_single_tile_and_flat_overlaps_are_well_posed():
    st = O.solve(torch.zeros(1, 0, 6, dtype=torch.float64), 1, 1)
    assert torch.allclose(st, torch.tensor([[[1.0, 0.0]]], dtype=torch.float64), rtol=0, atol=1e-15)
    H, W, tile, ov = 100, 300, (64, 96), 16
    oy, ox = O.grid(H, W, tile, ov)
    pred = torch.zeros(len(oy) * len(ox), 1, *tile, dtype=torch.float64)      # all-zero overlaps: s = 1, t = 0
    st = O.solve(O.moments(pred, 1, H, W, tile, ov), len(oy), len(ox))
    assert torch.allclose(st[..., 0], torch.ones_like(st[..., 0]), rtol=0, atol=1e-12)
    assert float(st[..., 1].abs().max()) <= 1e-12


def test_oracle_weights_positive_and_border_tiles_do_not_fade():
    for L, t, v in [(1000, 384, 64), (300, 384, 64), (385, 384, 64), (700, 256, 0)]:
        r = O.ramp(L, t, v)
        assert float(r.min()) >= 1.0 / (v + 1) - 1e-15
        assert float(r[0, 0]) == 1.0 and float(r[-1, min(t, L) - 1]) == 1.0


def test_merge_kernels_compile_without_spills(tmp_path):
    """The four merge kernels, compiled as the build compiles tiled.cu: registers stay out of local memory."""
    nvcc = build._nvcc()
    cmd = [nvcc, *build.NVCC_FLAGS, *(["--use_fast_math"] if "tiled.cu" in build.FAST_MATH_SOURCES else []),
           "-Xptxas", "-v", "-c", str(build.CSRC / "tiled.cu"), "-o", str(tmp_path / "tiled.o")]
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
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    names = ("tile_gather_kernel", "tile_moments_kernel", "tile_align_solve_kernel", "tile_blend_kernel")
    kernels = {k: v for k, v in found.items() if any(n in k for n in names)}
    assert len(kernels) == 4, sorted(found)
    assert all(v == (0, 0) for v in kernels.values()), kernels
