"""The float64 restatement of the fern place recognition (oracle/places_oracle.py) on its own: the invariances the codes
are built for, the rules for empty and flat channels, the top-k tie rule and the fern table's draw."""
import numpy as np
import pytest

from oracle import places_oracle as PO

TABLE = PO.fern_table(500, 0)


def _frame(rng, h=120, w=160):
    """Depth in (0.5, 3.5) m and colours in [0, 1), all multiples of 2^-10, so every cell sum is exact."""
    depth = (rng.integers(512, 3584, (h, w)) / 1024.0).astype(np.float32)
    rgb = (rng.integers(0, 1024, (3, h, w)) / 1024.0).astype(np.float32)
    return depth, rgb


def test_one_pixel_cells_are_the_pixels():
    rng = np.random.default_rng(0)
    depth, rgb = _frame(rng, 60, 80)
    depth[3, 4] = np.nan
    depth[5, 6] = -1.0
    rgb[1, 7, 8] = np.inf
    cells = PO.cell_means(depth, rgb)
    want = np.concatenate([depth.reshape(1, -1), rgb.reshape(3, -1)])
    want[0, 3 * 80 + 4] = want[0, 5 * 80 + 6] = want[2, 7 * 80 + 8] = np.nan
    assert np.array_equal(cells, want, equal_nan=True)


def test_uneven_cells_cover_every_pixel_once():
    h, w = 61, 81
    depth = np.ones((h, w), np.float32)
    rgb = np.zeros((3, h, w), np.float32)
    rgb[0] = np.arange(h * w, dtype=np.float32).reshape(h, w)
    cells = PO.cell_means(depth, rgb)
    counts = np.array([((r + 1) * h // 60 - r * h // 60) * ((c + 1) * w // 80 - c * w // 80)
                       for r in range(60) for c in range(80)])
    assert counts.sum() == h * w and set(counts) == {1, 2, 4}
    assert np.array_equal(cells[0], np.ones(4800, np.float32))


def test_identical_frames_give_distance_zero():
    rng = np.random.default_rng(1)
    depth, rgb = _frame(rng)
    a, b = PO.encode(depth, rgb, TABLE), PO.encode(depth.copy(), rgb.copy(), TABLE)
    assert PO.distances(a[None], b)[0] == 0
    assert 0 < np.count_nonzero(a) < a.size


@pytest.mark.parametrize("scale", [0.25, 2.0, 8.0])
def test_depth_scaled_by_a_power_of_two_gives_the_same_code(scale):
    rng = np.random.default_rng(2)
    depth, rgb = _frame(rng)
    depth[rng.random(depth.shape) < 0.1] = np.nan         # holes: cells of 1 to 4 samples
    assert np.array_equal(PO.encode(depth, rgb, TABLE), PO.encode(depth * np.float32(scale), rgb, TABLE))


def test_colour_gain_and_bias_give_the_same_code():
    rng = np.random.default_rng(3)
    depth, rgb = _frame(rng)
    gain = np.array([2.0, 0.5, 4.0], np.float32)[:, None, None]
    bias = np.array([0.25, -0.125, 1.5], np.float32)[:, None, None]
    rgb2 = rgb * gain + bias
    assert np.array_equal(rgb2 - bias, rgb * gain)              # exact in fp32
    a, b = PO.encode(depth, rgb, TABLE), PO.encode(depth, rgb2, TABLE)
    assert np.array_equal(a, b)
    c = PO.encode(depth, rgb[[1, 0, 2]], TABLE)                 # a colour change is not invariant
    assert PO.distances(a[None], c)[0] > 0


def test_empty_and_flat_channels_give_zero_bits():
    rng = np.random.default_rng(4)
    depth, rgb = _frame(rng)
    depth[:] = np.nan
    rgb[0] = 0.5
    code = PO.encode(depth, rgb, TABLE)
    assert not (code & 1).any() and not (code & 2).any()
    assert (code & 4).any() and (code & 8).any()
    cells = PO.cell_means(depth, rgb)
    m, s = PO.stats(cells)
    assert np.isnan(m[0]) and np.isnan(s[0]) and m[1] == 0.5 and s[1] == 0


def test_lower_median_is_an_order_statistic():
    v = np.array([5, np.nan, 1, 3, 2, np.nan], np.float32)
    assert PO.lower_median(v) == 2                              # rank 1 of (1, 2, 3, 5)
    assert np.isnan(PO.lower_median(np.full(4, np.nan, np.float32)))


def test_query_ties_and_limit():
    rng = np.random.default_rng(5)
    db = rng.integers(0, 2, (40, 6)).astype(np.uint8)           # few ferns: many tied distances
    code = np.zeros(6, np.uint8)
    d = PO.distances(db, code)
    idx, dist = PO.query(db, code, 40, 12)
    pairs = list(zip(dist.tolist(), idx.tolist()))
    assert pairs == sorted(zip(d.tolist(), range(40)))[:12]
    idx, dist = PO.query(db, code, 7, 10)
    assert (idx[7:] == -1).all() and (dist[7:] == -1).all() and sorted(idx[:7].tolist()) == list(range(7))
    idx, dist = PO.query(db, code, 0, 3)
    assert (idx == -1).all() and (dist == -1).all()


def test_fern_table_is_reproducible_from_the_seed():
    from omnidata_b200.places import fern_table
    c0, t0 = PO.fern_table(500, 7)
    c1, t1 = PO.fern_table(500, 7)
    assert np.array_equal(c0, c1) and np.array_equal(t0, t1)
    c2, _ = PO.fern_table(500, 8)
    assert not np.array_equal(c0, c2)
    assert c0.dtype == np.int32 and 0 <= c0.min() and c0.max() < 4800 and np.abs(t0).max() <= 1
    cp, tp = fern_table(500, 7)                                 # the package draws the same table
    assert np.array_equal(cp, c0) and np.array_equal(tp, t0)
