"""Float64 / numpy restatement of the randomized-fern place recognition of csrc/places.cu (include/omnidata_b200.h
odb_fern_encode, odb_fern_query): the fern table's draw, the 60 x 80 thumbnail's cell means in the kernel's summation
order, the per-channel lower medians, the bit rule, the distance and the top-k tie rule.  The GPU's codes and lookups
match it bit for bit."""
from __future__ import annotations

import numpy as np

GRID = (60, 80)
CELLS = GRID[0] * GRID[1]


def fern_table(n_ferns: int, seed: int):
    """(cells int32 [F] uniform over the 4800 cells, thresholds float64 [F,4] uniform in [-1, 1]) from
    numpy.random.default_rng(seed), cells drawn first."""
    rng = np.random.default_rng(seed)
    cells = rng.integers(0, CELLS, size=n_ferns).astype(np.int32)
    thresholds = rng.uniform(-1.0, 1.0, size=(n_ferns, 4))
    return cells, thresholds


def _mean(samples: np.ndarray) -> np.float32:
    """fp64 round-to-nearest sum in the given order (np.cumsum accumulates left to right), / count, to fp32."""
    if samples.size == 0:
        return np.float32(np.nan)
    return np.float32(np.cumsum(samples.astype(np.float64))[-1] / np.float64(samples.size))


def cell_means(depth: np.ndarray, rgb: np.ndarray) -> np.ndarray:
    """float32 [4, 4800]: each channel's (depth, R, G, B) mean over the usable samples of each cell, row-major pixel
    order; depth [H,W], rgb [3,H,W] float32."""
    h, w = depth.shape
    assert h >= GRID[0] and w >= GRID[1] and rgb.shape == (3, h, w)
    planes = [np.asarray(depth, np.float32)] + [np.asarray(rgb[c], np.float32) for c in range(3)]
    out = np.empty((4, CELLS), np.float32)
    for r in range(GRID[0]):
        y0, y1 = r * h // GRID[0], (r + 1) * h // GRID[0]
        for c in range(GRID[1]):
            x0, x1 = c * w // GRID[1], (c + 1) * w // GRID[1]
            for q, p in enumerate(planes):
                v = p[y0:y1, x0:x1].reshape(-1)
                ok = np.isfinite(v) & (v > 0) if q == 0 else np.isfinite(v)
                out[q, r * GRID[1] + c] = _mean(v[ok])
    return out


def lower_median(v: np.ndarray) -> np.float32:
    """The element of rank floor((n - 1) / 2) of the non-NaN entries (NaN when there are none)."""
    v = v[~np.isnan(v)]
    if v.size == 0:
        return np.float32(np.nan)
    return np.sort(v)[(v.size - 1) // 2]


def stats(cells: np.ndarray):
    """(m, s) float32 [4]: per channel the lower median of the non-NaN cells and of |v - m| (fp32 subtraction)."""
    m = np.empty(4, np.float32)
    s = np.empty(4, np.float32)
    for q in range(4):
        v = cells[q]
        m[q] = lower_median(v)
        with np.errstate(invalid="ignore", over="ignore"):
            s[q] = lower_median(np.abs(v - m[q]))
    return m, s


def codes_from_cells(cells: np.ndarray, table) -> np.ndarray:
    """uint8 [F]: bit c of fern f is (v_c(p_f) - m_c) > theta_f,c s_c in float64; a NaN cell, a channel without
    non-NaN cells or with s = 0 gives 0."""
    fc, th = table
    m, s = stats(cells)
    out = np.zeros(len(fc), np.uint8)
    for q in range(4):
        x = cells[q, fc].astype(np.float64)
        with np.errstate(invalid="ignore"):
            bit = ~np.isnan(x) & (s[q] > 0) & ((x - np.float64(m[q])) > th[:, q] * np.float64(s[q]))
        out |= (bit.astype(np.uint8) << q)
    return out


def encode(depth: np.ndarray, rgb: np.ndarray, table) -> np.ndarray:
    return codes_from_cells(cell_means(depth, rgb), table)


def distances(db: np.ndarray, code: np.ndarray) -> np.ndarray:
    """int64 [n_db]: the number of ferns whose codes differ."""
    return (np.asarray(db) != np.asarray(code)[None, :]).sum(axis=1)


def query(db: np.ndarray, code: np.ndarray, limit: int, k: int):
    """(index, distance) int32 [k]: entries i < limit in (distance, index) order, padded with -1."""
    d = distances(db[:limit], code) if limit else np.zeros(0, np.int64)
    order = np.lexsort((np.arange(limit), d))[:k]
    idx = np.full(k, -1, np.int32)
    dist = np.full(k, -1, np.int32)
    idx[:order.size] = order
    dist[:order.size] = d[order]
    return idx, dist
