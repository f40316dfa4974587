"""Fern place recognition on the GPU (csrc/places.cu through omnidata_b200/places.py) against oracle/places_oracle.py,
bit for bit.

- Kernels on guarded buffers (oracle/guard.py checked_launch: every output written, nothing else touched, a second run
  bit-identical).  The uint8 codes and int32 lookups are written through integer views of fp32 guarded buffers: codes
  are at most 15 per byte and indices and distances small non-negative integers, so every written word reads as a
  finite fp32 value and an unwritten one keeps its NaN fill.
- Codes at 60x80 (one pixel per cell), 61x81 (uneven cells), 120x160, 480x640 and 968x1296, with NaN holes, all-NaN
  depth and a constant channel; batches of 1, 5 and 17 against frame-by-frame calls.
- Lookups at 1, 2, 1000 and 1e5 entries, with many ties, k above the eligible count and limit 0.
- Argument checks before any launch, and encode + query captured in a CUDA graph."""
import numpy as np
import pytest
import torch

from oracle import places_oracle as PO
from oracle.guard import Guarded, checked_launch

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")
F = 500


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _frames(rng, n, h, w, kind="plain"):
    """n frames: smooth positive depth (a relative prediction's range) with a little noise, and colours in [0, 1]."""
    yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
    depth = np.empty((n, h, w), np.float32)
    rgb = np.empty((n, 3, h, w), np.float32)
    for q in range(n):
        a = rng.uniform(0.5, 3.0, 4)
        depth[q] = a[0] + a[1] * yy + a[2] * np.sin(4 * xx + a[3]) + 0.05 * rng.standard_normal((h, w))
        for c in range(3):
            b = rng.uniform(0, 1, 3)
            rgb[q, c] = np.clip(0.5 + 0.4 * np.sin(6 * b[0] * xx + 5 * b[1] * yy + 6 * b[2]) +
                                0.05 * rng.standard_normal((h, w)), 0, 1)
    if kind == "holes":
        depth[rng.random(depth.shape) < 0.2] = np.nan
        depth[:, : h // 3, : w // 4] = 0.0                          # a block of cells without depth
        rgb[rng.random(rgb.shape) < 0.05] = np.nan
    elif kind == "no_depth":
        depth[:] = np.nan
    elif kind == "constant":
        rgb[:, 1] = 0.25
    return depth, rgb


def _db(ferns=F, seed=0, size=(60, 80)):
    from omnidata_b200.places import FernDatabase
    return FernDatabase(size, ferns=ferns, seed=seed, device=dev)


def _guarded_encode(depth, rgb, db, gen):
    from omnidata_b200 import ops
    n, h, w = depth.shape
    bd, br = Guarded(depth.size, torch.float32, gen), Guarded(rgb.size, torch.float32, gen)
    bt, bc = Guarded(F * 4, torch.float64, gen), Guarded(n * F // 4, torch.float32, gen)
    d, r, t = bd.contiguous(n, h, w), br.contiguous(n, 3, h, w), bt.contiguous(F, 4)
    d.copy_(torch.from_numpy(depth))
    r.copy_(torch.from_numpy(rgb))
    t.copy_(db.thresholds)
    out = bc.contiguous(n * F // 4)
    codes = out.view(torch.uint8).view(n, F)
    ws = torch.empty(-(-ops.fern_encode_workspace_bytes(n) // 8), dtype=torch.float64, device=dev)
    checked_launch([bd, br, bt, bc], [out], lambda: ops.fern_encode(d, r, db.cells, t, codes, ws))
    return codes.cpu().numpy()


@pytest.mark.parametrize("size", [(60, 80), (61, 81), (120, 160), (480, 640), (968, 1296)])
@pytest.mark.parametrize("kind", ["plain", "holes", "no_depth", "constant"])
def test_codes_match_the_oracle(size, kind):
    if size[0] >= 480 and kind in ("no_depth", "constant"):
        pytest.skip("the two empty-channel kinds run at the three smaller sizes")
    rng = np.random.default_rng([size[0], size[1], ["plain", "holes", "no_depth", "constant"].index(kind)])
    db = _db(size=size)
    n = 2
    depth, rgb = _frames(rng, n, *size, kind=kind)
    got = _guarded_encode(depth, rgb, db, torch.Generator(device=dev).manual_seed(1))
    table = (db.cells.cpu().numpy(), db.thresholds.cpu().numpy())
    for q in range(n):
        want = PO.encode(depth[q], rgb[q], table)
        assert np.array_equal(got[q], want), (q, int((got[q] != want).sum()))
    if kind == "no_depth":
        assert not (got & 1).any()
    if kind == "constant":
        assert not (got & 4).any()
    assert (got & 8).any()


def test_batches_match_frame_by_frame():
    rng = np.random.default_rng(11)
    db = _db(size=(120, 160))
    depth, rgb = _frames(rng, 17, 120, 160, kind="holes")
    D, R = torch.from_numpy(depth).to(dev), torch.from_numpy(rgb).to(dev)
    single = np.stack([db.encode(D[q], R[q]).cpu().numpy()[0] for q in range(17)])
    for b in (1, 5, 17):
        got = np.concatenate([db.encode(D[s:s + b].contiguous(), R[s:s + b].contiguous()).cpu().numpy()
                              for s in range(0, 17 - b + 1, b)])
        assert np.array_equal(got, single[:got.shape[0]]), b


def _guarded_query(db_codes, code, limit, k, gen):
    from omnidata_b200 import ops
    n_db, f = db_codes.shape
    assert (n_db * f) % 4 == 0 and f % 4 == 0
    bdb, bq, bo = (Guarded(n_db * f // 4, torch.float32, gen), Guarded(f // 4, torch.float32, gen),
                   Guarded(2 * k, torch.float32, gen))
    dbv = bdb.contiguous(n_db * f // 4).view(torch.uint8).view(n_db, f)
    qv = bq.contiguous(f // 4).view(torch.uint8)
    dbv.copy_(torch.from_numpy(db_codes))
    qv.copy_(torch.from_numpy(code))
    out = bo.contiguous(2, k)
    idx, dist = out[0].view(torch.int32), out[1].view(torch.int32)
    ws = torch.empty(-(-ops.fern_query_workspace_bytes(n_db) // 8), dtype=torch.float64, device=dev)
    checked_launch([bdb, bq, bo], [out], lambda: ops.fern_query(dbv, qv, limit, k, idx, dist, ws))
    return idx.cpu().numpy(), dist.cpu().numpy()


def _plain_query(db_codes, code, limit, k):
    from omnidata_b200 import ops
    dbt, qt = torch.from_numpy(db_codes).to(dev), torch.from_numpy(code).to(dev)
    runs = []
    for _ in range(2):
        idx = torch.full((k,), 12345, dtype=torch.int32, device=dev)
        dist = torch.full((k,), 12345, dtype=torch.int32, device=dev)
        ws = torch.empty(-(-ops.fern_query_workspace_bytes(db_codes.shape[0]) // 8), dtype=torch.float64, device=dev)
        ops.fern_query(dbt, qt, limit, k, idx, dist, ws)
        runs.append((idx.cpu().numpy(), dist.cpu().numpy()))
    assert all(np.array_equal(a, b) for a, b in zip(*runs))
    return runs[0]


@pytest.mark.parametrize("n_db,ferns,limit,k", [
    (1, F, 1, 1), (2, F, 2, 2), (2, F, 1, 1), (1000, F, 1000, 8), (1000, F, 700, 700),
    (100000, F, 100000, 16), (100000, F, 99999, 1024),
    (1000, 8, 1000, 40), (100000, 4, 100000, 1000),                   # few ferns: many ties
])
def test_query_matches_the_oracle(n_db, ferns, limit, k):
    rng = np.random.default_rng(n_db + ferns + k)
    db_codes = rng.integers(0, 16, (n_db, ferns), dtype=np.uint8)
    code = db_codes[n_db // 2].copy() if n_db > 2 else rng.integers(0, 16, ferns, dtype=np.uint8)
    code[: ferns // 3] ^= 1
    got = _guarded_query(db_codes, code, limit, k, torch.Generator(device=dev).manual_seed(2))
    want = PO.query(db_codes, code, limit, k)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("n_db,ferns,limit,k", [(5, F, 3, 10), (1000, 8, 37, 100), (1000, F, 700, 1024), (16, F, 0, 4),
                                                (1, 4, 0, 1)])
def test_query_pads_beyond_the_eligible_entries(n_db, ferns, limit, k):
    rng = np.random.default_rng(n_db * 7 + k)
    db_codes = rng.integers(0, 16, (n_db, ferns), dtype=np.uint8)
    code = rng.integers(0, 16, ferns, dtype=np.uint8)
    got = _plain_query(db_codes, code, limit, k)
    want = PO.query(db_codes, code, limit, k)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert (got[0][limit:] == -1).all()


def test_database_grows_and_queries_its_entries():
    rng = np.random.default_rng(12)
    db = _db(size=(120, 160))
    depth, rgb = _frames(rng, 40, 120, 160)
    D, R = torch.from_numpy(depth).to(dev), torch.from_numpy(rgb).to(dev)
    for q in range(40):
        db.add(db.encode(D[q], R[q]))
    assert db.count == 40 and db._codes.shape[0] == 64
    idx, dist = db.query(db.codes[23], 3)
    assert int(idx[0]) == 23 and int(dist[0]) == 0
    idx, dist = db.query(db.codes[23], 3, limit=20)
    assert (idx.cpu().numpy() < 20).all() and int(dist[0]) > 0
    want = PO.query(db.codes.cpu().numpy(), db.codes[23].cpu().numpy(), 20, 3)
    assert np.array_equal(idx.cpu().numpy(), want[0]) and np.array_equal(dist.cpu().numpy(), want[1])
    assert db.dissimilarity(int(dist[0])) == int(dist[0]) / F


def test_bad_arguments_raise_before_any_launch():
    from omnidata_b200 import _capi
    from omnidata_b200.places import FernDatabase
    db = _db(size=(120, 160))
    good_d = torch.ones(120, 160, device=dev)
    good_r = torch.zeros(3, 120, 160, device=dev)
    db.add(db.encode(good_d, good_r))
    torch.cuda.synchronize()
    before = _capi.launch_count()
    bad = [
        lambda: FernDatabase((59, 80), device=dev),
        lambda: FernDatabase((60, 79), device=dev),
        lambda: FernDatabase((60, 80), ferns=0, device=dev),
        lambda: FernDatabase((60, 80), ferns=5000, device=dev),
        lambda: db.encode(torch.ones(60, 80, device=dev), torch.zeros(3, 60, 80, device=dev)),
        lambda: db.encode(good_d, torch.zeros(3, 120, 161, device=dev)),
        lambda: db.encode(good_d.double(), good_r),
        lambda: db.encode(good_d.t().contiguous().t(), good_r),
        lambda: db.encode(good_d.cpu(), good_r.cpu()),
        lambda: db.add(torch.zeros(F + 1, dtype=torch.uint8, device=dev)),
        lambda: db.add(torch.zeros(F, dtype=torch.int32, device=dev)),
        lambda: db.query(torch.zeros(F, dtype=torch.uint8, device=dev), 0),
        lambda: db.query(torch.zeros(F, dtype=torch.uint8, device=dev), 1025),
        lambda: db.query(torch.zeros(F, dtype=torch.uint8, device=dev), 1, limit=2),
        lambda: db.query(torch.zeros(F, dtype=torch.uint8, device=dev), 1, limit=-1),
        lambda: db.query(torch.zeros(F - 1, dtype=torch.uint8, device=dev), 1),
    ]
    for q, fn in enumerate(bad):
        with pytest.raises(ValueError):
            fn()
        assert _capi.launch_count() == before, q
    from omnidata_b200 import ops
    for n_db in (0, _capi.FERN_MAX_ENTRIES + 1, 2 ** 31 - 1):       # the C ABI refuses them too
        with pytest.raises(_capi.OdbError):
            ops.fern_query_workspace_bytes(n_db)
        assert _capi.lib().odb_fern_query_workspace_bytes(n_db) == -1
    assert _capi.launch_count() == before
    small = PO.cell_means  # the oracle refuses the same sizes
    with pytest.raises(AssertionError):
        small(np.ones((59, 80), np.float32), np.ones((3, 59, 80), np.float32))


def test_encode_and_query_capture_in_a_cuda_graph():
    rng = np.random.default_rng(13)
    db = _db(size=(120, 160))
    depth, rgb = _frames(rng, 9, 120, 160)
    D, R = torch.from_numpy(depth).to(dev), torch.from_numpy(rgb).to(dev)
    for q in range(8):
        db.add(db.encode(D[q], R[q]))
    frame_d, frame_r = D[8].clone(), R[8].clone()
    code = db.encode(frame_d, frame_r)                  # first call at the shape allocates outside the capture
    idx, dist = db.query(code[0], 4)
    want = (code.clone(), idx.clone(), dist.clone())
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        c = db.encode(frame_d, frame_r)
        i, d = db.query(c[0], 4)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        code.zero_()
        idx.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(c, want[0]) and torch.equal(i, want[1]) and torch.equal(d, want[2])
    frame_d.copy_(D[3])                                 # a replay on new input data finds keyframe 3
    frame_r.copy_(R[3])
    g.replay()
    torch.cuda.synchronize()
    assert int(i[0]) == 3 and int(d[0]) == 0
