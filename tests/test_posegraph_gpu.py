"""The pose-graph solve and the tracker's information matrix on the GPU (PoseGraph, ops.posegraph_optimize,
FrameTracker.information; csrc/posegraph.cu, csrc/track.cu).

- Oracle parity (oracle/posegraph_oracle.py) on random chains with loop edges and noisy measurements at N in {2, 11,
  22, 65, 66, 256, 1024}: n = 6 (N - 1) is one panel, crosses the panel edges (126, 384 = 6 * 64, 390) and reaches the
  cap.  One iteration agrees within 1e-10, a full solve within 1e-9 with the same status and iteration count.
- A consistent graph recovered from perturbed poses; a disconnected node; determinism, CUDA-graph replay and the launch
  sequence.
- FrameTracker.information() against the oracle's sum w J J^T of the last step, and the tracker's outputs unchanged."""
import numpy as np
import pytest
import torch

from oracle import posegraph_oracle as PG
from oracle import track_oracle as TO
from oracle import volume_oracle as VO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _graph(n, seed, noise=(0.01, 0.01)):
    rng = np.random.default_rng(seed)
    T, E, Z, W = PG.chain_graph(n, rng, loops=max(1, n // 5) if n > 2 else 0, noise=noise)
    P0 = np.stack([T[0]] + [TO.perturb(t, 0.02, np.radians(1.0), rng) for t in T[1:]])
    return T, P0, E, Z, W


@pytest.mark.parametrize("n", [2, 11, 22, 65, 66, 256, 1024])
def test_matches_the_oracle(n):
    from omnidata_b200.posegraph import PoseGraph
    T, P0, E, Z, W = _graph(n, n)
    for iters in (1, 10):
        out, rec = PoseGraph(iterations=iters).optimize(P0, E, Z, W)
        want, orec = PG.optimize(P0, E, Z, W, iterations=iters)
        got, rec = out.cpu().numpy(), rec.cpu().numpy()
        H, _, _ = PG.linearize(P0, E, Z, W)
        d = np.sqrt(np.diag(H))
        cond = np.linalg.cond(H / np.outer(d, d))
        diff = np.abs(got - want).max()
        print(f"N={n} E={len(E)} iterations={iters}: status {int(rec[0])}, {int(rec[1])} run (oracle "
              f"{int(orec[1])}), cost {rec[2]:.4e} -> {rec[3]:.4e}, pose diff {diff:.2e}, scaled cond {cond:.1e}")
        assert rec[0] == orec[0] == 0 and rec[1] == orec[1]
        assert tuple(rec[5:]) == (n, len(E))
        assert abs(rec[2] - orec[2]) <= 1e-9 * orec[2] and abs(rec[3] - orec[3]) <= 1e-9 * max(orec[2], 1.0)
        assert diff <= (1e-10 if iters == 1 else 1e-9)


def test_consistent_graph_is_recovered():
    from omnidata_b200.posegraph import PoseGraph
    rng = np.random.default_rng(3)
    T, E, Z, W = PG.chain_graph(40, rng, loops=8)
    P0 = np.stack([T[0]] + [TO.perturb(t, 0.05, np.radians(3.0), rng) for t in T[1:]])
    out, rec = PoseGraph(iterations=20).optimize(P0, E, Z, W)
    rec = rec.cpu().numpy()
    err = np.abs(out.cpu().numpy() - T).max()
    print(f"consistent graph: status {int(rec[0])}, {int(rec[1])} iterations, cost {rec[2]:.3e} -> {rec[3]:.3e}, "
          f"largest entry error {err:.2e}")
    assert rec[0] == 0 and err <= 1e-9 and rec[3] < 1e-15 * rec[2]


def test_disconnected_node_is_degenerate():
    from omnidata_b200.posegraph import STATUS, PoseGraph
    T, P0, E, Z, W = _graph(12, 5)
    keep = (E != 7).all(1)                      # node 7 loses its edges
    out, rec = PoseGraph().optimize(P0, E[keep], Z[keep], W[keep])
    rec = rec.cpu().numpy()
    assert STATUS[int(rec[0])] == "degenerate" and rec[1] == 1
    assert torch.equal(out.cpu(), torch.from_numpy(P0))
    assert rec[2] == rec[3]


def test_large_rotation_residual_is_nonfinite():
    from omnidata_b200.posegraph import STATUS, PoseGraph
    T, P0, E, Z, W = _graph(6, 9)
    Z = Z.copy()
    Z[2] = Z[2] @ PG.se3_exp_matrix([0, 0, 0, 0, 2.0, 0])   # a measurement 115 degrees off
    out, rec = PoseGraph().optimize(P0, E, Z, W)
    assert STATUS[int(rec[0].item())] == "nonfinite" and torch.equal(out.cpu(), torch.from_numpy(P0))


def test_determinism_graph_capture_and_launches():
    from omnidata_b200 import _capi
    from omnidata_b200.posegraph import PoseGraph
    T, P0, E, Z, W = _graph(70, 11)
    pg = PoseGraph(iterations=4, tol=1e-30)
    out, rec = (x.clone() for x in pg.optimize(P0, E, Z, W))
    l0 = _capi.launch_count()
    again = pg.optimize(P0, E, Z, W)
    torch.cuda.synchronize()
    P = -(-6 * 69 // 64)
    assert _capi.launch_count() - l0 == 2 + 4 * (4 * P + 2)
    assert torch.equal(out.view(torch.int64), again[0].view(torch.int64))
    assert torch.equal(rec.view(torch.int64), again[1].view(torch.int64))
    # the solve alone in a CUDA graph, after the inputs are on the device
    from omnidata_b200 import ops
    bufs = pg._bufs
    n, e = len(P0), len(E)
    flat = bufs["inputs"]
    args = (bufs["edges"], flat[:16 * n].view(n, 4, 4), flat[16 * n:16 * (n + e)].view(e, 4, 4),
            flat[16 * (n + e):].view(e, 6, 6), 4, 1e-30, bufs["workspace"], bufs["poses"], bufs["record"])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.posegraph_optimize(*args)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.posegraph_optimize(*args)
    bufs["poses"].zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(bufs["poses"].view(torch.int64), out.view(torch.int64))
    assert torch.equal(bufs["record"].view(torch.int64), rec.view(torch.int64))


def test_refusals_before_any_launch():
    from omnidata_b200 import _capi
    from omnidata_b200.posegraph import PoseGraph
    T, P0, E, Z, W = _graph(5, 2)
    pg = PoseGraph()
    n = _capi.launch_count()
    bad_z = Z.copy()
    bad_z[0, 0, 0] = 1.1
    bad_w = W.copy()
    bad_w[0, 0, 1] = 1.0
    for args in ((P0, np.r_[E, [[0, 5]]], np.r_[Z, Z[:1]], np.r_[W, W[:1]]),
                 (P0, np.r_[E, [[3, 3]]], np.r_[Z, Z[:1]], np.r_[W, W[:1]]),
                 (P0, E, bad_z, W), (P0, E, Z, bad_w)):
        with pytest.raises(ValueError):
            pg.optimize(*args)
    assert _capi.launch_count() == n


def _depth(pose, size, k):
    return VO.sphere_room_depth(k, pose, size, CENTER, RADIUS, ROOM_LO, ROOM_HI)


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(dev)


@pytest.mark.parametrize("affine", [False, True])
def test_tracker_information_matches_the_oracle(affine):
    """The normal matrix of the last step: iterations = 1 (linearised at the initial pose) and 3 (at the pose the
    oracle reaches after 2), relative to its largest entry."""
    from omnidata_b200.track import FrameTracker
    h, w = 61, 83
    rng = np.random.default_rng(4 + affine)
    k = (0.9 * w, 0.9 * w, (w - 1) / 2 + 0.3, (h - 1) / 2 - 0.2)
    ref = TO.camera_path(1, CENTER, seed=h)[0]
    truth = TO.perturb(ref, 0.02, np.radians(1.5), rng)
    d_ref = _depth(ref, (h, w), k).astype(np.float32)
    s1, t1 = (1.3, 0.1) if affine else (1.0, 0.0)
    pred = (s1 * _depth(truth, (h, w), k) + t1).astype(np.float32)
    init = (1 / s1 * 1.01, -t1 / s1 + 0.01) if affine else None
    nodes0 = _t(np.array(init), torch.float64).reshape(1, 1, 1, 2) if affine else None
    for iters in (1, 3):
        tr = FrameTracker(affine=affine, iterations=iters, tol=1e-12)
        pose, nodes, rec = tr.track(_t(pred), _t(d_ref), k, ref, init_nodes=nodes0)
        before = [x.clone() for x in (pose, nodes, rec)]
        info = tr.information().cpu().numpy()
        for x, y in zip(before, (pose, nodes, rec)):
            assert torch.equal(x.view(torch.int64), y.view(torch.int64))
        normals = tr._bufs["normals"][0].cpu().numpy()
        T, st = ref.copy(), init if affine else (1.0, 0.0)
        if iters > 1:
            T, st, orec = TO.track(pred, d_ref, k, ref, None, init, affine=affine, iterations=iters - 1,
                                   normals=normals)
            assert orec[1] == 0 and orec[4] == iters - 1
        Rm, tm = TO.relative_pose(ref, T)
        A = TO.associate(pred, d_ref, normals, k, Rm, tm, st[0], st[1], 0.1, 0.02)
        J, wt = A["J"].reshape(-1, 8), A["w"].reshape(-1)
        n = 8 if affine else 6
        H = ((J * wt[:, None]).T @ J)[:n, :n]
        rel = np.abs(info - H).max() / np.abs(H).max()
        print(f"affine={affine} iterations={iters}: information {info.shape}, relative difference {rel:.2e}")
        assert rec[1] == 0 and rec[4] == iters and info.shape == (n, n)
        assert np.array_equal(info, info.T) and rel <= 1e-10
    again = tr.track(_t(pred), _t(d_ref), k, ref, init_nodes=nodes0)
    for x, y in zip(before, again):
        assert torch.equal(x.view(torch.int64), y.view(torch.int64))
