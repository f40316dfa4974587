"""The tracker's information matrix, the pose-graph solve and LoopClosure's bookkeeping against float64 at the frames
and graphs loop closure builds (csrc/track.cu track_information_kernel, csrc/posegraph.cu, omnidata_b200/loop.py;
oracle/track_oracle.py, photometric_oracle.py, posegraph_oracle.py).  test_posegraph_gpu.py compares them on
diagonal-information chains and one small geometric frame; here:

- Information: every tracking geometry of test_geometry_shapes_gpu.py, affine on and off, with and without the
  photometric term, after one iteration and at the defaults (20 iterations, tol 1e-6: the run usually stops early,
  and information() is then the last step that ran).  Against the oracle's sum w J J^T at the pose it reaches after
  k - 1 steps (1e-10 of the largest entry); bit for bit the ordered_sum8 fold of the workspace's chunk partials, so
  exactly the matrix the step factored (its solve reproduces the step the tracker took); bit for bit a run of exactly
  k iterations; and after a tracker was used at another size, a fresh tracker's.
- Pose graph: full SPD information with eigenvalue spreads of 1e2 and 1e6 at N from 2 to 1024, real tracker
  information mixed with LoopClosure's fallback, E = 8 N, parallel and reversed edges, a hub, a star, descending edge
  order, the SE(3) logarithm's series switch and pi / 2 rule on one edge, the pivot rule, a rank-3 leaf, a status
  that turns nonfinite at the third iteration, and the stop rule.  One iteration within 1e-10 and a full solve within
  1e-9 of the oracle, or 3e-15 times the scaled normal matrix's condition number where that is larger.
- LoopClosure on a closed orbit of 96 frames: the graph it hands the solver (Z and W of every edge bit for bit a
  separate tracker's), the solve, the re-posing of every frame, the stored frames across three capacity doublings, and
  the fallback edge of a frame whose odometry fails."""
import math

import numpy as np
import pytest
import torch

from oracle import color_volume_oracle as CO
from oracle import photometric_oracle as PO
from oracle import posegraph_oracle as PG
from oracle import track_oracle as TO
from oracle import volume_oracle as VO
from test_geometry_shapes_gpu import LAMBDA, TRACK_CASES, _tracking_scene

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)
SIZE, F = (120, 160), 150.0
K = (F, F, (SIZE[1] - 1) / 2, (SIZE[0] - 1) / 2)

# The tracker's workspace (csrc/track.cu, the constants after kChunk and odb_track_information): one double holding the
# ticket, the state (kState = 34 doubles), then kPart = 64 partial sums per chunk of kChunk = 2048 pixels.  Columns
# 0..35 are the upper triangle of sum w J J^T, row-major (tri_index), and 36..43 sum w J e.
PART0, PART, CHUNK, GRAD = 1 + 34, 64, 2048, 36


def _tri_index(i, j):
    return i * 8 - i * (i - 1) // 2 + (j - i)


@pytest.fixture(scope="module", autouse=True)
def _setup(lib_built):
    yield


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).to(dev)


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a, np.float64), np.ascontiguousarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def _case_id(case):
    (h, w), c = case
    return f"{h}x{w}" + ("" if c == "room" else f"-{c}")


# ------------------------------------------------------------------------------------------------ tracker information
def _scene(hw, scene, affine):
    return _tracking_scene(hw, affine, np.random.default_rng(hw[0] * 7 + hw[1] + affine), scene)


def _track(scene, affine, lam, iterations=20, tol=1e-6, tracker=None):
    """One FrameTracker call (LoopClosure's defaults unless given): pose, nodes, record, information(), the chunk
    partials of the workspace and the model normals, on the host."""
    from omnidata_b200.track import FrameTracker
    pred, d_ref, rgb, c_ref, k, ref, init = scene
    tr = tracker or FrameTracker(affine=affine, iterations=iterations, tol=tol, photometric=lam)
    nodes0 = _t(np.array(init), torch.float64).reshape(1, 1, 1, 2) if affine else None
    kw = dict(rgb=_t(rgb), ref_rgb=_t(c_ref)) if lam else {}
    pose, nodes, rec = tr.track(_t(pred), _t(d_ref), k, ref, init_nodes=nodes0, **kw)
    info = tr.information().cpu().numpy()
    chunks = -(-pred.size // CHUNK)
    part = tr._bufs["workspace"].cpu().numpy()[PART0:PART0 + chunks * PART].reshape(chunks, PART)
    return dict(pose=pose.cpu().numpy(), nodes=nodes.reshape(2).cpu().numpy(), rec=rec.cpu().numpy(), info=info,
                part=part, normals=tr._bufs["normals"][0].cpu().numpy())


def _oracle_normal(scene, normals, affine, lam, steps):
    """The oracle's (H, g) linearised at the pose (and s, t) it reaches after `steps` iterations."""
    pred, d_ref, rgb, c_ref, k, ref, init = scene
    T, (s, t) = ref, (init if affine else (1.0, 0.0))
    if steps:
        if lam:
            T, (s, t), orec = PO.track(pred, d_ref, k, ref, rgb, c_ref, None, init, affine=affine, iterations=steps,
                                       photometric=lam, normals=normals)
        else:
            T, (s, t), orec = TO.track(pred, d_ref, k, ref, None, init, affine=affine, iterations=steps,
                                       normals=normals)
        assert orec[1] == TO.OK and orec[4] == steps
    Rm, tm = TO.relative_pose(ref, T)
    if lam:
        A = PO.associate(pred, d_ref, normals, k, Rm, tm, s, t, 0.1, 0.02)
        H, g = PO.normal_matrix(A, PO.photometric(A, rgb, PO.intensity_gradient(d_ref, c_ref, normals), k, Rm, 0.1),
                                lam)
    else:
        H, g = TO.normal_matrix(TO.associate(pred, d_ref, normals, k, Rm, tm, s, t, 0.1, 0.02))
    n = 8 if affine else 6
    return H[:n, :n], g[:n]


def _fold(part, n):
    """(H, g) of the chunk partials folded as track.cu folds them."""
    tot = TO.ordered_sum8(part[:, :GRAD + 8])
    H = np.array([[tot[_tri_index(min(p, q), max(p, q))] for q in range(n)] for p in range(n)])
    return H, tot[GRAD:GRAD + n]


@pytest.mark.parametrize("photometric", [False, True], ids=["geometric", "photometric"])
@pytest.mark.parametrize("affine", [True, False], ids=["affine", "metric"])
@pytest.mark.parametrize("hw,scene", TRACK_CASES, ids=[_case_id(c) for c in TRACK_CASES])
def test_information_matches_the_oracle_and_the_fold(hw, scene, affine, photometric):
    h, w = hw
    strip = min(h, w) < 3
    n = 8 if affine else 6
    lam = LAMBDA if photometric else 0.0
    sc = _scene(hw, scene, affine)
    one = _track(sc, affine, lam, iterations=1)
    full = _track(sc, affine, lam)
    k = int(full["rec"][4])
    print(f"information {h}x{w} ({-(-h * w // CHUNK)} chunks, {scene}) affine={affine} photometric={lam}: the "
          f"defaults run {k} of 20 iterations, status {int(full['rec'][1])}")
    for what, r, before in (("1 iteration", one, 0), (f"{k} iterations", full, k - 1)):
        info = r["info"]
        H, _ = _oracle_normal(sc, r["normals"], affine, lam, before)
        big = np.abs(H).max()
        rel = np.abs(info - H).max() / big if big > 0 else np.abs(info).max()
        # the fold: ordered_sum8 of the partials, bit for bit, and exactly symmetric
        Hf, gf = _fold(r["part"], n)
        extra = f", {int(r['rec'][8])} photometric terms" if photometric else ""
        print(f"  {what}: status {int(r['rec'][1])}{extra}, relative difference to the oracle {rel:.2e} (bound "
              f"1e-10), fold bit-identical {_bits_equal(info, Hf)}")
        assert info.shape == (n, n) and rel <= 1e-10
        assert _bits_equal(info, Hf) and _bits_equal(info, info.T)
        if photometric and not strip and hw != (3, 3):
            assert r["rec"][8] > 0                         # the photometric rows are in the matrix
        if int(r["rec"][1]) != TO.OK:
            continue
        # the matrix is the one the step solved: H x = -g reproduces the step from the previous run's state
        d = np.sqrt(np.diag(Hf))
        cond = float(np.linalg.cond(Hf / np.outer(d, d)))
        x = np.linalg.solve(Hf / np.outer(d, d), -gf / d) / d
        if before:
            prev = _track(sc, affine, lam, iterations=before)
            assert prev["rec"][1] == TO.OK and prev["rec"][4] == before
            T0, st0 = prev["pose"], prev["nodes"]
        else:
            T0, st0 = sc[5], np.array(sc[6] if affine else (1.0, 0.0))
        xi, _ = PG.se3_log(PG._pose(*TO.relative_pose(T0, r["pose"])))
        dx = np.abs(xi - x[:6]).max()
        if affine:
            dx = max(dx, np.abs((r["nodes"] - st0) - x[6:]).max())
        bound = max(1e-10, 3e-15 * cond)
        print(f"  {what}: solve of the folded matrix against the step taken {dx:.2e} (bound {bound:.1e}, scaled "
              f"condition {cond:.1e}, |x| {np.abs(x).max():.1e})")
        assert dx <= bound
    if photometric and strip:                             # no Sobel window: exactly the geometric tracker's matrix
        geo = _track(sc, affine, 0.0, iterations=1)
        assert one["rec"][8] == 0 and _bits_equal(one["info"], geo["info"])
    if k < 20:                                            # stopped early: the information of exactly k iterations
        again = _track(sc, affine, lam, iterations=k, tol=1e-300)
        assert again["rec"][4] == k and _bits_equal(again["info"], full["info"])


FULL_SIZE = [c for c in TRACK_CASES if min(c[0]) > 3]


@pytest.mark.parametrize("photometric", [False, True], ids=["geometric", "photometric"])
@pytest.mark.parametrize("affine", [True, False], ids=["affine", "metric"])
def test_early_stop_is_exercised(affine, photometric):
    """LoopClosure's tracker runs the defaults (20 iterations, tol 1e-6); the early-stop comparisons above are not
    vacuous only if some full-size geometry stops before 20."""
    lam = LAMBDA if photometric else 0.0
    ks = {_case_id(c): int(_track(_scene(*c, affine), affine, lam)["rec"][4]) for c in FULL_SIZE}
    print(f"affine={affine} photometric={lam}: iterations run at the defaults {ks}")
    assert min(ks.values()) < 20


@pytest.mark.parametrize("photometric", [False, True], ids=["geometric", "photometric"])
@pytest.mark.parametrize("affine", [True, False], ids=["affine", "metric"])
def test_information_after_another_size(affine, photometric):
    from omnidata_b200.track import FrameTracker
    lam = LAMBDA if photometric else 0.0
    tr = FrameTracker(affine=affine, photometric=lam)
    big = _track(_scene((968, 1296), "room", affine), affine, lam, tracker=tr)
    small = _scene((120, 160), "room", affine)
    reused = _track(small, affine, lam, tracker=tr)
    fresh = _track(small, affine, lam)
    print(f"affine={affine} photometric={lam}: 968x1296 ({int(big['rec'][4])} iterations) then 120x160 "
          f"({int(reused['rec'][4])} iterations, status {int(reused['rec'][1])})")
    assert reused["rec"][1] == TO.OK
    for key in ("info", "pose", "nodes", "rec"):
        assert _bits_equal(reused[key], fresh[key]), key


# ------------------------------------------------------------------------------------------------ pose graph
def _perturbed(T, rng, dist=0.02, angle=np.radians(1.0)):
    return np.stack([T[0]] + [TO.perturb(t, dist, angle, rng) for t in T[1:]])


def _scaled_cond(P, E, Z, W):
    H, _, _ = PG.linearize(P, E, Z, W)
    d = np.diag(H)
    if not np.all(d > 0):
        return math.inf
    d = np.sqrt(d)
    return float(np.linalg.cond(H / np.outer(d, d)))


RATIOS = []                                               # (difference / bound) of every compared solve


def _compare(what, P0, E, Z, W, iterations, tol=1e-8, status=PG.OK, cond=None):
    """PoseGraph against PG.optimize: status, iterations, N, E, both costs and the poses."""
    from omnidata_b200.posegraph import PoseGraph
    out, rec = PoseGraph(iterations=iterations, tol=tol).optimize(P0, E, Z, W)
    got, rec = out.cpu().numpy(), rec.cpu().numpy()
    want, orec = PG.optimize(P0, E, Z, W, iterations=iterations, tol=tol)
    cond = _scaled_cond(P0, E, Z, W) if cond is None else cond
    bound = max(1e-10 if iterations == 1 else 1e-9, 3e-15 * cond)
    diff = float(np.abs(got - want).max())
    n, e = len(P0), len(E)
    lam = np.linalg.eigvalsh(W)
    spread = float((lam.max(1) / np.maximum(lam.min(1), 1e-300)).max())
    RATIOS.append((diff / bound, what, iterations, cond))
    print(f"{what}: N={n} E={e} largest degree {np.bincount(E.reshape(-1), minlength=n).max()}, eigenvalue spread "
          f"{spread:.1e}, iterations={iterations}: status {int(rec[0])} (oracle {int(orec[0])}), {int(rec[1])} run "
          f"(oracle {int(orec[1])}), cost {rec[2]:.4e} -> {rec[3]:.4e}; pose diff {diff:.2e}, bound {bound:.1e}, "
          f"scaled condition {cond:.1e}")
    assert rec[0] == orec[0] == status and rec[1] == orec[1]
    assert tuple(rec[5:]) == (n, e)
    assert abs(rec[2] - orec[2]) <= 1e-9 * orec[2] and abs(rec[3] - orec[3]) <= 1e-9 * max(orec[2], 1.0)
    if status == PG.OK:
        assert diff <= bound
    else:                                                 # a failed solve returns its input bit for bit
        assert _bits_equal(got, P0) and rec[3] == rec[2]
    return got, rec, orec


@pytest.mark.parametrize("spread", [1e2, 1e6], ids=["spread1e2", "spread1e6"])
@pytest.mark.parametrize("n", [2, 11, 33, 65, 66, 256, 1024])
def test_full_information_graphs(n, spread):
    """n = 6 (N - 1) is one panel (N <= 11), crosses the trsm-row and panel edges (33: 192 = three full panels; 65, 66:
    384 and 390) and reaches the cap.  At N = 1024 one and three iterations bound the oracle's time."""
    rng = np.random.default_rng(n + int(spread))
    T, E, Z, W = PG.loop_graph(n, rng, n_edges=n - 1 + max(1, n // 5), spread=spread)
    P0 = _perturbed(T, rng)
    cond = _scaled_cond(P0, E, Z, W)
    for iters in (1, 3 if n == 1024 else 10):
        _compare(f"full W, spread {spread:.0e}", P0, E, Z, W, iters, cond=cond)


@pytest.fixture(scope="module")
def tracker_information():
    """Eight FrameTracker(affine=False, photometric=1e-2).information() matrices at 120x160 on the analytic scene."""
    out = []
    for q in range(8):
        sc = _tracking_scene(SIZE, False, np.random.default_rng(100 + q), "room")
        r = _track(sc, False, LAMBDA)
        assert r["rec"][1] == TO.OK
        out.append(r["info"])
    return np.stack(out)


def test_real_tracker_information(tracker_information):
    from omnidata_b200.loop import FALLBACK_SIGMA
    lam = np.linalg.eigvalsh(tracker_information)
    print(f"tracker information: eigenvalues {lam.min():.2e} .. {lam.max():.2e}, spread per matrix "
          f"{(lam.max(1) / lam.min(1)).min():.1e} .. {(lam.max(1) / lam.min(1)).max():.1e}")
    fallback = np.diag([FALLBACK_SIGMA[0] ** -2] * 3 + [FALLBACK_SIGMA[1] ** -2] * 3)
    rng = np.random.default_rng(40)
    T, E, Z, _ = PG.loop_graph(40, rng, n_edges=39 + 8)
    W = np.stack([fallback if e % 5 == 4 else tracker_information[e % 8] for e in range(len(E))])
    P0 = _perturbed(T, rng)
    cond = _scaled_cond(P0, E, Z, W)
    for iters in (1, 10):
        _compare("tracker information + fallback", P0, E, Z, W, iters, cond=cond)


TOPOLOGIES = {
    "parallel-N2-E16": dict(n=2, n_edges=16, reverse=True),   # 16 edges between 0 and 1, half listed as (1, 0)
    "N65-E520": dict(n=65, n_edges=8 * 65),
    "N1024-E8192": dict(n=1024, n_edges=8 * 1024),
    "hub": dict(n=100, hubs=(50,)),
    "star": dict(n=65, star=True),
    "descending": dict(n=65, n_edges=200, reverse=True),
}


@pytest.mark.parametrize("case", list(TOPOLOGIES))
def test_topologies(case):
    kw = dict(TOPOLOGIES[case])
    n = kw.pop("n")
    rng = np.random.default_rng(len(case) + n)
    T, E, Z, W = PG.loop_graph(n, rng, **kw)
    if case == "parallel-N2-E16":
        assert (E == [1, 0]).all(1).sum() == 8 and (E == [0, 1]).all(1).sum() == 8
    if case == "hub":                                     # node 50 is joined to every other node
        assert {int(k) for k in E[(E == 50).any(1)].reshape(-1)} == set(range(n))
    if case == "star":
        assert (E == 0).any(1).all()                      # every trailing update subtracts zeros
    if case == "descending":                              # every incidence list in the opposite order
        E, Z, W = E[::-1].copy(), Z[::-1].copy(), W[::-1].copy()
    P0 = _perturbed(T, rng)
    cond = _scaled_cond(P0, E, Z, W)
    for iters in ((1, 3) if n == 1024 else (1, 10)):
        _compare(case, P0, E, Z, W, iters, cond=cond)


THETAS = [0.0, 1e-8, 1e-4, 1e-2 * (1 - 1e-9), 1e-2, 1e-2 * (1 + 1e-9), 0.3, 1.5, np.pi / 2 - 1e-9, np.pi / 2 + 1e-9,
          3.0]


@pytest.mark.parametrize("full_w", [False, True], ids=["identity", "full"])
@pytest.mark.parametrize("theta", THETAS)
def test_single_edge_log(theta, full_w):
    """One edge whose residual rotates by theta: the series / closed-form switch at 1e-2 and the pi / 2 rule."""
    from omnidata_b200.posegraph import PoseGraph
    rng = np.random.default_rng(5)
    Z = PG.se3_exp_matrix([0.3, -0.2, 0.5, 0.4, -0.3, 0.2])
    a = rng.standard_normal(3)
    P0 = np.stack([np.eye(4), Z @ PG.se3_exp_matrix(np.r_[0.05, -0.02, 0.03, theta * a / np.linalg.norm(a)])])
    E = np.array([[0, 1]])
    W = PG.full_information(rng)[None] if full_w else np.eye(6)[None]
    r, th, _ = PG.residual(P0[0], P0[1], Z)
    assert abs(th - theta) <= 1e-12                       # the oracle's angle lies on the intended side of 1e-2, pi / 2
    ok = theta < np.pi / 2
    out, rec = PoseGraph(iterations=1).optimize(P0, E, Z[None], W)
    got, rec = out.cpu().numpy(), rec.cpu().numpy()
    want, orec = PG.optimize(P0, E, Z[None], W, iterations=1)
    c = PG.cost(P0, E, Z[None], W)
    diff = float(np.abs(got - want).max())
    print(f"theta {theta!r} (oracle {th!r}), W {'full' if full_w else 'I'}: status {int(rec[0])}, cost {rec[2]:.17e} "
          f"(oracle {c:.17e}, relative {abs(rec[2] - c) / c:.1e}), pose diff {diff:.1e}")
    assert abs(rec[2] - c) <= 1e-13 * c
    assert rec[0] == orec[0] == (PG.OK if ok else PG.NONFINITE) and rec[1] == 1
    if ok:
        assert diff <= 1e-10
    else:
        assert _bits_equal(got, P0) and rec[3] == rec[2]


def test_component_without_node_0_is_degenerate():
    """Nodes 20 and 21 are joined (twice) only to each other: their diagonal is positive, so the pivot rule, in the
    second panel, finds it."""
    rng = np.random.default_rng(21)
    T, _, _, _ = PG.loop_graph(40, rng)
    E = [(k, k + 1) for k in range(39) if not {k, k + 1} & {20, 21}] + [(19, 22), (20, 21), (21, 20)]
    E = np.array(E)
    Z = np.stack([np.linalg.inv(T[i]) @ T[j] for i, j in E])
    Z[:, :3, :3] = [PG._orthonormal(R) for R in Z[:, :3, :3]]
    W = np.stack([PG.full_information(rng) for _ in E])
    P0 = _perturbed(T, rng)
    H, _, _ = PG.linearize(P0, E, Z, W)
    assert (np.diag(H) > 0).all()
    _compare("component without node 0", P0, E, Z, W, 10, status=PG.DEGENERATE, cond=0.0)


def test_rank3_leaf_is_degenerate():
    """Node 11's only edge carries a plane's information (rank 3, positive diagonal)."""
    rng = np.random.default_rng(12)
    T, E, Z, W = PG.loop_graph(12, rng, n_edges=14)
    keep = ~(E == 11).any(1) | (np.arange(len(E)) == 10)  # the chain edge (10, 11) only
    E, Z, W = E[keep], Z[keep], W[keep].copy()
    Q, _ = np.linalg.qr(rng.standard_normal((6, 6)))
    Wp = (Q * np.r_[1e3, 1e4, 1e5, 0.0, 0.0, 0.0]) @ Q.T
    W[(E == 11).any(1)] = (Wp + Wp.T) / 2
    P0 = _perturbed(T, rng)
    H, _, _ = PG.linearize(P0, E, Z, W)
    assert (E == 11).any(1).sum() == 1 and (np.diag(H) > 0).all()
    _compare("rank-3 leaf", P0, E, Z, W, 10, status=PG.DEGENERATE, cond=0.0)


def _late_failure_graph():
    """Seed 0 of this family, found by searching seeds with the oracle: iterations 1 and 2 solve with every residual
    rotation at least 0.17 rad from pi / 2, and at iteration 3 one lies beyond it."""
    rng = np.random.default_rng(0)
    T, E, Z, W = PG.loop_graph(6, rng, n_edges=10, noise=(0.05, 0.5), spread=1e4)
    return _perturbed(T, rng, 0.05, 0.3), E, Z, W


def test_status_turns_nonfinite_at_a_later_iteration():
    P0, E, Z, W = _late_failure_graph()
    P, thetas = P0, []
    for it in range(1, 4):
        thetas.append(np.array([PG.residual(P[i], P[j], Z[k])[1] for k, (i, j) in enumerate(E)]))
        status, P, _ = PG.step(P, E, Z, W)
        assert (status == PG.OK) == (it < 3)
    margin = min(np.abs(t - np.pi / 2).min() for t in thetas)
    print(f"late failure: largest residual rotation per iteration {[round(float(t.max()), 4) for t in thetas]}, "
          f"margin to pi / 2 {margin:.3f}")
    assert margin >= 1e-6 and thetas[-1].max() > np.pi / 2
    _, rec, _ = _compare("late failure", P0, E, Z, W, 10, status=PG.NONFINITE, cond=0.0)
    assert rec[1] == 3


def test_stop_rule():
    """A tol between two iterations' largest |delta| (a factor of 10 on each side) stops where the oracle stops, and
    a tiny tol runs all 100 iterations."""
    rng = np.random.default_rng(33)
    T, E, Z, W = PG.loop_graph(33, rng, n_edges=50, noise=(0.0, 0.0))
    P0 = _perturbed(T, rng)
    P, d = P0, []
    for _ in range(6):
        status, P, dmax = PG.step(P, E, Z, W)
        assert status == PG.OK
        d.append(dmax)
    i = next(q for q in range(5) if d[q] >= 100 * d[q + 1])
    tol = math.sqrt(d[i] * d[i + 1])
    print(f"stop rule: largest |delta| per iteration {['%.1e' % v for v in d]}, tol {tol:.1e}")
    assert min(d[:i + 1]) >= 10 * tol and d[i + 1] <= tol / 10
    _, rec, orec = _compare("stop rule", P0, E, Z, W, 10, tol=tol)
    assert rec[1] == orec[1] == i + 2
    assert abs(rec[4] - orec[4]) <= 1e-6 * orec[4]
    T, E, Z, W = PG.loop_graph(11, rng, n_edges=20)
    _, rec, _ = _compare("100 iterations", _perturbed(T, rng), E, Z, W, 100, tol=1e-300)
    assert rec[1] == 100


def test_largest_ratio_to_the_bound():
    """Summary of the comparisons above (run in file order): the largest measured difference over its bound."""
    if not RATIOS:
        pytest.skip("no pose-graph comparison ran in this session")
    r, what, iters, cond = max(RATIOS)
    print(f"largest pose difference / bound: {r:.2f} ({what}, {iters} iterations, scaled condition {cond:.1e}) over "
          f"{len(RATIOS)} solves")
    assert r <= 1.0


# ------------------------------------------------------------------------------------------------ LoopClosure
def _orbit(n, radius=1.2):
    """n poses on a closed circle around the sphere, looking at it: pose n would be pose 0."""
    c = np.asarray(CENTER)
    return np.stack([VO.look_at(c + np.array([radius * math.cos(p), radius * math.sin(p), 0.1 * math.sin(p)]), c)
                     for p in 2 * np.pi * np.arange(n) / n])


def _frame(T):
    d = VO.sphere_room_depth(K, T, SIZE, CENTER, RADIUS, ROOM_LO, ROOM_HI).astype(np.float32)
    return d, CO.sphere_room_rgb(K, T, SIZE, CENTER, RADIUS, ROOM_LO, ROOM_HI).astype(np.float32)


def test_loop_closure_bookkeeping():
    """96 frames 3.75 degrees apart on a closed orbit with drifting poses: a keyframe every other frame, one loop
    between the last keyframe (frame 94, 16 cm from frame 0) and keyframe 0."""
    from omnidata_b200.loop import FALLBACK_SIGMA, LoopClosure
    from omnidata_b200.track import FrameTracker
    rng = np.random.default_rng(96)
    truth = _orbit(96)
    drift, given = np.eye(4), []
    for T in truth:
        given.append(T @ drift)
        drift = drift @ PG.se3_exp_matrix(np.r_[0.001 * rng.standard_normal(3), 0.001 * rng.standard_normal(3)])
    frames = [_frame(T) for T in truth]
    loop = LoopClosure(K, SIZE, min_gap=10, radius=0.2, photometric=LAMBDA)
    calls, orig = [], loop.graph.optimize

    def spy(poses, edges, Z, W):
        out, rec = orig(poses, edges, Z, W)
        calls.append([np.array(a, copy=True) for a in (poses, edges, Z, W)] + [out.cpu().numpy(), rec.cpu().numpy()])
        return out, rec

    loop.graph.optimize = spy
    closed_at, before, after = [], None, None
    for q, (T, (d, c)) in enumerate(zip(given, frames)):
        if loop.add(_t(d), T, rgb=_t(c)):
            closed_at.append(q)
            before, after = np.stack(given[:q + 1]), loop.poses
    kfs = loop.keyframes
    print(f"loop closure: {loop.frames} frames, {len(kfs)} keyframes, capacity {loop._metres.shape[0]}, loops "
          f"{loop.loops} closed at frames {closed_at}, {len(calls)} solves")
    assert closed_at == [94] and len(calls) == 1 and loop._metres.shape[0] == 128
    # the stored frames survive the doublings 16 -> 32 -> 64 -> 128
    assert torch.equal(loop._metres[:96].cpu(), torch.from_numpy(np.stack([d for d, _ in frames])))
    assert torch.equal(loop._rgb[:96].cpu(), torch.from_numpy(np.stack([c for _, c in frames])))
    # the graph handed to the solver: every edge's Z and W from a separate tracker on the stored frames
    P, E, Z, W, out, rec = calls[0]
    kf_old = P
    assert _bits_equal(P, before[kfs[:len(P)]]) and len(P) == len(kfs)
    tr = FrameTracker(affine=False, photometric=LAMBDA)
    n_fallback = 0
    for e, (i, j) in enumerate(E):
        fi, fj = kfs[i], kfs[j]
        pose, _, r = tr.track(_t(frames[fj][0]), _t(frames[fi][0]), K, kf_old[i], kf_old[j], rgb=_t(frames[fj][1]),
                              ref_rgb=_t(frames[fi][1]))
        if int(r[1].item()) == 0:
            want_z, want_w = np.linalg.inv(kf_old[i]) @ pose.cpu().numpy(), tr.information().cpu().numpy()
        else:
            assert j == i + 1                             # only an odometry edge falls back
            n_fallback += 1
            want_z = np.linalg.inv(kf_old[i]) @ kf_old[j]
            want_w = np.diag([FALLBACK_SIGMA[0] ** -2] * 3 + [FALLBACK_SIGMA[1] ** -2] * 3)
        assert _bits_equal(Z[e], want_z) and _bits_equal(W[e], want_w), (e, i, j)
    loops = [(int(i), int(j)) for i, j in E if j != i + 1]
    print(f"  {len(E)} edges: {len(E) - len(loops)} odometry ({n_fallback} fallback), loop edges {loops}")
    assert loops == [(0, len(kfs) - 1)] and [(int(i), int(j)) for i, j in E[:len(kfs) - 1]] == \
        [(k, k + 1) for k in range(len(kfs) - 1)]
    # the solve on exactly these inputs
    want, orec = PG.optimize(P, E, Z, W)
    diff = float(np.abs(out - want).max())
    print(f"  solve: status {int(rec[0])}, {int(rec[1])} iterations (oracle {int(orec[1])}), cost {rec[2]:.3e} -> "
          f"{rec[3]:.3e}, pose diff {diff:.2e}")
    assert rec[0] == orec[0] == PG.OK and rec[1] == orec[1] and diff <= 1e-9
    # every frame moves with its keyframe: T_kf,new T_kf,old^-1 T_frame,old
    kf_of = np.searchsorted(np.asarray(kfs), np.arange(95), side="right") - 1
    expect = np.stack([out[a] @ np.linalg.inv(kf_old[a]) @ before[q] for q, a in enumerate(kf_of)])
    repose = float(np.abs(after - expect).max())
    print(f"  re-posing: largest difference {repose:.1e}, largest move {np.abs(after - before).max():.2e}")
    assert after.shape == (95, 4, 4) and repose <= 1e-12
    assert np.abs(after - before).max() > 1e-3           # the closure moved the frames


def test_failed_odometry_gets_the_fallback_edge():
    from omnidata_b200.loop import FALLBACK_SIGMA, LoopClosure
    T = _orbit(96)
    d0, c0 = _frame(T[0])
    _, c2 = _frame(T[2])
    loop = LoopClosure(K, SIZE, photometric=LAMBDA)
    assert not loop.add(_t(d0), T[0], rgb=_t(c0))
    assert not loop.add(_t(np.full(SIZE, np.nan, np.float32)), T[2], rgb=_t(c2))
    assert loop.keyframes == [0, 1] and loop._edges == [(0, 1)]
    W = loop._W[0]
    print(f"fallback edge: W diagonal {np.diag(W)}")
    assert _bits_equal(loop._Z[0], np.linalg.inv(T[0]) @ T[2])
    assert FALLBACK_SIGMA == (0.01, math.radians(0.5))
    assert _bits_equal(W, np.diag([0.01 ** -2] * 3 + [math.radians(0.5) ** -2] * 3))
