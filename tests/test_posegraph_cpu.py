"""The pose-graph oracle and the host side of the pose graph and loop closure (no GPU needed): the SE(3) logarithm
against scipy and the exponential, the first-order Jacobians against central differences, recovery of a consistent
graph, loop_graph's graphs accepted by the host checks and recovered, the host refusals of ops.check_posegraph, the reconstruct.py --loop_closure rules, and the ptxas check of
csrc/posegraph.cu and csrc/track.cu (no spills or stack frames)."""
import re
import subprocess

import numpy as np
import pytest
import scipy.linalg

from oracle import posegraph_oracle as PG
from oracle import track_oracle as TO


def _twist(rng, theta, v=0.3):
    a = rng.standard_normal(3)
    return np.r_[v * rng.standard_normal(3), a * theta / np.linalg.norm(a)]


@pytest.mark.parametrize("theta", [0.0, 1e-6, 1e-3, 0.0099, 0.01, 0.0101, 0.1, 1.0, np.pi / 2])
def test_log_against_logm_and_round_trips(theta):
    rng = np.random.default_rng(int(theta * 1e6) + 1)
    for _ in range(5):
        xi = _twist(rng, theta)
        T = PG.se3_exp_matrix(xi)
        r, th = PG.se3_log(T)
        L = scipy.linalg.logm(T).real
        want = np.r_[L[:3, 3], L[2, 1], L[0, 2], L[1, 0]]
        assert abs(th - theta) <= 1e-12
        # just above the series threshold, 1 - A / (2 B) loses ~6 digits to cancellation (still 1e-12 absolute)
        assert np.abs(r - want).max() <= 1e-12 and np.abs(r - xi).max() <= 1e-12
        assert np.abs(PG.se3_exp_matrix(r) - T).max() <= 1e-12


def test_jacobians_against_central_differences():
    """Near the optimum (small residuals) the first-order Jacobians match the derivative of r to O(|r|)."""
    rng = np.random.default_rng(1)
    Ti = PG.se3_exp_matrix(_twist(rng, 0.7, 1.0))
    Tj = PG.se3_exp_matrix(_twist(rng, 0.7, 1.0))
    Z = np.linalg.inv(Ti) @ Tj @ PG.se3_exp_matrix(_twist(rng, 1e-4, 1e-4))
    r, Ji, Jj = PG.jacobians(Ti, Tj, Z)
    h = 1e-6
    for which, J in ((0, Ji), (1, Jj)):
        num = np.empty((6, 6))
        for k in range(6):
            e = np.zeros(6)
            e[k] = h
            P = [Ti, Tj]
            Pp, Pm = list(P), list(P)
            Pp[which] = P[which] @ PG.se3_exp_matrix(e)
            Pm[which] = P[which] @ PG.se3_exp_matrix(-e)
            num[:, k] = (PG.residual(*Pp, Z)[0] - PG.residual(*Pm, Z)[0]) / (2 * h)
        assert np.abs(num - J).max() <= 1e-3 * max(1.0, np.abs(J).max()), (which, np.abs(num - J).max())


def test_oracle_recovers_a_consistent_graph():
    rng = np.random.default_rng(2)
    T, E, Z, W = PG.chain_graph(30, rng, loops=6)
    P0 = np.stack([T[0]] + [TO.perturb(t, 0.05, np.radians(3.0), rng) for t in T[1:]])
    P, rec = PG.optimize(P0, E, Z, W, iterations=20)
    assert rec[0] == PG.OK and rec[1] < 20 and np.abs(P - T).max() <= 1e-9
    assert rec[3] < 1e-15 * rec[2]


@pytest.mark.parametrize("kw", [dict(n=2, n_edges=16, reverse=True), dict(n=12, hubs=(0, 5), reverse=True),
                                dict(n=12, star=True), dict(n=65, n_edges=8 * 65, spread=1e6)],
                         ids=["parallel", "hubs", "star", "8N"])
def test_loop_graph_is_accepted_and_recovered(kw):
    """loop_graph's graphs pass the host checks (full, exactly symmetric W), have the asked-for topology, and without
    noise the oracle recovers the truth from perturbed poses."""
    from omnidata_b200 import ops
    rng = np.random.default_rng(7)
    n = kw["n"]
    T, E, Z, W = PG.loop_graph(n, rng, noise=(0.0, 0.0), **{k: v for k, v in kw.items() if k != "n"})
    ops.check_posegraph("t", T, E, Z, W)
    lam = np.linalg.eigvalsh(W)
    spread = kw.get("spread", 1e2)
    assert np.allclose(lam.min(1), 1e3) and np.allclose(lam.max(1), 1e3 * spread)
    assert (np.abs(W[:, :3, 3:]) > 0).all()                    # v-omega coupling
    if "n_edges" in kw:
        assert len(E) == kw["n_edges"]
    if n == 2:
        assert (E == [1, 0]).all(1).sum() == (E == [0, 1]).all(1).sum() == 8
    if kw.get("hubs"):
        for h in kw["hubs"]:
            assert {int(k) for k in E[(E == h).any(1)].reshape(-1)} == set(range(n))
    if kw.get("star"):
        assert len(E) == n - 1 and (E == 0).any(1).all()
    P0 = np.stack([T[0]] + [TO.perturb(t, 0.02, np.radians(1.0), rng) for t in T[1:]])
    P, rec = PG.optimize(P0, E, Z, W, iterations=20)
    assert rec[0] == PG.OK and rec[1] < 20 and np.abs(P - T).max() <= 1e-9


def test_oracle_status_rules():
    rng = np.random.default_rng(3)
    T, E, Z, W = PG.chain_graph(8, rng, loops=2)
    keep = (E != 4).all(1)
    P, rec = PG.optimize(T, E[keep], Z[keep], W[keep])
    assert rec[0] == PG.DEGENERATE and np.array_equal(P, T)
    Z2 = Z.copy()
    Z2[0] = Z2[0] @ PG.se3_exp_matrix([0, 0, 0, 2.0, 0, 0])
    P, rec = PG.optimize(T, E, Z2, W)
    assert rec[0] == PG.NONFINITE and np.array_equal(P, T)


def test_host_refusals():
    from omnidata_b200 import _capi, ops
    rng = np.random.default_rng(4)
    T, E, Z, W = PG.chain_graph(6, rng, loops=1)
    ops.check_posegraph("t", T, E, Z, W)
    bad_z = Z.copy()
    bad_z[1, :3, :3] *= 1.01
    bad_w = W.copy()
    bad_w[0, 1, 2] = 5.0
    nan_w = W.copy()
    nan_w[0, 0, 0] = np.nan
    big = np.stack([np.eye(4)] * (_capi.POSEGRAPH_MAX_NODES + 1))
    cases = [(T, np.r_[E, [[0, 6]]], np.r_[Z, Z[:1]], np.r_[W, W[:1]]),          # index out of range
             (T, np.r_[E, [[-1, 2]]], np.r_[Z, Z[:1]], np.r_[W, W[:1]]),
             (T, np.r_[E, [[2, 2]]], np.r_[Z, Z[:1]], np.r_[W, W[:1]]),           # i = j
             (T[:1], E[:0], Z[:0], W[:0]),                                        # N < 2
             (big, np.array([[0, 1]]), Z[:1], W[:1]),                             # N beyond the limit
             (T, np.tile(E, (10, 1)), np.tile(Z, (10, 1, 1)), np.tile(W, (10, 1, 1))),   # E > 8 N
             (T, E[:0], Z[:0], W[:0]),                                            # E < 1
             (T, E, bad_z, W), (T, E, Z, bad_w), (T, E, Z, nan_w), (T, E, Z[:-1], W),
             (T, E.astype(np.float64), Z, W)]
    for args in cases:
        with pytest.raises(_capi.OdbError):
            ops.check_posegraph("t", *args)


def test_reconstruct_loop_closure_arguments():
    import reconstruct
    base = ["--img_path", "i", "--intrinsics", "500,500,319.5,239.5", "--voxel", "0.02", "--bounds=-1,-1,-1,1,1,1",
            "--out", "m.ply", "--synthetic_weights", "--sparse_path", "s"]
    photo = ["--photometric", "1e-2"]
    assert not reconstruct.parse_args(base).loop_closure
    assert reconstruct.parse_args(base + ["--loop_closure"] + photo).loop_closure
    assert reconstruct.parse_args(base + ["--pose_path", "p", "--track", "--loop_closure"] + photo).loop_closure
    for argv in (base + ["--pose_path", "p", "--loop_closure"] + photo,          # nothing tracked
                 base + ["--loop_closure"]):                                     # geometry-only edges
        with pytest.raises(SystemExit):
            reconstruct.parse_args(argv)


@pytest.mark.parametrize("src", ["posegraph.cu", "track.cu"])
def test_kernels_do_not_spill(tmp_path, src):
    """Compiled as the build compiles them (without fast-math): no stack frame, no spills."""
    from omnidata_b200 import build
    assert src in build.SOURCES and src not in build.FAST_MATH_SOURCES
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / src), "-o",
           str(tmp_path / (src + ".o"))]
    try:
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600).stdout
    except FileNotFoundError:
        pytest.skip("nvcc not available")
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert len(frames) >= (10 if src == "posegraph.cu" else 6), out
    assert all(f == ("0", "0", "0") for f in frames), out
