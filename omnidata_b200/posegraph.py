"""Optimise an SE(3) pose graph on the device (csrc/posegraph.cu): camera-to-world poses joined by relative-pose edges,
as loop closure needs them (omnidata_b200/loop.py LoopClosure).

    from omnidata_b200.posegraph import PoseGraph
    poses_out, record = PoseGraph(iterations=10, tol=1e-8).optimize(poses, edges, measurements, information)

poses host float64 [N,4,4] (camera-to-world, checked like every pose here), edges integers [E,2] of pairs (i, j) with
i != j, measurements host float64 [E,4,4] (rigid, Z_ij ~ T_i^-1 T_j), information host float64 [E,6,6] (finite and
exactly symmetric, in the (v, omega) right-increment coordinates of node j: what FrameTracker.information() returns for
a frame j tracked against a model rendered at T_i).  2 <= N <= MAX_NODES (1024) and 1 <= E <= 8 N.  Node 0 is fixed.

Gauss-Newton on sum r^T W r with r = Log(Z^-1 T_i^-1 T_j), increments T <- T exp(delta), first-order Jacobians
(J_r^-1 ~ I), the normal matrix scaled to a unit diagonal and solved by a dense blocked Cholesky in fp64
(DESIGN.md §3 "Loop closure and pose graphs").  Outputs on the device: poses fp64 [N,4,4] and record fp64 [7] =
(status, iterations run, cost at the input poses, cost at the returned poses, largest |delta| of the last step, N, E);
status indexes STATUS.  A failed solve (degenerate: a node no edge reaches, or a scaled pivot below 1e-12; nonfinite:
a NaN, or a residual rotation above pi / 2) returns the input poses bit for bit.  The inputs are checked on the host
and copied to the device once per call; the solve itself neither synchronises nor allocates beyond its outputs after
the first call at a size.  The dense matrix takes 8 (6 (N - 1))^2 bytes: 301 MB at N = 1024.
Definition: include/omnidata_b200.h; oracle/posegraph_oracle.py restates it in float64.
"""
from __future__ import annotations

from typing import Tuple

import torch

from . import _capi, ops
from .losses import _StepBuffers
from .track import _value_error

STATUS = ("ok", "degenerate", "nonfinite")      # record column 0
MAX_NODES = _capi.POSEGRAPH_MAX_NODES


class PoseGraph(_StepBuffers):
    """Gauss-Newton over an SE(3) pose graph (module docstring)."""

    def __init__(self, iterations: int = 10, tol: float = 1e-8, device=None):
        if isinstance(iterations, bool) or not isinstance(iterations, int) or \
                not 1 <= iterations <= ops.POSEGRAPH_MAX_ITERATIONS:
            raise ValueError(f"PoseGraph: iterations must be an integer in [1, {ops.POSEGRAPH_MAX_ITERATIONS}], got "
                             f"{iterations!r}")
        if isinstance(tol, bool) or not (isinstance(tol, (int, float)) and 0 < tol < float("inf")):
            raise ValueError(f"PoseGraph: tol must be finite and > 0, got {tol!r}")
        self.iterations, self.tol = iterations, float(tol)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._bufs = {}

    @torch.no_grad()
    def optimize(self, poses, edges, measurements, information) -> Tuple[torch.Tensor, torch.Tensor]:
        """(poses fp64 [N,4,4], record fp64 [7]) on self.device; kept for the next call at this size, which
        overwrites them."""
        T, E, Z, W = _value_error(ops.check_posegraph, "PoseGraph.optimize", poses, edges, measurements, information)
        n, e = T.shape[0], E.shape[0]
        dev = self.device
        with torch.cuda.device(dev):
            host = torch.from_numpy(T.reshape(-1)), torch.from_numpy(Z.reshape(-1)), torch.from_numpy(W.reshape(-1))
            flat = self._buf("inputs", (16 * n + 16 * e + 36 * e,), torch.float64, dev)
            flat.copy_(torch.cat(host))
            edges_d = self._buf("edges", (e, 2), torch.int32, dev)
            edges_d.copy_(torch.from_numpy(E))
            poses_d = flat[:16 * n].view(n, 4, 4)
            meas_d = flat[16 * n:16 * (n + e)].view(e, 4, 4)
            info_d = flat[16 * (n + e):].view(e, 6, 6)
            ws = self._buf("workspace", (-(-ops.posegraph_workspace_bytes(n, e) // 8),), torch.float64, dev)
            out = self._buf("poses", (n, 4, 4), torch.float64, dev)
            rec = self._buf("record", (_capi.POSEGRAPH_RECORD,), torch.float64, dev)
            ops.posegraph_optimize(edges_d, poses_d, meas_d, info_d, self.iterations, self.tol, ws, out, rec)
        return out, rec
