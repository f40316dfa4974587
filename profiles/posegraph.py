"""Pose-graph solve and loop-closure costs (csrc/posegraph.cu, omnidata_b200/loop.py).

- PoseGraph at N = 16, 64, 256 and 1024 keyframes (a random chain with E ~ 1.2 N edges, oracle/posegraph_oracle.py
  chain_graph): ms per call and per Gauss-Newton iteration with the inputs already on the device (10 iterations, tol
  so small that all run; CUDA events), the Cholesky kernels' share of the device time (torch.profiler, a run of its
  own) and their achieved fp64 rate, n^3 / 3 FLOP per factorisation, against the H100 SXM data sheet's 34 TFLOP/s fp64
  (FMA, not tensor-core) figure.
- Re-fusion: one integrate of 240 frames at 160x120 and 640x480 into 256^3 and 512^3 grids after a reset.
- The per-keyframe overhead of an edge: FrameTracker(affine=False).track plus information() at 160x120 and 640x480.

Prints one JSON line with the card's name, power limit and max SM clock (`--out FILE` also writes it)."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle import posegraph_oracle as PG  # noqa: E402
from oracle import track_oracle as TO  # noqa: E402
from oracle import volume_oracle as VO  # noqa: E402
from profiles.volume import CENTER, HI, LO, RADIUS, _card, _time  # noqa: E402

FP64_PEAK = 34e12          # H100 SXM data sheet, fp64 (non-tensor-core)
CHOLESKY = ("pg_factor_kernel", "pg_trsm_kernel", "pg_trailing_kernel")


def solve(n_nodes, iters=10):
    from omnidata_b200 import ops
    from omnidata_b200.posegraph import PoseGraph
    rng = np.random.default_rng(n_nodes)
    T, E, Z, W = PG.chain_graph(n_nodes, rng, loops=max(1, n_nodes // 5), noise=(0.01, 0.01))
    P0 = np.stack([T[0]] + [TO.perturb(t, 0.02, np.radians(1.0), rng) for t in T[1:]])
    pg = PoseGraph(iterations=iters, tol=1e-300)
    pg.optimize(P0, E, Z, W)
    b, n, e = pg._bufs, len(P0), len(E)
    flat = b["inputs"]
    args = (b["edges"], flat[:16 * n].view(n, 4, 4), flat[16 * n:16 * (n + e)].view(e, 4, 4),
            flat[16 * (n + e):].view(e, 6, 6), iters, 1e-300, b["workspace"], b["poses"], b["record"])
    ms = _time(lambda: ops.posegraph_optimize(*args), 3 if n_nodes >= 1024 else 20)
    assert int(b["record"][1]) == iters and int(b["record"][0]) == 0
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        ops.posegraph_optimize(*args)
        torch.cuda.synchronize()
    total = chol = 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if ev.key.startswith("pg_") or "odb::pg_" in ev.key:
            total += t
            if any(k in ev.key for k in CHOLESKY):
                chol += t
    m = 6 * (n - 1)
    chol_s = chol * 1e-6 / iters
    return {"nodes": n, "edges": e, "unknowns": m, "ms_per_call": round(ms, 3), "ms_per_iteration": round(ms / iters, 3),
            "cholesky_share": round(chol / total, 3) if total else None,
            "cholesky_ms_per_iteration": round(chol_s * 1e3, 3),
            "cholesky_tflops": round(m ** 3 / 3 / chol_s / 1e12, 2) if chol_s else None,
            "cholesky_share_of_fp64_peak": round(m ** 3 / 3 / chol_s / FP64_PEAK, 3) if chol_s else None}


def refusion(size, n):
    from omnidata_b200.volume import TSDFVolume
    h, w = size
    f = 0.8 * w
    K = (f, f, (w - 1) / 2, (h - 1) / 2)
    T = TO.camera_path(240, CENTER, step_deg=1.5)
    depth = torch.from_numpy(np.stack([VO.sphere_room_depth(K, t, size, CENTER, RADIUS, LO, HI)
                                       for t in T[:8]]).astype(np.float32)).cuda().repeat(30, 1, 1).contiguous()
    vol = TSDFVolume((-1.6, -1.6, -1.6), 3.2 / (n - 1), (n, n, n))

    def run():
        vol.reset()
        vol.integrate(depth, K, T)
    return {"size": f"{w}x{h}", "grid": n, "frames": 240, "ms": round(_time(run, 3), 2)}


def edge(size):
    from omnidata_b200.track import FrameTracker
    h, w = size
    f = 0.8 * w
    K = (f, f, (w - 1) / 2, (h - 1) / 2)
    ref = TO.camera_path(1, CENTER)[0]
    cur = TO.perturb(ref, 0.03, np.radians(2.0), np.random.default_rng(0))
    d_ref = torch.from_numpy(VO.sphere_room_depth(K, ref, size, CENTER, RADIUS, LO, HI).astype(np.float32)).cuda()
    d = torch.from_numpy(VO.sphere_room_depth(K, cur, size, CENTER, RADIUS, LO, HI).astype(np.float32)).cuda()
    tr = FrameTracker(affine=False)

    def run():
        tr.track(d, d_ref, K, ref, ref)
        tr.information()
    return {"size": f"{w}x{h}", "ms_per_edge": round(_time(run, 20), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/posegraph.py measures on the GPU"
    name, power, clock = _card()
    res = {"card": name, "power_limit": power, "max_sm_clock": clock,
           "solve": [solve(n) for n in (16, 64, 256, 1024)],
           "refusion": [refusion(s, n) for s in ((120, 160), (480, 640)) for n in (256, 512)],
           "edge_tracking": [edge(s) for s in ((120, 160), (480, 640))]}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
