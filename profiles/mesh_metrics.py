"""Mesh metrics on one GPU: `mesh.sample_surface` and `mesh.nearest` at 10^6, 10^7 and 10^8 points per side on the
analytic room's exact mesh (each call timed with a host clock ending in a device synchronise, best of three after a
warm-up; both calls synchronise once themselves), scipy's cKDTree on the same host as a reference at 10^6, and one
`MeshMetrics.update` of a fused room, with the card's name and power limit (`--out FILE` writes the JSON)."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from omnidata_b200 import mesh  # noqa: E402
from oracle import mesh_oracle as MO  # noqa: E402
from oracle import volume_oracle as VO  # noqa: E402

CENTER, RADIUS, LO, HI = (0.03, -0.02, 0.01), 0.5, (-1.5,) * 3, (1.5,) * 3


def _best(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return min(times) * 1e3, out


def _grid_stats(G):
    """The default grid of `nearest` over the reference set G (its box, `mesh.default_cell`): cell size, cells, and
    the occupied cells and mean points per occupied cell (surface samples leave most cells empty)."""
    lo, hi = G.min(0).values.double(), G.max(0).values.double()
    h = mesh.default_cell(lo.tolist(), hi.tolist(), int(G.shape[0]))
    n = torch.floor((hi - lo) / h).long() + 1
    c = torch.minimum(torch.floor((G.double() - lo) / h).long().clamp_min(0), n - 1)
    occupied = int(torch.unique((c[:, 2] * n[1] + c[:, 1]) * n[0] + c[:, 0]).numel())
    return {"cell_m": h, "cells": int(n.prod()), "occupied_cells": occupied,
            "points_per_occupied_cell": round(G.shape[0] / occupied, 1)}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--sizes", default="1e6,1e7,1e8")
    args = ap.parse_args(argv)
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    gv, gf = MO.sphere_room_mesh(CENTER, RADIUS, LO, HI, 6)
    v, f = torch.from_numpy(gv.astype(np.float32)).to(dev), torch.from_numpy(gf.astype(np.int32)).to(dev)
    area = float(MO.face_areas(gv.astype(np.float32), gf).sum())
    res = {"card": card, "sizes": []}
    for n in (float(s) for s in args.sizes.split(",")):
        rho = n / area
        ms_s, P = _best(lambda: mesh.sample_surface(v, f, rho, 0, 0))
        G = mesh.sample_surface(v, f, rho, 0, 1)
        ms_n, (d, _) = _best(lambda: mesh.nearest(P, G))
        row = {"points": int(P.shape[0]), "sample_ms": round(ms_s, 3), "nearest_ms": round(ms_n, 3),
               **_grid_stats(G),
               "mean_distance_mm": float(d.mean()) * 1e3}
        if n <= 1e6:
            from scipy.spatial import cKDTree
            p, g = P.cpu().numpy().astype(np.float64), G.cpu().numpy().astype(np.float64)
            t0 = time.perf_counter()
            cKDTree(g).query(p, k=1, workers=-1)
            row["ckdtree_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)
        del P, G, d
        torch.cuda.empty_cache()
    from omnidata_b200.metrics import MeshMetrics
    from omnidata_b200.volume import SparseTSDFVolume
    K, T = (150.0, 150.0, 79.5, 59.5), VO.orbit_poses(20, 1.2, CENTER)
    depth = np.stack([VO.sphere_room_depth(K, t, (120, 160), CENTER, RADIUS, LO, HI) for t in T])
    vol = SparseTSDFVolume(0.0125, device=dev)
    vol.integrate(torch.from_numpy(depth.astype(np.float32)).to(dev), K, T)
    pv, pf, _ = vol.extract_mesh()
    m = MeshMetrics(thresholds=(0.0125, 0.025, 0.05))
    ms_u, _ = _best(lambda: m.update(pv, pf, v, f, views=(K, (120, 160), T)))
    res["update_fused_room_ms"] = round(ms_u, 3)
    print(json.dumps(res))
    if args.out:
        Path(args.out).write_text(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
