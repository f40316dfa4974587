"""Sparse metric alignment (SparseDepthAligner): device time of fit + apply at 384x384 batch 32 and 4032x3024 batch 1,
with 200 points per image, 5 % LiDAR-like density and a dense map, grids 1x1 and 16x12, plain least squares and 5 Huber
iterations; and, from a torch.profiler run of the same calls, the mean time of each kernel, with the moments and apply
passes against their HBM byte bound (moments: 8 B per pixel read, pred and sparse; apply: 4 B read and 4 B written)
at 3.35 TB/s.  The card's name and power limit are read in the same run.

    python profiles/sparse_align.py [--iters 20] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from omnidata_b200.sparse import SparseDepthAligner                 # noqa: E402

SHAPES = [(32, 384, 384), (1, 3024, 4032)]
DENSITIES = [("200_points", 200), ("5pct", 0.05), ("dense", 1.0)]
GRIDS = [(1, 1), (16, 12)]
ROBUST = [None, 0.05]
HBM = 3.35e12


def scene(b, h, w, density, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    pred = torch.rand(b, h, w, device="cuda", generator=g) + 0.2
    depth = 2.5 * pred + 0.4
    if isinstance(density, int):
        keys = torch.rand(b, h * w, device="cuda", generator=g)
        take = torch.zeros(b, h * w, dtype=torch.bool, device="cuda")
        take.scatter_(1, keys.topk(density, dim=1).indices, True)
        take = take.view(b, h, w)
    else:
        take = torch.rand(b, h, w, device="cuda", generator=g) < density
    return pred, torch.where(take, depth, torch.zeros_like(depth))


def device_ms(fn, iters):
    fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def kernel_us(fn, iters):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "sparse_" in ev.key:
            name = ev.key.split("(")[0].split("::")[-1]
            out[name] = {"count_per_call": ev.count // iters, "mean_us": round(ev.device_time, 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = []
    for b, h, w in SHAPES:
        for dname, density in DENSITIES:
            pred, sparse = scene(b, h, w, density)
            for grid in GRIDS:
                for robust in ROBUST:
                    al = SparseDepthAligner(grid=grid, robust=robust)
                    nodes, _ = al.fit(pred, sparse)
                    fit_ms = device_ms(lambda: al.fit(pred, sparse), args.iters)
                    apply_ms = device_ms(lambda: al.apply(pred, nodes), args.iters)
                    ks = kernel_us(lambda: al(pred, sparse), 5)
                    px = b * h * w
                    row = {"batch": b, "size": [h, w], "points": dname, "grid": list(grid), "huber": robust,
                           "fit_ms": round(fit_ms, 3), "apply_ms": round(apply_ms, 3), "kernels": ks}
                    if "sparse_moments_kernel" in ks:
                        t = ks["sparse_moments_kernel"]["mean_us"]
                        row["moments_bound_us"] = round(8 * px / HBM * 1e6, 1)
                        row["moments_share_of_hbm"] = round(8 * px / HBM * 1e6 / t, 3)
                    if "sparse_apply_kernel" in ks:
                        t = ks["sparse_apply_kernel"]["mean_us"]
                        row["apply_bound_us"] = round(8 * px / HBM * 1e6, 1)
                        row["apply_share_of_hbm"] = round(8 * px / HBM * 1e6 / t, 3)
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    result = {"gpu": gpu, "rows": rows}
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))
    print(json.dumps({"gpu": gpu}))


if __name__ == "__main__":
    main()
