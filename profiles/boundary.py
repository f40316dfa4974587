"""Depth-boundary errors (BoundaryMetrics): device time of a CUDA-graph-replayed `update` (edges detected in both maps)
at 384x384 batch 32 and 4032x3024 batch 1, three alternated repetitions of 20 replays, and each stage's share of one
eager update's kernel time (torch.profiler, CUDA activity).  Then, reported and not asserted, the DBE of two
upsamplings of a seeded synthetic scene (constant-depth regions, bars 1-3 px wide, an RGB guide coloured by region) at
1080x1920 against its own edges: the depth at 1/4 resolution resized back with ops.resize_bilinear, and the same
low-resolution depth refined with ops.guided_coefficients / ops.guided_apply (radius 4, eps 1e-3).  The card's name and
power limit are read in the same run.

    python profiles/boundary.py [--reps 3] [--iters 20] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from omnidata_b200 import ops                                      # noqa: E402
from omnidata_b200.metrics import BoundaryMetrics                  # noqa: E402

SHAPES = [(32, 384, 384), (1, 3024, 4032)]
STAGES = {"edge_stats_kernel": "statistics", "slab_reduce_kernel": "slab reductions", "smooth_h_kernel": "smoothing",
          "smooth_v_kernel": "smoothing", "sobel_nms_kernel": "sobel + nms", "ccl_merge_kernel": "hysteresis",
          "ccl_resolve_kernel": "hysteresis", "edge_select_kernel": "hysteresis",
          "edt_col_kernel": "distance transform", "edt_row_kernel": "distance transform",
          "chamfer_kernel": "chamfer + fold", "boundary_fold_kernel": "chamfer + fold"}


def scene(b, h, w, seed, regions=16):
    """(depth [b,h,w], guide [b,3,h,w]): Voronoi regions of constant depth, bars 1-3 px wide, region colours."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    yy = torch.arange(h, device="cuda").view(h, 1).float()
    xx = torch.arange(w, device="cuda").view(1, w).float()
    depth = torch.empty(b, h, w, device="cuda")
    guide = torch.empty(b, 3, h, w, device="cuda")
    for i in range(b):
        seeds = torch.rand(regions, 2, generator=g, device="cuda") * torch.tensor([h, w], device="cuda")
        lab = ((yy[None] - seeds[:, 0].view(-1, 1, 1)) ** 2 + (xx[None] - seeds[:, 1].view(-1, 1, 1)) ** 2).argmin(0)
        n = regions
        for k in range(6):                                          # bars 1, 2, 3 px wide, vertical and horizontal
            wd = k % 3 + 1
            at = int(torch.randint(0, (w if k < 3 else h) - wd, (1,), generator=g, device="cuda"))
            if k < 3:
                lab[:, at:at + wd] = n
            else:
                lab[at:at + wd, :] = n
            n += 1
        levels = torch.rand(n, generator=g, device="cuda") * 9.0 + 1.0
        colours = torch.rand(n, 3, generator=g, device="cuda")
        depth[i] = levels[lab]
        guide[i] = colours[lab].permute(2, 0, 1)
    return depth.contiguous(), guide.contiguous()


def graph_ms(fn, iters, reps):
    """Mean device ms per replay of a captured fn, `reps` windows of `iters` replays."""
    fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        graph.replay()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            graph.replay()
        b.record()
        torch.cuda.synchronize()
        out.append(round(a.elapsed_time(b) / iters, 3))
    return out


def stage_shares(fn):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        for k, stage in STAGES.items():
            if k in e.key:
                us[stage] = us.get(stage, 0.0) + e.device_time_total
    total = sum(us.values())
    return {"kernel_us": round(total, 1), "share": {k: round(v / total, 3) for k, v in sorted(us.items())}}


def dbe_of_upsampling(h=1080, w=1920, seed=7):
    depth, guide = scene(1, h, w, seed)
    lo = (h // 4, w // 4)
    d_lo = torch.empty(1, 1, *lo, device="cuda")
    g_lo = torch.empty(1, 3, *lo, device="cuda")
    ops.resize_bilinear(depth[:, None].contiguous(), d_lo)
    ops.resize_bilinear(guide, g_lo)
    bilinear = torch.empty(1, 1, h, w, device="cuda")
    ops.resize_bilinear(d_lo, bilinear)
    coef = torch.empty(1, 4, *lo, device="cuda")
    ws = torch.empty(ops.guided_workspace_bytes(1, 1, *lo) // 8, device="cuda", dtype=torch.float64)
    ops.guided_coefficients(g_lo, d_lo, 4, 1e-3, ws, coef)
    guided = torch.empty(1, 1, h, w, device="cuda")
    ops.guided_apply(guide, coef, guided)
    out = {"scene": f"{w}x{h}, 1/4 resolution {lo[1]}x{lo[0]}"}
    for name, pred in (("bilinear", bilinear), ("guided", guided)):
        m = BoundaryMetrics()
        m.update(pred, depth)
        r = m.compute()
        out[name] = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/boundary.py measures on a CUDA device; none found")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    cases = []
    for b, h, w in SHAPES:
        gt, _ = scene(b, h, w, 1)
        pred = (0.5 * gt.roll(1, dims=2) + 0.3 + 0.02 * torch.randn(gt.shape, device="cuda")).contiguous()
        m = BoundaryMetrics()
        cases.append(((b, h, w), lambda m=m, p=pred, g=gt: m.update(p, g)))
    times = {c[0]: [] for c in cases}
    for _ in range(a.reps):                                         # alternated
        for shape, fn in cases:
            times[shape] += graph_ms(fn, a.iters, 1)
    rows = []
    for shape, fn in cases:
        b, h, w = shape
        r = {"batch": b, "size": f"{w}x{h}", "update_ms": times[shape],
             "ms_per_megapixel": round(min(times[shape]) / (b * h * w / 1e6), 3), **stage_shares(fn)}
        print(json.dumps(r), flush=True)
        rows.append(r)
    dbe = dbe_of_upsampling()
    print(json.dumps(dbe), flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps({"card": card, "results": rows, "dbe": dbe}, indent=1))


if __name__ == "__main__":
    main()
