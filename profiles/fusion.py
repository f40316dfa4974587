"""Depth-normal fusion (DepthNormalFusion, default settings) at 384x384 batch 32, 1080x1920 and 3024x4032 on seeded
piecewise-planar scenes with 1 % depth noise: iterations to converge, device time per call, per CG iteration (a call
stopped at the converged count against a call of one iteration) and of a launch sequence after convergence (the
default 1000-iteration call against the one stopped at convergence); from a torch.profiler run, the mean time of the
matvec and update kernels against their HBM byte bound (128 B per pixel and iteration: matvec reads z, p and the four
edge coefficients and writes p and q; update reads x, r, q, p and D^-1 and writes x, r and z) at 3.35 TB/s; and the
launches per iteration.  The card's name and power limit are read in the same run.

    python profiles/fusion.py [--reps 5] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from omnidata_b200 import _capi                                     # noqa: E402
from omnidata_b200.fusion import DepthNormalFusion                  # noqa: E402
from oracle import fusion_oracle as FO                              # noqa: E402

SHAPES = [(32, 384, 384), (1, 1080, 1920), (1, 3024, 4032)]
HBM = 3.35e12
BYTES_PER_PIXEL_ITER = 128


def scene(b, h, w, seed=0):
    f = 0.9 * max(h, w)
    K = (f, f, (w - 1) / 2, (h - 1) / 2)
    rng = np.random.default_rng(seed)
    zs, cs = [], []
    for i in range(b):
        z, c = FO.planes_scene(h, w, K, seed + i)
        zs.append(z + 0.01 * rng.standard_normal((h, w)))
        cs.append(c)
    return (torch.from_numpy(np.stack(zs).astype(np.float32)).cuda(),
            torch.from_numpy(np.stack(cs).astype(np.float32)).cuda(), K)


def device_ms(fn, reps):
    fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def kernel_us(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "fusion_" in ev.key:
            name = ev.key.split("(")[0].split("::")[-1]
            out[name] = {"count": ev.count, "mean_us": round(ev.device_time, 2)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = []
    for b, h, w in SHAPES:
        d, n, K = scene(b, h, w)
        full = DepthNormalFusion()
        _, rec = full.fit(d, n, K)
        rec = rec.cpu()
        iters = int(rec[:, 3].max())
        stopped = DepthNormalFusion(iterations=max(iters, 2))
        one = DepthNormalFusion(iterations=1)
        c0 = _capi.launch_count()
        stopped(d, n, K)
        launches = _capi.launch_count() - c0
        t_full = device_ms(lambda: full(d, n, K), args.reps)
        t_stop = device_ms(lambda: stopped(d, n, K), args.reps)
        t_one = device_ms(lambda: one(d, n, K), args.reps)
        per_iter = (t_stop - t_one) / (max(iters, 2) - 1)
        after = (t_full - t_stop) / (1000 - max(iters, 2))
        ks = kernel_us(lambda: stopped(d, n, K))
        px = b * h * w
        bound_us = BYTES_PER_PIXEL_ITER * px / HBM * 1e6
        cg_us = ks.get("fusion_matvec_kernel", {}).get("mean_us", 0) + ks.get("fusion_update_kernel", {}).get("mean_us", 0)
        row = {"batch": b, "size": [h, w], "status": [int(s) for s in rec[:, 1].unique()],
               "iterations_max": iters, "iterations_mean": float(rec[:, 3].mean()),
               "ms_per_call_default": round(t_full, 3), "ms_per_call_stopped_at_convergence": round(t_stop, 3),
               "ms_per_cg_iteration": round(per_iter, 4), "us_per_iteration_after_convergence": round(1e3 * after, 2),
               "launches_per_call_stopped": launches, "launches_per_iteration": 2,
               "cg_kernels_us_per_iteration": round(cg_us, 2), "cg_bound_us": round(bound_us, 2),
               "cg_share_of_hbm": round(bound_us / cg_us, 3) if cg_us else None, "kernels": ks}
        rows.append(row)
        print(json.dumps(row), flush=True)
    result = {"gpu": gpu, "rows": rows}
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))
    print(json.dumps({"gpu": gpu}))


if __name__ == "__main__":
    main()
