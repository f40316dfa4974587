"""Test-time ensembles (EnsemblePredictor) with the DPT-Hybrid depth and normal models in bf16, CUDA graphs on: images/s
for K = 1 (the model alone), K = 2 (flip) and K = 6 (three input sizes x flip) at 384^2 batch 32 and 1024^2 batch 8,
the three alternated, with the spread over repeats; and, from one eager call per K > 1, the per-launch device times of
the gram, solve and merge kernels, their share of the call's device time (all library launches) and the merge's GB/s
against 3.35 TB/s.  The card's name and power limit are read in the same run.

    python profiles/ensemble.py [--reps 3] [--iters 5] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
import time
from collections import defaultdict
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from omnidata_b200 import ops                                      # noqa: E402
from omnidata_b200.ensemble import EnsemblePredictor               # noqa: E402
from omnidata_b200.model import DPTDepthModel                       # noqa: E402

# (H, W, batch, the two extra sizes of K = 6): the extra sizes stay within 4 096 patches
SHAPES = [(384, 384, 32, [(320, 320), (448, 448)]), (1024, 1024, 8, [(768, 768), (896, 896)])]
MERGE = ("odb_ensemble_gram", "odb_ensemble_align_solve", "odb_ensemble_merge_depth", "odb_ensemble_merge_normal")
HBM = 3.35e12


def seconds(fn, x, iters):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn(x)
    torch.cuda.synchronize()
    return time.perf_counter() - t


def launches(ens, x):
    """Per-launch device times (us) of the merge kernels in one eager call, their share of the device time of all
    library launches of the call, and the merge's GB/s."""
    ens(x)
    torch.cuda.synchronize()
    with ops.LaunchTimer() as lt:
        ens(x)
    res = lt.results()
    total = sum(ms for _, _, ms in res)
    agg, gbs, mine = defaultdict(list), [], 0.0
    for name, info, ms in res:
        if name in MERGE:
            agg[name[len("odb_"):]].append(round(ms * 1000, 1))
            mine += ms
            if name.startswith("odb_ensemble_merge"):
                gbs.append(round(info["bytes"] / (ms * 1e-3) / 1e9, 1))
    return {"launch_us": dict(agg), "merge_share_of_device_time": round(mine / total, 5),
            "merge_GBps": gbs, "merge_share_of_hbm_peak": [round(g * 1e9 / HBM, 3) for g in gbs]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/ensemble.py measures on a CUDA device; none found")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    rows = []
    for c, task in ((1, "depth"), (3, "normal")):
        torch.manual_seed(0)
        m = DPTDepthModel(num_channels=c).cuda().eval()
        with torch.no_grad():
            for h, w, b, extra in SHAPES:
                ens = {1: EnsemblePredictor(m, flip=False, max_batch=b), 2: EnsemblePredictor(m, flip=True, max_batch=b),
                       6: EnsemblePredictor(m, sizes=[None, *extra], flip=True, max_batch=b)}
                x = torch.rand(b, 3, h, w, device="cuda")
                m.use_cuda_graph = True
                for e in ens.values():                     # warm up every shape, graphs captured
                    for _ in range(2):
                        e(x)
                r = {"task": task, "size": f"{w}x{h}", "batch": b, "k6_sizes": [f"{w}x{h}"] +
                     [f"{q}x{p}" for p, q in extra], "images_per_s": {k: [] for k in ens}}
                for _ in range(a.reps):                    # the three alternated
                    for k, e in ens.items():
                        r["images_per_s"][k].append(round(a.iters * b / seconds(e, x, a.iters), 1))
                m.use_cuda_graph = False
                m._graphs.clear()
                r["kernels"] = {k: launches(ens[k], x) for k in (2, 6)}
                print(json.dumps(r), flush=True)
                rows.append(r)
                torch.cuda.empty_cache()
        del m
        torch.cuda.empty_cache()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps({"card": card, "results": rows}, indent=1))


if __name__ == "__main__":
    main()
