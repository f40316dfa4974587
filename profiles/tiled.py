"""Tiled inference (omnidata_b200/tiled.py) with the DPT-Hybrid depth model in bf16, CUDA graphs on: images/s at
1920x1080 and 4032x3024 (tile 384, overlap 64) and at 1024x1024 (tile 384) beside the direct model(x) at 1024x1024;
per-launch times of the four merge kernels, their share of the call, and the gather / blend bandwidth against the
3.35 TB/s HBM3 data-sheet figure.  The card's name and power limit are read in the same run.

    python profiles/tiled.py [--reps 3] [--out FILE]
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
from omnidata_b200.model import DPTDepthModel                       # noqa: E402
from omnidata_b200.tiled import TiledPredictor, tile_grid           # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SIZES = [(1080, 1920, (384, 384)), (3024, 4032, (384, 384)), (1024, 1024, (384, 384))]


def images_per_s(fn, x, iters):
    with torch.no_grad():
        for _ in range(3):
            fn(x)
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(iters):
            fn(x)
        torch.cuda.synchronize()
    return iters * x.shape[0] / (time.perf_counter() - t)


def merge_launches(p, x):
    """Mean device time (us) per launch of the merge kernels in one call, under LaunchTimer (model launches too: their
    sum is the call's device time)."""
    with torch.no_grad():
        p(x)
        torch.cuda.synchronize()
        with ops.LaunchTimer() as lt:
            p(x)
        res = lt.results()
    agg, total = defaultdict(list), 0.0
    for name, _, ms in res:
        total += ms
        if name.startswith("odb_tile_"):
            agg[name[len("odb_"):]].append(ms * 1000)
    return {k: round(sum(v) / len(v), 1) for k, v in agg.items()}, total * 1000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/tiled.py measures on a CUDA device; none found")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    torch.manual_seed(0)
    m = DPTDepthModel(backbone="vitb_rn50_384").cuda().eval()
    m.use_cuda_graph = True
    rows = []
    for h, w, tile in SIZES:
        p = TiledPredictor(m, tile=tile, overlap=64, max_batch=32)
        x = torch.rand(1, 3, h, w, device="cuda")
        oy, ox = tile_grid(h, w, tile, 64)
        r = {"size": f"{w}x{h}", "tile": tile[0], "tiles": len(oy) * len(ox),
             "tiled_images_per_s": [round(images_per_s(p, x, a.iters), 2) for _ in range(a.reps)]}
        if (h, w) == (1024, 1024):
            r["direct_images_per_s"] = [round(images_per_s(m, x, a.iters), 2) for _ in range(a.reps)]
        # the merge kernels' share: their device time over the call's device time, eager (LaunchTimer brackets each call)
        m.use_cuda_graph = False
        launch_us, call_us = merge_launches(p, x)
        m.use_cuda_graph = True
        merge_us = sum(launch_us.values())
        r["merge_launch_us"] = launch_us
        r["merge_share_of_device_time"] = round(merge_us / call_us, 4)
        T, pix = r["tiles"], h * w
        covered = T * min(tile[0], h) * min(tile[1], w)                         # tile pixels inside the image
        gather_bytes = 4 * 3 * (pix + T * tile[0] * tile[1])                    # image read once, tiles written
        blend_bytes = 4 * (covered + pix)                                      # covering tile pixels read, output written
        if "tile_gather" in launch_us:
            r["gather_GBps"] = round(gather_bytes / (launch_us["tile_gather"] * 1e-6) / 1e9, 1)
            r["gather_share_of_hbm"] = round(gather_bytes / (launch_us["tile_gather"] * 1e-6) / HBM_BYTES_PER_S, 3)
        if "tile_blend" in launch_us:
            r["blend_GBps"] = round(blend_bytes / (launch_us["tile_blend"] * 1e-6) / 1e9, 1)
            r["blend_share_of_hbm"] = round(blend_bytes / (launch_us["tile_blend"] * 1e-6) / HBM_BYTES_PER_S, 3)
        print(json.dumps(r), flush=True)
        rows.append(r)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps({"card": card, "results": rows}, indent=1))


if __name__ == "__main__":
    main()
