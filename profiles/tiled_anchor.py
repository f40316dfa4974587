"""Anchored tiled inference (TiledPredictor(anchor=...)) against plain tiled inference, DPT-Hybrid depth model in bf16,
CUDA graphs on, one image per call, tile 384, overlap 64: images/s of the two alternated at 1920x1080, 4032x3024 and
1024x1024, and the per-launch device times of the anchor's kernels (the two resizes, the anchor moments, the anchored
solve, beside the ridge solve).  The card's name and power limit are read in the same run.

    python profiles/tiled_anchor.py [--reps 3] [--iters 5] [--out FILE]
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

# (H, W, anchor): the anchor keeps the image's aspect ratio within the hybrid's limits (W <= 1 792, <= 4 096 patches)
SIZES = [(1080, 1920, (576, 1024)), (3024, 4032, (768, 1024)), (1024, 1024, (1024, 1024))]
TIMED = ("odb_resize_bilinear_f32", "odb_tile_anchor_moments", "odb_tile_align_solve_anchored", "odb_tile_align_solve")


def seconds(fn, x, iters):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn(x)
    torch.cuda.synchronize()
    return time.perf_counter() - t


def launches(p, x):
    """Device time (us) per launch of the anchor's kernels in one eager call (CUDA events around each C-ABI call)."""
    p(x)
    torch.cuda.synchronize()
    with ops.LaunchTimer() as lt:
        p(x)
    agg = defaultdict(list)
    for name, _, ms in lt.results():
        if name in TIMED:
            agg[name[len("odb_"):]].append(round(ms * 1000, 1))
    return dict(agg)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/tiled_anchor.py measures on a CUDA device; none found")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    torch.manual_seed(0)
    m = DPTDepthModel(backbone="vitb_rn50_384").cuda().eval()
    rows = []
    with torch.no_grad():
        for h, w, anchor in SIZES:
            tiled = TiledPredictor(m, tile=(384, 384), overlap=64, max_batch=32)
            anchored = TiledPredictor(m, tile=(384, 384), overlap=64, max_batch=32, anchor=anchor)
            x = torch.rand(1, 3, h, w, device="cuda")
            oy, ox = tile_grid(h, w, (384, 384), 64)
            m.use_cuda_graph = True
            for p in (tiled, anchored):                    # warm up both, graphs captured
                for _ in range(3):
                    p(x)
            r = {"size": f"{w}x{h}", "tiles": len(oy) * len(ox), "anchor": f"{anchor[1]}x{anchor[0]}",
                 "tiled_images_per_s": [], "anchored_images_per_s": []}
            for _ in range(a.reps):                        # the two alternated
                r["tiled_images_per_s"].append(round(a.iters / seconds(tiled, x, a.iters), 2))
                r["anchored_images_per_s"].append(round(a.iters / seconds(anchored, x, a.iters), 2))
            t_ms = 1000 / (sum(r["tiled_images_per_s"]) / a.reps)
            a_ms = 1000 / (sum(r["anchored_images_per_s"]) / a.reps)
            r["tiled_ms"], r["anchored_ms"] = round(t_ms, 2), round(a_ms, 2)
            r["anchor_cost"] = round(a_ms / t_ms - 1, 4)
            m.use_cuda_graph = False
            r["launch_us"] = {**launches(anchored, x), **launches(tiled, x)}
            print(json.dumps(r), flush=True)
            rows.append(r)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps({"card": card, "results": rows}, indent=1))


if __name__ == "__main__":
    main()
