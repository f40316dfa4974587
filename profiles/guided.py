"""Guided upsampling (GuidedPredictor) against tiled and anchored tiled inference, DPT-Hybrid depth and normal models in
bf16, CUDA graphs on, batch 1: images/s at 1920x1080 (guided size 576x1024) and 4032x3024 (768x1024), tile 384 overlap
64, the predictors alternated, three repetitions of 5 calls; and, from one eager guided call, the per-launch device
times of the input resize, the coefficient launches and the apply, with the apply's GB/s against 3.35 TB/s (bytes it
must move: 12 B of image read and 4 C B of output written per pixel).  The card's name and power limit are read in the
same run.

    python profiles/guided.py [--reps 3] [--iters 5] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from omnidata_b200 import ops                                      # noqa: E402
from omnidata_b200.guided import GuidedPredictor                   # noqa: E402
from omnidata_b200.model import DPTDepthModel                       # noqa: E402
from omnidata_b200.tiled import TiledPredictor                      # noqa: E402

SHAPES = [(1080, 1920, (576, 1024)), (3024, 4032, (768, 1024))]
HBM = 3.35e12


def seconds(fn, x, iters):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn(x)
    torch.cuda.synchronize()
    return time.perf_counter() - t


def launches(gp, x, c):
    """Per-launch device times (us) of one eager guided call outside the forward, and the apply's GB/s."""
    gp(x)
    torch.cuda.synchronize()
    with ops.LaunchTimer() as lt:
        gp(x)
    res = lt.results()
    out, forward = {}, 0.0
    for name, info, ms in res:
        if name in ("odb_resize_bilinear_f32", "odb_guided_coefficients", "odb_guided_apply"):
            out.setdefault(name[len("odb_"):], []).append(round(ms * 1000, 1))
        else:
            forward += ms
    H, W = x.shape[2:]
    nbytes = (12 + 4 * c) * H * W
    apply_us = out["guided_apply"][0]
    out["forward_launches_us"] = round(forward * 1000, 1)
    out["apply_bytes"] = nbytes
    out["apply_GBps"] = round(nbytes / (apply_us * 1e-6) / 1e9, 1)
    out["apply_share_of_hbm_peak"] = round(nbytes / (apply_us * 1e-6) / HBM, 3)
    out["apply_lower_bound_us"] = round(nbytes / HBM * 1e6, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/guided.py measures on a CUDA device; none found")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    rows = []
    for c, task in ((1, "depth"), (3, "normal")):
        torch.manual_seed(0)
        m = DPTDepthModel(num_channels=c).cuda().eval()
        with torch.no_grad():
            for H, W, size in SHAPES:
                preds = {"guided": GuidedPredictor(m, size=size), "tiled": TiledPredictor(m, tile=(384, 384), overlap=64)}
                if c == 1:
                    preds["tiled_anchor"] = TiledPredictor(m, tile=(384, 384), overlap=64, anchor=size)
                x = torch.rand(1, 3, H, W, device="cuda") * (2 if c == 1 else 1) - (1 if c == 1 else 0)
                m.use_cuda_graph = True
                for p in preds.values():                   # warm up every shape, graphs captured
                    for _ in range(2):
                        p(x)
                r = {"task": task, "size": f"{W}x{H}", "guided_size": f"{size[1]}x{size[0]}", "batch": 1,
                     "images_per_s": {k: [] for k in preds}}
                for _ in range(a.reps):                    # alternated
                    for k, p in preds.items():
                        r["images_per_s"][k].append(round(a.iters / seconds(p, x, a.iters), 2))
                m.use_cuda_graph = False
                m._graphs.clear()
                r["guided_launches"] = launches(preds["guided"], x, c)
                print(json.dumps(r), flush=True)
                rows.append(r)
                del preds
                torch.cuda.empty_cache()
        del m
        torch.cuda.empty_cache()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps({"card": card, "results": rows}, indent=1))


if __name__ == "__main__":
    main()
