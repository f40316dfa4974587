"""fp8 inference mode against bf16: images/s of the three backbones (CUDA graph on, the two precisions alternated in one
run) and the per-launch times of the ViT blocks' GEMMs and the row-quantise passes, with the card's name and power
limit read in the same run.

    python profiles/fp8.py [--reps 3] [--out FILE]
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

CONFIGS = [(bb, b, s) for bb in ("vitb_rn50_384", "vitb16_384", "vitl16_384") for b, s in ((32, 384), (8, 1024))]


def images_per_s(m, x, iters):
    with torch.no_grad():
        for _ in range(3):
            m(x)
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(iters):
            m(x)
        torch.cuda.synchronize()
    return iters * x.shape[0] / (time.perf_counter() - t)


def launch_times(m, x):
    """Mean time per launch of the ViT layers by (entry point, N, K), one eager forward under LaunchTimer."""
    with torch.no_grad():
        m.use_cuda_graph = False
        m(x)
        torch.cuda.synchronize()
        with ops.LaunchTimer() as lt:
            m(x)
        res = lt.results()
        m.use_cuda_graph = True
    agg = defaultdict(list)
    D = m.arch["embed"]
    rows = x.shape[0] * ((x.shape[2] // 16) * (x.shape[3] // 16) + 1)   # the ViT token rows: not the readout or patch GEMMs
    names = {(3 * D, D): "qkv", (D, D): "proj", (4 * D, D): "fc1", (D, 4 * D): "fc2"}
    for name, info, ms in res:
        if name in ("odb_conv_gemm", "odb_conv_gemm_scaled") and info.get("taps") == 1 and info.get("m") == rows:
            key = names.get((info["n"], info["k"]))
            if key:
                agg[key].append(ms * 1000)
        elif name == "odb_rowquant_e4m3":       # before proj (D columns) and before fc2 (4D columns)
            agg["rowquant_proj_in" if info["cols"] == D else "rowquant_fc2_in"].append(ms * 1000)
    return {k: round(sum(v) / len(v), 2) for k, v in agg.items() if k}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/fp8.py measures on a CUDA device; none found")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    rows = []
    for bb, b, s in CONFIGS:
        torch.manual_seed(0)
        m = DPTDepthModel(backbone=bb).cuda().eval()
        m.use_cuda_graph = True
        x = torch.rand(b, 3, s, s, device="cuda")
        r = {"backbone": bb, "batch": b, "size": s, "bf16": [], "fp8": []}
        for _ in range(a.reps):
            for prec in ("bf16", "fp8"):
                m.precision = prec
                r[prec].append(round(images_per_s(m, x, a.iters), 1))
        for prec in ("bf16", "fp8"):
            m.precision = prec
            r[prec + "_launch_us"] = launch_times(m, x)
        print(json.dumps(r), flush=True)
        rows.append(r)
        del m
        torch.cuda.empty_cache()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps({"card": card, "results": rows}, indent=1))


if __name__ == "__main__":
    main()
