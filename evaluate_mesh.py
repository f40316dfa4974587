#!/usr/bin/env python
"""Measure a reconstructed mesh against a ground-truth mesh on the device (`MeshMetrics`, DESIGN.md §3 "Mesh metrics"),
for meshes made by any tool:

    python evaluate_mesh.py --pred mesh.ply --gt gt.ply [--pose_path DIR --intrinsics FX,FY,CX,CY --size HxW]
                            [--density 1e4] [--thresholds 0.05,...] [--seed 0]

Both meshes (PLY, binary little-endian or ascii; polygons are fan-triangulated) are sampled at --density points per
m^2; accuracy is the mean distance from the prediction's samples to the truth's, completion the reverse, and precision,
recall and F-score count the samples within each threshold.  With --pose_path (the <stem>.txt camera-to-world poses
reconstruct.py reads and writes) both sample sets are culled to what those cameras see at --intrinsics and --size,
without modelling occlusion.  Prints one JSON line.  Runs on cuda:0; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

import evaluate
import reconstruct


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Accuracy, completion and F-score of a mesh against a ground-truth mesh")
    ap.add_argument("--pred", required=True, help="the reconstructed mesh (PLY)")
    ap.add_argument("--gt", required=True, help="the ground-truth mesh (PLY)")
    ap.add_argument("--pose_path", default=None, help="cull to the cameras of these <stem>.txt poses")
    ap.add_argument("--intrinsics", type=evaluate._intrinsics, default=None, metavar="FX,FY,CX,CY")
    ap.add_argument("--size", type=evaluate._size, default=None, metavar="HxW", help="the cameras' image size")
    ap.add_argument("--density", type=float, default=1e4, help="samples per m^2 (default 1e4, about 1 cm apart)")
    ap.add_argument("--thresholds", type=reconstruct._float_list, default=(0.05,), metavar="T1,...",
                    help="precision / recall distances in metres (1 to 4; default 0.05)")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args(argv)
    if (args.pose_path is None) != (args.intrinsics is None) or (args.pose_path is None) != (args.size is None):
        ap.error("culling needs --pose_path, --intrinsics and --size together")
    return args


def main(argv=None) -> dict:
    from omnidata_b200.metrics import MeshMetrics
    from omnidata_b200.volume import read_ply
    args = parse_args(argv)
    if not torch.cuda.is_available():
        print("evaluate_mesh.py: a CUDA (sm_90a) device is required; this implementation has no CPU path")
        sys.exit(1)
    dev = torch.device("cuda:0")
    metric = MeshMetrics(thresholds=args.thresholds, density=args.density, seed=args.seed)
    pv, pf, _ = read_ply(args.pred)
    gv, gf, _ = read_ply(args.gt)
    views = None
    if args.pose_path is not None:
        files = sorted(Path(args.pose_path).glob("*.txt"))
        if not files:
            raise FileNotFoundError(f"no poses in {args.pose_path}")
        views = (args.intrinsics, args.size, np.stack([reconstruct.load_pose(f) for f in files]))
    t = lambda a: torch.from_numpy(a).to(dev)                  # noqa: E731
    metric.update(t(pv), t(pf), t(gv), t(gf), views=views)
    result = metric.compute()
    print(json.dumps(result))
    return result


if __name__ == "__main__":
    main()
