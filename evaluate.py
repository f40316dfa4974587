#!/usr/bin/env python
"""Evaluate a depth or surface-normal model over a directory of images and ground truth:

    python evaluate.py --task {depth,normal} --img_path DIR --gt_path DIR [--mask_path DIR]
                       [--checkpoint CKPT | --synthetic_weights] [--backbone ...] [--precision {fp32,bf16,fp8}]
                       [--mode {tiled,direct,guided}] [--tile 384 --overlap 64] [--anchor HxW]
                       [--guided_size HxW [--radius R] [--eps E]] [--ensemble_sizes HxW,... --flip]
                       [--space {depth,disparity}] [--min_depth] [--max_depth] [--depth_scale] [--depth_invalid]
                       [--boundary [--edge_path DIR]]

Images (PNG / JPEG) are matched to ground truth, and to masks, by file stem.  Preprocessing is that of
`demo.py --full_res` (RGB in [0, 1]; depth normalised to [-1, 1]).  `--mode tiled` predicts at the image's own size with
`TiledPredictor`; `--mode direct` runs `model(x)` at the image's own size and refuses, naming the file, a size the forward
does not take.  `--anchor HxW` (depth, `--mode tiled` only) fits the tiles to a whole-image forward at H x W
(`TiledPredictor(anchor=...)`).  `--mode guided --guided_size HxW` runs one forward at H x W and upsamples it with the
image as the guide (`GuidedPredictor`, radius `--radius`, ridge `--eps`).  `--ensemble_sizes` and `--flip` wrap the
direct, tiled or guided predictor in an
`EnsemblePredictor`: one member per listed size (`native`: the image's own) and, with `--flip`, its mirror; `--flip`
alone ensembles the image with its mirror at its own size.  Predictions are clamped to [0, 1] (demo.py, the training step) and evaluated at the ground truth's
resolution, which must equal the image's: nothing is resampled.

Ground truth: `.npy` float (depth in metres [H,W]; normals in [0, 1], [3,H,W] or [H,W,3]); depth as a 16-bit PNG,
depth = value / --depth_scale with --depth_invalid marking no depth (defaults 512 and 65535: our reading of the Omnidata
starter dataset's depth_zbuffer files; check them against a real file before relying on them); normals as an 8-bit RGB
PNG / 255.  Masks: 8-bit PNG or `.npy`, nonzero = valid.  `--boundary` (depth) adds the depth-boundary errors
(`BoundaryMetrics`, under the `boundary` key) against ground-truth edge maps from `--edge_path` (8-bit PNG or `.npy`,
nonzero = edge, matched by file stem) or, without it, edges detected in the ground-truth depth.  Prints one JSON line: the metrics (omnidata_b200.metrics),
the mode, precision, tile settings and the number of images.  Runs on cuda:0; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch
from PIL import Image

IMAGE_EXT = (".png", ".jpg", ".jpeg")


def _find(directory: str, stem: str, what: str) -> Path:
    for ext in (".npy", ".png"):
        p = Path(directory) / (stem + ext)
        if p.exists():
            return p
    raise FileNotFoundError(f"no {what} for {stem!r} in {directory} (expected {stem}.npy or {stem}.png)")


def load_gt(path: Path, task: str, depth_scale: float, depth_invalid: int) -> np.ndarray:
    """float32 [H,W] depth in metres (NaN where there is none) or [3,H,W] normals in [0, 1]."""
    if path.suffix == ".npy":
        a = np.load(path).astype(np.float32)
        if task == "depth":
            return a.reshape(a.shape[-2:]) if a.ndim == 3 and a.shape[0] == 1 else a
        return a.transpose(2, 0, 1) if a.ndim == 3 and a.shape[-1] == 3 and a.shape[0] != 3 else a
    img = Image.open(path)
    if task == "depth":
        v = np.asarray(img).astype(np.int64)
        d = (v / depth_scale).astype(np.float32)
        d[v == depth_invalid] = np.nan
        return d
    return (np.asarray(img.convert("RGB"), dtype=np.float32) / 255.0).transpose(2, 0, 1)


def load_mask(path: Path) -> np.ndarray:
    a = np.load(path) if path.suffix == ".npy" else np.asarray(Image.open(path))
    if a.ndim == 3:
        a = a[..., 0] if a.shape[-1] in (3, 4) else a[0]
    return (a != 0).astype(np.uint8)


def load_edges(path: Path) -> np.ndarray:
    """uint8 [H,W], 1 = edge, from an 8-bit PNG or a `.npy` (nonzero = edge)."""
    return load_mask(path)


def build_model(task: str, backbone: str, checkpoint, synthetic: bool, precision: str, device):
    from omnidata_b200 import synthetic as syn
    from omnidata_b200.model import DPTDepthModel, state_dict_spec
    c = 3 if task == "normal" else 1
    model = DPTDepthModel(backbone=backbone, num_channels=c)
    if checkpoint:
        import hubconf
        hubconf._load_checkpoint(model, checkpoint)
    elif synthetic:
        model.load_state_dict(syn.make_state_dict(0, c, spec=state_dict_spec(c, backbone=backbone)))
    else:
        raise FileNotFoundError("pass --checkpoint CKPT, or --synthetic_weights to run with seeded random weights")
    model = model.to(device).eval()
    model.precision = precision
    return model


def image_tensor(path: Path, task: str) -> torch.Tensor:
    """[1,3,H,W] on the CPU, preprocessed as demo.py --full_res does."""
    from demo import to_tensor
    t = to_tensor(Image.open(path).convert("RGB"))
    if task == "depth":
        t = (t - 0.5) / 0.5
    return t.unsqueeze(0)


def predict(model, x: torch.Tensor, mode: str, tile, overlap: int, name: str, anchor=None, ensemble=None,
            flip: bool = False, guided=None) -> torch.Tensor:
    """The clamped fp32 prediction at x's size: [1,H,W] (depth) or [1,3,H,W] (normals).  `ensemble` (a list of sizes,
    None: the image's own) or `flip`: an EnsemblePredictor around the tiled, direct or guided predictor.  `guided`
    (mode "guided"): (size, radius, eps) of the GuidedPredictor."""
    from omnidata_b200.ensemble import EnsemblePredictor
    from omnidata_b200.guided import GuidedPredictor
    from omnidata_b200.model import check_input_size
    from omnidata_b200.tiled import TiledPredictor
    with torch.no_grad():
        if mode == "guided":
            size, radius, eps = guided
            base = GuidedPredictor(model, size=size, radius=radius, eps=eps)
            try:
                y = EnsemblePredictor(base, sizes=ensemble, flip=flip)(x) if ensemble is not None or flip else base(x)
            except ValueError as e:
                raise ValueError(f"{name}: the guided predictor cannot take this image: {e}") from None
        elif ensemble is not None or flip:
            base = TiledPredictor(model, tile=tile, overlap=overlap, anchor=anchor) if mode == "tiled" else model
            try:
                y = EnsemblePredictor(base, sizes=ensemble, flip=flip)(x)
            except ValueError as e:
                raise ValueError(f"{name}: the ensemble cannot take this image: {e}") from None
        elif mode == "tiled":
            y = TiledPredictor(model, tile=tile, overlap=overlap, anchor=anchor)(x)
        else:
            try:
                check_input_size(x.shape[2], x.shape[3], model.arch["hybrid"], autograd=False)
            except ValueError as e:
                raise ValueError(f"{name}: --mode direct cannot take this image: {e}") from None
            y = model(x)
    return y.float().clamp(0, 1).contiguous()


def evaluate(args) -> dict:
    from omnidata_b200.metrics import BoundaryMetrics, DepthMetrics, NormalMetrics
    device = torch.device("cuda:0")
    images = sorted(p for p in Path(args.img_path).iterdir() if p.suffix.lower() in IMAGE_EXT)
    if not images:
        raise FileNotFoundError(f"no images in {args.img_path}")
    model = build_model(args.task, args.backbone, args.checkpoint, args.synthetic_weights, args.precision, device)
    if args.task == "depth":
        metric = DepthMetrics(space=args.space, min_depth=args.min_depth, max_depth=args.max_depth)
    else:
        metric = NormalMetrics()
    boundary = BoundaryMetrics(min_depth=args.min_depth, max_depth=args.max_depth) if args.boundary else None
    tile = (args.tile, args.tile)
    guided = (args.guided_size, args.radius, args.eps) if args.mode == "guided" else None
    if guided is not None:                          # a refused size or setting fails here, before the first image
        from omnidata_b200.guided import GuidedPredictor
        GuidedPredictor(model, size=args.guided_size, radius=args.radius, eps=args.eps)
    for p in images:
        gt = load_gt(_find(args.gt_path, p.stem, "ground truth"), args.task, args.depth_scale, args.depth_invalid)
        x = image_tensor(p, args.task)
        if tuple(gt.shape[-2:]) != tuple(x.shape[-2:]):
            raise ValueError(f"{p.name}: ground truth is {gt.shape[-2]}x{gt.shape[-1]}, the image "
                             f"{x.shape[2]}x{x.shape[3]}; nothing is resampled")
        mask = None
        if args.mask_path:
            mask = torch.from_numpy(load_mask(_find(args.mask_path, p.stem, "mask"))).unsqueeze(0).to(device)
        pred = predict(model, x.to(device), args.mode, tile, args.overlap, p.name, args.anchor, args.ensemble_sizes,
                       args.flip, guided)
        gt_t = torch.from_numpy(np.ascontiguousarray(gt)).unsqueeze(0).to(device)
        metric.update(pred, gt_t, mask)
        if boundary is not None:
            edges = None
            if args.edge_path:
                edges = torch.from_numpy(load_edges(_find(args.edge_path, p.stem, "edge map"))).unsqueeze(0).to(device)
                if tuple(edges.shape[-2:]) != tuple(gt.shape[-2:]):
                    raise ValueError(f"{p.name}: the edge map is {edges.shape[-2]}x{edges.shape[-1]}, the ground "
                                     f"truth {gt.shape[-2]}x{gt.shape[-1]}")
            boundary.update(pred, gt_t, mask, edges)
    result = {"task": args.task, "backbone": args.backbone, "mode": args.mode, "precision": args.precision,
              "tile": list(tile) if args.mode == "tiled" else None,
              "overlap": args.overlap if args.mode == "tiled" else None,
              "anchor": list(args.anchor) if args.anchor else None, "images": len(images),
              "guided": {"size": list(args.guided_size), "radius": args.radius, "eps": args.eps} if guided else None}
    if args.ensemble_sizes is not None or args.flip:
        result["ensemble"] = {"sizes": [list(s) if s else None for s in args.ensemble_sizes or [None]],
                              "flip": args.flip}
    if args.task == "depth":
        result.update(space=args.space, min_depth=args.min_depth, max_depth=args.max_depth)
    result["metrics"] = metric.compute()
    if boundary is not None:
        result["boundary"] = dict(boundary.compute(), edges="given" if args.edge_path else "detected")
    return result


def _size(text: str):
    try:
        h, w = (int(v) for v in text.lower().split("x"))
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected HxW, e.g. 768x1024, got {text!r}") from None
    return h, w


def _sizes(text: str):
    """HxW,... -> [(H, W) or None]; `native` stands for the image's own size."""
    return [None if part.strip().lower() == "native" else _size(part) for part in text.split(",")]


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Evaluate depth or surface-normal predictions against ground truth")
    ap.add_argument("--task", required=True, choices=("depth", "normal"))
    ap.add_argument("--img_path", required=True, help="directory of RGB images")
    ap.add_argument("--gt_path", required=True, help="directory of ground truth, matched by file stem")
    ap.add_argument("--mask_path", default=None, help="directory of masks (nonzero = valid), matched by file stem")
    w = ap.add_mutually_exclusive_group(required=True)
    w.add_argument("--checkpoint", default=None)
    w.add_argument("--synthetic_weights", action="store_true", help="seeded random weights (no checkpoint)")
    ap.add_argument("--backbone", default="vitb_rn50_384", choices=("vitb_rn50_384", "vitl16_384", "vitb16_384"))
    ap.add_argument("--precision", default="bf16", choices=("fp32", "bf16", "fp8"))
    ap.add_argument("--mode", default="tiled", choices=("tiled", "direct", "guided"))
    ap.add_argument("--tile", type=int, default=384)
    ap.add_argument("--overlap", type=int, default=64)
    ap.add_argument("--anchor", type=_size, default=None, metavar="HxW",
                    help="depth, --mode tiled: fit the tiles to the model's prediction of the image resized to HxW")
    ap.add_argument("--guided_size", type=_size, default=None, metavar="HxW",
                    help="--mode guided: the input size of the one forward, upsampled with the image as the guide")
    ap.add_argument("--radius", type=int, default=None,
                    help="--mode guided: window radius in low-resolution pixels (default 4, untuned)")
    ap.add_argument("--eps", type=float, default=None,
                    help="--mode guided: ridge, in squared units of the model's input (default 1e-3, untuned)")
    ap.add_argument("--ensemble_sizes", type=_sizes, default=None, metavar="HxW,...",
                    help="ensemble the predictions at these input sizes (`native`: the image's own), merged on the "
                         "device (EnsemblePredictor)")
    ap.add_argument("--flip", action="store_true",
                    help="ensemble each size with its horizontal mirror (alone: the image and its mirror)")
    ap.add_argument("--space", default="depth", choices=("depth", "disparity"))
    ap.add_argument("--min_depth", type=float, default=1e-3)
    ap.add_argument("--max_depth", type=float, default=None)
    ap.add_argument("--depth_scale", type=float, default=512.0, help="16-bit PNG units per metre")
    ap.add_argument("--depth_invalid", type=int, default=65535, help="16-bit PNG value marking no depth")
    ap.add_argument("--boundary", action="store_true",
                    help="depth: also report the depth-boundary errors (BoundaryMetrics) under the `boundary` key")
    ap.add_argument("--edge_path", default=None, metavar="DIR",
                    help="--boundary: ground-truth edge maps (8-bit PNG or .npy, nonzero = edge) matched by file "
                         "stem; without it, edges are detected in the ground-truth depth")
    args = ap.parse_args(argv)
    if args.boundary and args.task != "depth":
        ap.error("--boundary applies to --task depth only")
    if args.edge_path is not None and not args.boundary:
        ap.error("--edge_path applies with --boundary only")
    if args.anchor is not None and (args.mode != "tiled" or args.task != "depth"):
        ap.error("--anchor applies to --task depth with --mode tiled only")
    if args.mode == "guided":
        if args.guided_size is None:
            ap.error("--mode guided needs --guided_size HxW")
        args.radius = 4 if args.radius is None else args.radius
        args.eps = 1e-3 if args.eps is None else args.eps
    elif args.guided_size is not None or args.radius is not None or args.eps is not None:
        ap.error("--guided_size, --radius and --eps apply to --mode guided only")
    return args


def main(argv=None) -> dict:
    args = parse_args(argv)
    if not torch.cuda.is_available():
        print("evaluate.py: a CUDA (sm_90a) device is required; this implementation has no CPU path")
        sys.exit(1)
    result = evaluate(args)
    print(json.dumps(result))
    return result


if __name__ == "__main__":
    main()
