#!/usr/bin/env python
"""Evaluate a depth or surface-normal model over a directory of images and ground truth:

    python evaluate.py --task {depth,normal} --img_path DIR --gt_path DIR [--mask_path DIR]
                       [--checkpoint CKPT | --synthetic_weights] [--backbone ...] [--precision {fp32,bf16,fp8}]
                       [--mode {tiled,direct,guided}] [--tile 384 --overlap 64] [--anchor HxW]
                       [--guided_size HxW [--radius R] [--eps E]] [--ensemble_sizes HxW,... --flip]
                       [--space {depth,disparity}] [--min_depth] [--max_depth] [--depth_scale] [--depth_invalid]
                       [--boundary [--edge_path DIR]]
                       [--sparse_points N [--sparse_seed S] | --sparse_path DIR] [--sparse_grid GYxGX]
                       [--sparse_smooth L] [--huber D [--huber_iterations K]]
                       [--fuse_normals --intrinsics FX,FY,CX,CY [--normal_checkpoint CKPT] [--fusion_weight W]
                        [--no_shift]]

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
nonzero = edge, matched by file stem) or, without it, edges detected in the ground-truth depth.  `--sparse_points N` or
`--sparse_path DIR` (depth) also scores metric depth: the evaluated prediction is aligned in `--space` to sparse
depths (`SparseDepthAligner`, grid `--sparse_grid`, smoothing `--sparse_smooth`, Huber IRLS with `--huber`) and scored
without a further fit (`DepthMetrics(align=False)`), under the `sparse` key.  The sparse depths are N valid
ground-truth pixels per image, drawn without replacement by numpy `default_rng([--sparse_seed, crc32(stem)])` (all of
them when fewer are valid; 200 is the sparse-to-dense protocol of Ma & Karaman on NYUv2), or read from DIR by file
stem: a 16-bit PNG under --depth_scale / --depth_invalid (0 is also no measurement) or a float `.npy` in metres (0 /
NaN: none).  `--fuse_normals` (depth) also runs the normal model (`--normal_checkpoint`, or seeded weights with
`--synthetic_weights`) with the same mode, ensemble and guided settings on the image in [0, 1], fuses the depth
prediction with its normals (`DepthNormalFusion`, intrinsics in pixels of the image, weight `--fusion_weight`, no shift
with `--no_shift`) and reports, under the `fusion` key, the depth metrics of the fused depth, the angular agreement of
the normals implied by the predicted and by the fused depth with the normal prediction (`depth_normals`,
`NormalMetrics`), and the fusion records.  Prints one JSON
line: the metrics (omnidata_b200.metrics), the mode, precision, tile settings and the number of images.  Runs on cuda:0;
there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import math
import sys
import zlib
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


def load_sparse(path: Path, depth_scale: float, depth_invalid: int) -> np.ndarray:
    """float32 [H,W] sparse depth in metres, 0 where there is no measurement."""
    if path.suffix == ".npy":
        a = np.load(path).astype(np.float32)
        a = a.reshape(a.shape[-2:]) if a.ndim == 3 and a.shape[0] == 1 else a
        return np.where(np.isfinite(a), a, 0.0).astype(np.float32)
    v = np.asarray(Image.open(path)).astype(np.int64)
    return np.where((v == depth_invalid) | (v == 0), 0.0, v / depth_scale).astype(np.float32)


def sample_sparse(gt: np.ndarray, n: int, seed: int, stem: str, min_depth: float, max_depth: float,
                  mask: np.ndarray = None) -> np.ndarray:
    """float32 [H,W]: n of gt's valid pixels (DepthMetrics' rule: mask != 0, finite, in (min_depth, max_depth]), drawn
    without replacement by default_rng([seed, crc32(stem)]) from the valid pixels in row-major order (all of them when
    fewer are valid); 0 elsewhere."""
    with np.errstate(invalid="ignore"):
        valid = np.isfinite(gt) & (gt > min_depth) & (gt <= max_depth)
    if mask is not None:
        valid &= mask != 0
    idx = np.flatnonzero(valid)
    if idx.size > n:
        idx = np.sort(np.random.default_rng([seed, zlib.crc32(stem.encode())]).choice(idx, n, replace=False))
    out = np.zeros(gt.size, np.float32)
    out[idx] = gt.reshape(-1)[idx]
    return out.reshape(gt.shape)


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
    sparse_on = args.sparse_points is not None or args.sparse_path is not None
    if sparse_on:
        from omnidata_b200.sparse import SparseDepthAligner
        aligner = SparseDepthAligner(space=args.space, grid=args.sparse_grid, smooth=args.sparse_smooth,
                                     robust=args.huber, iterations=args.huber_iterations, min_depth=args.min_depth,
                                     max_depth=args.max_depth)
        sparse_metric = DepthMetrics(min_depth=args.min_depth, max_depth=args.max_depth, align=False)
        sparse_records = []
    if args.fuse_normals:
        from omnidata_b200.fusion import DepthNormalFusion, depth_normals
        normal_model = build_model("normal", args.backbone, args.normal_checkpoint, args.synthetic_weights,
                                   args.precision, device)
        fusion = DepthNormalFusion(weight=args.fusion_weight, shift=not args.no_shift)
        fused_metric = DepthMetrics(space=args.space, min_depth=args.min_depth, max_depth=args.max_depth)
        agree = {"pred": NormalMetrics(), "fused": NormalMetrics()}
        fusion_records = []
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
        if sparse_on:
            if args.sparse_path:
                sp = load_sparse(_find(args.sparse_path, p.stem, "sparse depth"), args.depth_scale, args.depth_invalid)
                if tuple(sp.shape) != tuple(gt.shape):
                    raise ValueError(f"{p.name}: the sparse depth is {sp.shape[0]}x{sp.shape[1]}, the ground truth "
                                     f"{gt.shape[0]}x{gt.shape[1]}")
            else:
                sp = sample_sparse(gt, args.sparse_points, args.sparse_seed, p.stem, args.min_depth,
                                   math.inf if args.max_depth is None else args.max_depth,
                                   None if mask is None else mask[0].cpu().numpy())
            nodes, rec = aligner.fit(pred, torch.from_numpy(sp).unsqueeze(0).to(device))
            sparse_records.append(rec.clone())
            sparse_metric.update(aligner.apply(pred, nodes), gt_t, mask)
        if args.fuse_normals:
            normals = predict(normal_model, image_tensor(p, "normal").to(device), args.mode, tile, args.overlap,
                              p.name, None, args.ensemble_sizes, args.flip, guided)
            fused, rec = fusion.fit(pred, normals, args.intrinsics, mask)
            fusion_records.append(rec.clone())
            fused_metric.update(fused, gt_t, mask)
            for key, d in (("pred", pred), ("fused", fused)):
                agree[key].update(depth_normals(d, args.intrinsics, mask=mask), normals, mask)
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
    if sparse_on:
        rec = torch.cat(sparse_records).cpu()
        status = rec[:, 1].long()
        result["sparse"] = {
            "source": "path" if args.sparse_path else "points", "points": args.sparse_points,
            "seed": args.sparse_seed if args.sparse_points is not None else None, "grid": list(args.sparse_grid),
            "smooth": args.sparse_smooth, "huber": args.huber,
            "huber_iterations": aligner.iterations if args.huber is not None else None,
            "metrics": sparse_metric.compute(),
            "records": {"ok": int((status == 0).sum()), "no_points": int((status == 1).sum()),
                        "degenerate": int((status == 2).sum()), "nonfinite": int((status == 3).sum()),
                        "mean_points": float(rec[:, 0].mean())}}
    if args.fuse_normals:
        rec = torch.cat(fusion_records).cpu()
        status = rec[:, 1].long()
        result["fusion"] = {
            "intrinsics": list(args.intrinsics), "weight": args.fusion_weight, "shift": not args.no_shift,
            "metrics": fused_metric.compute(),
            "consistency": {"pred": agree["pred"].compute(), "fused": agree["fused"].compute()},
            "records": {"converged": int((status == 0).sum()), "empty": int((status == 1).sum()),
                        "flat": int((status == 2).sum()), "not_converged": int((status == 3).sum()),
                        "mean_iterations": float(rec[:, 3].mean())}}
    return result


def _intrinsics(text: str):
    try:
        k = tuple(float(v) for v in text.split(","))
    except ValueError:
        k = ()
    if len(k) != 4 or not all(math.isfinite(v) for v in k) or k[0] <= 0 or k[1] <= 0:
        raise argparse.ArgumentTypeError(f"expected FX,FY,CX,CY (pixels, fx, fy > 0), got {text!r}")
    return k


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
    ap.add_argument("--sparse_points", type=int, default=None, metavar="N",
                    help="depth: also score metric depth aligned to N ground-truth samples per image (`sparse` key)")
    ap.add_argument("--sparse_path", default=None, metavar="DIR",
                    help="depth: also score metric depth aligned to sparse depths read from DIR by file stem "
                         "(16-bit PNG or .npy in metres)")
    ap.add_argument("--sparse_seed", type=int, default=None, help="--sparse_points: sampler seed (default 0)")
    ap.add_argument("--sparse_grid", type=_size, default=None, metavar="GYxGX",
                    help="sparse alignment: scale / shift node grid (default 1x1: one global fit)")
    ap.add_argument("--sparse_smooth", type=float, default=None,
                    help="sparse alignment: smoothness between neighbouring nodes (default 0.1, untuned)")
    ap.add_argument("--huber", type=float, default=None, metavar="D",
                    help="sparse alignment: Huber IRLS threshold on the relative residual (default: plain least "
                         "squares)")
    ap.add_argument("--huber_iterations", type=int, default=None,
                    help="--huber: number of reweighted solves in [2, 32] (default 5)")
    ap.add_argument("--fuse_normals", action="store_true",
                    help="depth: also fuse the depth with the normal model's prediction (`fusion` key)")
    ap.add_argument("--normal_checkpoint", default=None, help="--fuse_normals: the normal model's checkpoint")
    ap.add_argument("--intrinsics", type=_intrinsics, default=None, metavar="FX,FY,CX,CY",
                    help="--fuse_normals: camera intrinsics in pixels of the image")
    ap.add_argument("--fusion_weight", type=float, default=None,
                    help="--fuse_normals: weight of the depth prediction (default 0.1, untuned)")
    ap.add_argument("--no_shift", action="store_true", help="--fuse_normals: do not recover a shift")
    args = ap.parse_args(argv)
    if args.fuse_normals:
        if args.task != "depth":
            ap.error("--fuse_normals applies to --task depth only")
        if args.intrinsics is None:
            ap.error("--fuse_normals needs --intrinsics FX,FY,CX,CY")
        if args.normal_checkpoint is None and not args.synthetic_weights:
            ap.error("--fuse_normals needs --normal_checkpoint, or --synthetic_weights")
        if args.normal_checkpoint is not None and args.synthetic_weights:
            ap.error("--normal_checkpoint and --synthetic_weights exclude each other")
        args.fusion_weight = 0.1 if args.fusion_weight is None else args.fusion_weight
        from omnidata_b200.fusion import DepthNormalFusion
        try:
            DepthNormalFusion(weight=args.fusion_weight, shift=not args.no_shift)
        except ValueError as e:
            ap.error(f"fusion: {e}")
    elif any(v is not None for v in (args.normal_checkpoint, args.intrinsics, args.fusion_weight)) or args.no_shift:
        ap.error("--normal_checkpoint, --intrinsics, --fusion_weight and --no_shift apply with --fuse_normals only")
    sparse_on = args.sparse_points is not None or args.sparse_path is not None
    if args.sparse_points is not None and args.sparse_path is not None:
        ap.error("give one of --sparse_points and --sparse_path")
    if sparse_on and args.task != "depth":
        ap.error("--sparse_points / --sparse_path apply to --task depth only")
    if not sparse_on and any(v is not None for v in (args.sparse_grid, args.sparse_smooth, args.huber,
                                                     args.huber_iterations, args.sparse_seed)):
        ap.error("--sparse_grid, --sparse_smooth, --huber, --huber_iterations and --sparse_seed apply with "
                 "--sparse_points or --sparse_path only")
    if args.sparse_seed is not None and args.sparse_points is None:
        ap.error("--sparse_seed applies with --sparse_points only")
    if args.sparse_points is not None and args.sparse_points < 1:
        ap.error("--sparse_points must be at least 1")
    if args.huber_iterations is not None and args.huber is None:
        ap.error("--huber_iterations applies with --huber only")
    if sparse_on:
        args.sparse_grid = (1, 1) if args.sparse_grid is None else args.sparse_grid
        args.sparse_smooth = 0.1 if args.sparse_smooth is None else args.sparse_smooth
        if args.sparse_points is not None:
            args.sparse_seed = 0 if args.sparse_seed is None else args.sparse_seed
        from omnidata_b200.sparse import SparseDepthAligner
        try:
            SparseDepthAligner(space=args.space, grid=args.sparse_grid, smooth=args.sparse_smooth, robust=args.huber,
                               iterations=args.huber_iterations, min_depth=args.min_depth, max_depth=args.max_depth)
        except ValueError as e:
            ap.error(f"sparse alignment: {e}")
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
