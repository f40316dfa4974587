#!/usr/bin/env python
"""Reconstruct a scene from images, posed or not: predict each frame's depth, align it to metres and to what is
already fused, track its camera when it has no pose, integrate it into a TSDF volume on the device, and write the
extracted mesh as a PLY:

    python reconstruct.py --img_path DIR [--pose_path DIR [--track]] --intrinsics FX,FY,CX,CY --voxel V
                          [--bounds X0,Y0,Z0,X1,Y1,Z1] --out mesh.ply [--pose_out DIR]
                          [--checkpoint CKPT | --synthetic_weights] [--backbone ...] [--precision {fp32,bf16,fp8}]
                          [--mode {tiled,direct,guided}] [--tile 384 --overlap 64] [--guided_size HxW]
                          [--sparse_path DIR [--depth_scale 1000]] [--trunc T] [--color] [--photometric LAMBDA]
                          [--loop_closure [--place_recognition]]

Frames are the images of --img_path (PNG / JPEG) in file-name order.  Each has a pose, the 4 x 4 camera-to-world matrix
as text (ScanNet's pose/<stem>.txt), in --pose_path by file stem.  The intrinsics are in pixels of the images.  With
--bounds a dense grid (`TSDFVolume`) covers that box with points every --voxel metres (write `--bounds=-1,...` when X0
is negative).  Without it the volume is sparse (`SparseTSDFVolume`, DESIGN.md §3 "Sparse TSDF volumes"): blocks of 8^3
points every --voxel metres from the world's zero are allocated where frames see depth, so the scene needs no box and
memory goes to observed surfaces only; the summary then reports `blocks` and the allocated `bounds` instead of `dims`.

Per frame: the depth model predicts at the image's size (evaluate.py's predictor and preprocessing; `--mode`, `--tile`,
`--overlap`, `--guided_size`).  `SparseDepthAligner(grid=(1, 1), robust=0.05)` then fits one scale and shift (Huber IRLS, so that
rays that pass through not-yet-observed space and hit a surface behind it do not pull the fit).  The target is the
frame's sparse depths when --sparse_path has a file for it (16-bit PNG / --depth_scale units per metre, or a `.npy` in
metres; 0 is no measurement).  Otherwise it is the volume's own raycast at the frame's pose, so each frame is aligned
to what is already fused.  Frame 0 must have sparse depths: they fix the scene's metric scale.  The aligned depth is
integrated.  A frame whose fit fails (fewer than two target pixels, a flat prediction) is skipped and
named in the summary.

Without --pose_path the cameras are tracked (`FrameTracker`, point-to-plane ICP against the volume).  This mode and
--track are experimental: tracking against the fused model drifts (on the analytic test scene at 12.5 mm voxels, 13.5
mm over 48 frames, and refined poses end a mean 6.8 mm from the truth when given 20 mm off; with --photometric 1e-2 on
its textured version 3.4 mm and 1.45 mm; DESIGN.md §6).  Frame 0's pose is
the identity, so --bounds (when given) are in frame 0's camera coordinates (x right, y down, z forward); frame 0 still
needs sparse depths.  Every later frame starts from the last tracked pose: the volume is raycast there, one scale and shift is fitted
as above (to the frame's sparse depths when it has them, then the aligned metres are tracked with the pose alone;
otherwise to that raycast, then the scale and shift are tracked with the pose), and the frame is integrated at the
tracked pose.  A frame whose fit or tracking fails is skipped and named with its status; the next frame starts from the
last good pose.  With --pose_path and --track the given poses are the initial guesses (pose refinement).  --pose_out
DIR writes each used frame's pose as <stem>.txt, in the format --pose_path reads.

--color also fuses each frame's image (RGB in [0, 1] at the prediction's size, before the network's normalisation)
into a colour volume and writes a coloured PLY.  --photometric LAMBDA (implies --color; needs tracking, so no
--pose_path without --track) adds a photometric term to the tracking (`FrameTracker(photometric=LAMBDA)`): each frame's
image against the volume's coloured raycast at the initial pose.  It constrains motions the geometry leaves free (a
textured wall); 1e-2 is what the sweep on the analytic scene chose (DESIGN.md §6), not tuned on real data, and there is
no exposure compensation between frames.  It is experimental like the tracking it refines.

--loop_closure (needs tracking, so no --pose_path or --track, and --photometric) corrects drift when the camera comes back to a place it has
seen (`LoopClosure`, DESIGN.md §3 "Loop closure and pose graphs"): keyframes, loop candidates by pose proximity
verified by tracking, an SE(3) pose-graph solve over the keyframes, and re-fusion of the volume from every stored frame
at the corrected poses.  The next frame is tracked from the corrected last pose, and --pose_out writes the final poses.
It keeps every frame's aligned depth on the device (4 bytes per pixel, 16 with --color).  Experimental like the
tracking it corrects.

--place_recognition (needs --loop_closure) adds appearance to it (`LoopClosure(places=True)`, DESIGN.md §3 "Place
recognition and relocalisation"): every keyframe gets a randomized-fern code, loop candidates also come from the
keyframes that look alike, whatever the drifted poses say, and a frame whose fit or tracking fails is relocalised:
`LoopClosure.relocalise` finds its pose against the most similar keyframes, and the frame then runs through the
tracking from that pose (raycast, fit, tracking against the model, integration).  A frame that cannot be relocalised is
skipped with status "relocalise: failed".  So a covered lens, a fast turn or a cut in the video no longer loses the
rest of it.  Relocalisation starts only from a failure: a frame that tracks to a wrong pose is not detected.

--gt_mesh PLY evaluates the extracted mesh against a ground-truth mesh in the world frame of --pose_path (so it needs
--pose_path) with `MeshMetrics` (DESIGN.md §3 "Mesh metrics"): both meshes sampled at --eval_density points per m^2,
accuracy, completion, Chamfer-L1 and precision / recall / F-score at --eval_thresholds metres.  --gt_cull keeps only
what the used frames' cameras see (their final poses, after loop closure), without modelling occlusion.  The result is
the `mesh_metrics` key of the JSON line.

Prints one JSON line: frames used and skipped, vertices, faces, the grid's dims (without --bounds the blocks and the
allocated bounds) and seconds (with --loop_closure also the keyframes,
the accepted loops as (frame i, frame j) index pairs of the used frames, and the number of re-fusions; with
--place_recognition also the names of the relocalised frames).  Runs on cuda:0; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import math
import sys
import time
from pathlib import Path

import numpy as np
import torch

import evaluate

# Huber threshold on the relative residual of the per-frame fit.  A raycast ray can pass through space no frame has
# observed yet (the pair of valid samples breaks) and hit a fused surface behind it; those pixels are outliers that a
# plain least-squares fit follows.  5 IRLS solves, 0.05 not tuned.
ROBUST = 0.05


def _floats(n: int, what: str):
    def parse(text: str):
        try:
            v = tuple(float(x) for x in text.split(","))
        except ValueError:
            v = ()
        if len(v) != n or not all(math.isfinite(x) for x in v):
            raise argparse.ArgumentTypeError(f"expected {what} ({n} finite numbers), got {text!r}")
        return v
    return parse


def _float_list(text: str):
    try:
        v = tuple(float(x) for x in text.split(","))
    except ValueError:
        v = ()
    if not v or not all(math.isfinite(x) for x in v):
        raise argparse.ArgumentTypeError(f"expected comma-separated finite numbers, got {text!r}")
    return v


def load_pose(path: Path) -> np.ndarray:
    """float64 [4,4] camera-to-world from a whitespace-separated text file."""
    T = np.loadtxt(path, dtype=np.float64)
    if T.shape != (4, 4):
        raise ValueError(f"{path}: a pose is a 4 x 4 matrix, got {T.shape}")
    return T


def parse_args(argv=None):
    from omnidata_b200.volume import MAX_DIM, MAX_POINTS
    ap = argparse.ArgumentParser(description="Fuse depth predictions of posed images into a TSDF volume and a mesh")
    ap.add_argument("--img_path", required=True, help="directory of RGB frames")
    ap.add_argument("--pose_path", default=None,
                    help="directory of <stem>.txt camera-to-world 4 x 4 poses (without it the cameras are tracked, "
                         "experimental)")
    ap.add_argument("--track", action="store_true",
                    help="experimental: with --pose_path, refine the given poses by tracking against the volume")
    ap.add_argument("--pose_out", default=None, metavar="DIR", help="write each used frame's pose as <stem>.txt")
    ap.add_argument("--intrinsics", required=True, type=evaluate._intrinsics, metavar="FX,FY,CX,CY",
                    help="camera intrinsics in pixels of the frames")
    ap.add_argument("--voxel", required=True, type=float, help="grid spacing in metres")
    ap.add_argument("--bounds", default=None, type=_floats(6, "X0,Y0,Z0,X1,Y1,Z1"), metavar="X0,Y0,Z0,X1,Y1,Z1",
                    help="world-space box a dense grid covers (default: a sparse volume, no box)")
    ap.add_argument("--out", required=True, help="output mesh (binary PLY)")
    w = ap.add_mutually_exclusive_group(required=True)
    w.add_argument("--checkpoint", default=None)
    w.add_argument("--synthetic_weights", action="store_true", help="seeded random weights (no checkpoint)")
    ap.add_argument("--backbone", default="vitb_rn50_384", choices=("vitb_rn50_384", "vitl16_384", "vitb16_384"))
    ap.add_argument("--precision", default="bf16", choices=("fp32", "bf16", "fp8"))
    ap.add_argument("--mode", default="tiled", choices=("tiled", "direct", "guided"))
    ap.add_argument("--tile", type=int, default=384)
    ap.add_argument("--overlap", type=int, default=64)
    ap.add_argument("--guided_size", type=evaluate._size, default=None, metavar="HxW",
                    help="--mode guided: the input size of the one forward")
    ap.add_argument("--sparse_path", default=None, metavar="DIR",
                    help="sparse depths by file stem (16-bit PNG or .npy in metres); frame 0 must have one")
    ap.add_argument("--depth_scale", type=float, default=1000.0, help="16-bit PNG units per metre (default mm)")
    ap.add_argument("--trunc", type=float, default=None, help="truncation distance in metres (default 3 voxels)")
    ap.add_argument("--color", action="store_true", help="fuse the images' colour and write a coloured PLY")
    ap.add_argument("--photometric", type=float, default=None, metavar="LAMBDA",
                    help="experimental: track with a photometric term of this weight (m^2 per squared intensity "
                         "step; implies --color)")
    ap.add_argument("--loop_closure", action="store_true",
                    help="experimental: correct tracking drift at revisits (pose graph over keyframes, re-fusion; "
                         "needs --photometric)")
    ap.add_argument("--place_recognition", action="store_true",
                    help="experimental: with --loop_closure, find loops by appearance and relocalise frames whose "
                         "tracking fails")
    ap.add_argument("--gt_mesh", default=None, metavar="PLY",
                    help="evaluate the mesh against this ground-truth mesh (world frame of --pose_path)")
    ap.add_argument("--gt_cull", action="store_true",
                    help="with --gt_mesh, keep only surface the used frames' cameras see (final poses)")
    ap.add_argument("--eval_density", type=float, default=1e4,
                    help="with --gt_mesh, surface samples per m^2 of both meshes (default 1e4, about 1 cm apart)")
    ap.add_argument("--eval_thresholds", type=_float_list, default=(0.05,), metavar="T1,...",
                    help="with --gt_mesh, the precision / recall distances in metres (1 to 4; default 0.05)")
    args = ap.parse_args(argv)
    if not (math.isfinite(args.voxel) and args.voxel > 0):
        ap.error(f"--voxel must be finite and > 0, got {args.voxel}")
    if args.bounds is None:
        args.origin, args.dims = (0.0, 0.0, 0.0), None
    else:
        lo, hi = args.bounds[:3], args.bounds[3:]
        if not all(h > l for l, h in zip(lo, hi)):
            ap.error(f"--bounds must have X1 > X0, Y1 > Y0 and Z1 > Z0, got {args.bounds}")
        args.origin = tuple(lo)
        args.dims = tuple(int(math.floor((h - l) / args.voxel + 1e-9)) + 1 for l, h in zip(lo, hi))
        if not all(2 <= d <= MAX_DIM for d in args.dims) or math.prod(args.dims) > MAX_POINTS:
            ap.error(f"--bounds / --voxel give a {args.dims} grid; each dimension must lie in [2, {MAX_DIM}] and the "
                     f"grid hold at most {MAX_POINTS} points")
    if args.sparse_path is None:
        ap.error("--sparse_path is required: frame 0's sparse depths fix the scene's metric scale")
    if not (math.isfinite(args.depth_scale) and args.depth_scale > 0):
        ap.error(f"--depth_scale must be finite and > 0, got {args.depth_scale}")
    if args.trunc is not None and not (math.isfinite(args.trunc) and args.trunc > 0):
        ap.error(f"--trunc must be finite and > 0, got {args.trunc}")
    if args.track and args.pose_path is None:
        ap.error("--track refines the poses of --pose_path; without --pose_path every frame is tracked already")
    if args.photometric is not None:
        if not (math.isfinite(args.photometric) and args.photometric > 0):
            ap.error(f"--photometric must be finite and > 0, got {args.photometric}")
        if args.pose_path is not None and not args.track:
            ap.error("--photometric weights a term of the tracking; with --pose_path nothing is tracked without "
                     "--track")
        args.color = True
    if args.loop_closure and args.pose_path is not None and not args.track:
        ap.error("--loop_closure corrects tracked poses; with --pose_path nothing is tracked without --track")
    if args.loop_closure and args.photometric is None:
        ap.error("--loop_closure needs --photometric: pose-graph edges from geometry alone bent the analytic test "
                 "scene's trajectory instead of correcting it (DESIGN.md §6)")
    if args.place_recognition and not args.loop_closure:
        ap.error("--place_recognition needs --loop_closure (it keeps the keyframes it looks up)")
    if args.pose_out is not None and Path(args.pose_out).exists() and not Path(args.pose_out).is_dir():
        ap.error(f"--pose_out must be a directory, got the file {args.pose_out}")
    if args.gt_mesh is None:
        if args.gt_cull:
            ap.error("--gt_cull culls the ground truth of --gt_mesh")
    elif args.pose_path is None:
        ap.error("--gt_mesh needs --pose_path: without it the world frame is frame 0's camera, not the ground truth's "
                 "frame")
    if not (math.isfinite(args.eval_density) and args.eval_density > 0):
        ap.error(f"--eval_density must be finite and > 0, got {args.eval_density}")
    if not 1 <= len(args.eval_thresholds) <= 4 or not all(t > 0 for t in args.eval_thresholds):
        ap.error(f"--eval_thresholds takes 1 to 4 distances > 0, got {args.eval_thresholds}")
    if args.mode == "guided":
        if args.guided_size is None:
            ap.error("--mode guided needs --guided_size HxW")
    elif args.guided_size is not None:
        ap.error("--guided_size applies to --mode guided only")
    return args


def align_and_integrate(volume, aligner, pred: torch.Tensor, intrinsics, pose: np.ndarray, sparse=None, rgb=None,
                        loop=None):
    """One frame of the loop: fit pred fp32 [1,H,W] to sparse [1,H,W] (metres, 0 = none) or, without it, to the
    volume's raycast at pose; integrate the aligned depth (and rgb fp32 [3,H,W] into a colour volume) when the fit is
    ok, and store it in loop (a LoopClosure) when given.  Returns the aligner's record (fp64 [8], on the host) and the
    nodes (scale, shift)."""
    h, w = pred.shape[-2:]
    target = sparse if sparse is not None else volume.raycast(intrinsics, pose, (h, w)).unsqueeze(0)
    nodes, rec = aligner.fit(pred, target)
    rec, st = rec[0].cpu(), nodes.reshape(2).cpu()
    if int(rec[1]) == 0:
        metres = aligner.apply(pred, nodes)
        volume.integrate(metres, intrinsics, pose, None if rgb is None else rgb.unsqueeze(0))
        if loop is not None and loop.add(metres, pose, rgb):
            loop.refuse(volume)
    return rec, (float(st[0]), float(st[1]))


def track_and_integrate(volume, aligner, trackers, pred: torch.Tensor, intrinsics, init_pose: np.ndarray,
                        sparse=None, rgb=None, loop=None):
    """One frame of the tracking loop: raycast the volume at init_pose, fit pred fp32 [1,H,W] with the aligner to
    sparse [1,H,W] (metres, 0 = none) or, without it, to that raycast, track it (trackers[False] on the aligned metres
    with sparse, else trackers[True] on pred with the fitted (s, t) as initial nodes), and integrate the aligned depth at
    the tracked pose.  rgb fp32 [3,H,W] (a colour volume): integrated with the depth and, for trackers with a
    photometric term, tracked against the coloured raycast.  Returns (failure, pose, (s, t)): failure None when the
    frame was integrated, else "fit: <status>" or "track: <status>"; pose the tracked host float64 [4,4] (None on
    failure).  With loop (a LoopClosure) the integrated frame is stored there; when that closes a loop the volume is
    re-fused and pose is the frame's corrected pose."""
    from omnidata_b200.sparse import STATUS as FIT_STATUS
    from omnidata_b200.track import STATUS as TRACK_STATUS
    h, w = pred.shape[-2:]
    photo = trackers[True].photometric > 0
    ref, ref_rgb = volume.raycast(intrinsics, init_pose, (h, w), color=True) if photo else \
        (volume.raycast(intrinsics, init_pose, (h, w)), None)
    colour = dict(rgb=rgb, ref_rgb=ref_rgb) if photo else {}
    nodes, rec = aligner.fit(pred, sparse if sparse is not None else ref.unsqueeze(0))
    status = int(rec[0, 1].item())
    if status != 0:
        return f"fit: {FIT_STATUS[status]}", None, None
    if sparse is not None:
        metres = aligner.apply(pred, nodes)
        pose, _, trec = trackers[False].track(metres, ref, intrinsics, init_pose, **colour)
    else:
        pose, nodes, trec = trackers[True].track(pred, ref, intrinsics, init_pose, init_nodes=nodes, **colour)
        metres = aligner.apply(pred, nodes)
    status = int(trec[1].item())
    if status != 0:
        return f"track: {TRACK_STATUS[status]}", None, None
    pose = pose.cpu().numpy()
    volume.integrate(metres, intrinsics, pose, None if rgb is None else rgb.unsqueeze(0))
    if loop is not None and loop.add(metres, pose, rgb):
        loop.refuse(volume)
        pose = loop.poses[-1]
    st = nodes.reshape(2).cpu()
    return None, pose, (float(st[0]), float(st[1]))


def relocalise_and_integrate(volume, aligner, trackers, loop, pred: torch.Tensor, intrinsics, sparse=None, rgb=None):
    """A lost frame: its pose from loop.relocalise (a LoopClosure with places=True), then track_and_integrate from
    there.  Returns (failure, pose, (s, t)) as track_and_integrate does; failure is "relocalise: failed" when no
    keyframe gives a pose or the frame fails from the pose it gives."""
    init = loop.relocalise(pred, rgb, sparse)
    if init is None:
        return "relocalise: failed", None, None
    failure, pose, st = track_and_integrate(volume, aligner, trackers, pred, intrinsics, init, sparse, rgb, loop)
    if failure is not None:
        loop.cancel_relocalisation()
        return "relocalise: failed", None, None
    return None, pose, st


def reconstruct(args) -> dict:
    from omnidata_b200.loop import LoopClosure
    from omnidata_b200.sparse import STATUS, SparseDepthAligner
    from omnidata_b200.track import FrameTracker
    from omnidata_b200.volume import SparseTSDFVolume, TSDFVolume, write_ply
    t0 = time.perf_counter()
    device = torch.device("cuda:0")
    images = sorted(p for p in Path(args.img_path).iterdir() if p.suffix.lower() in evaluate.IMAGE_EXT)
    if not images:
        raise FileNotFoundError(f"no images in {args.img_path}")
    posed = args.pose_path is not None
    poses = [load_pose(Path(args.pose_path) / (p.stem + ".txt")) for p in images] if posed else [None] * len(images)
    evaluate._find(args.sparse_path, images[0].stem, "sparse depth for frame 0")
    model = evaluate.build_model("depth", args.backbone, args.checkpoint, args.synthetic_weights, args.precision,
                                 device)
    guided = (args.guided_size, 4, 1e-3) if args.mode == "guided" else None
    if args.dims is None:
        volume = SparseTSDFVolume(args.voxel, trunc=args.trunc, color=args.color, origin=args.origin, device=device)
    else:
        volume = TSDFVolume(args.origin, args.voxel, args.dims, trunc=args.trunc, color=args.color, device=device)
    aligner = SparseDepthAligner(grid=(1, 1), robust=ROBUST)
    tracking = args.track or not posed
    lam = 0.0 if args.photometric is None else args.photometric
    trackers = {a: FrameTracker(affine=a, photometric=lam) for a in (False, True)} if tracking else None
    if args.pose_out is not None:
        Path(args.pose_out).mkdir(parents=True, exist_ok=True)
    loop = None
    last = np.eye(4)                                  # the last good pose: frame 0's without --pose_path
    used, used_poses, skipped, relocalised = [], [], [], []
    for q, (p, pose) in enumerate(zip(images, poses)):
        image = evaluate.image_tensor(p, "rgb")                   # [1,3,H,W] in [0, 1]
        x = ((image - 0.5) / 0.5).to(device)                       # image_tensor(p, "depth")'s normalisation
        rgb = image[0].to(device) if args.color else None
        pred = evaluate.predict(model, x, args.mode, (args.tile, args.tile), args.overlap, p.name, guided=guided)
        sparse = None
        try:
            sp = evaluate.load_sparse(evaluate._find(args.sparse_path, p.stem, "sparse depth"), args.depth_scale,
                                      65535)
        except FileNotFoundError:
            sp = None
        if sp is not None:
            if tuple(sp.shape) != tuple(pred.shape[-2:]):
                raise ValueError(f"{p.name}: the sparse depth is {sp.shape[0]}x{sp.shape[1]}, the image "
                                 f"{pred.shape[-2]}x{pred.shape[-1]}")
            sparse = torch.from_numpy(sp).unsqueeze(0).to(device)
        if args.loop_closure and loop is None:
            loop = LoopClosure(args.intrinsics, tuple(pred.shape[-2:]), photometric=lam,
                               places=args.place_recognition, device=device)
        if tracking and used:
            failure, pose, _ = track_and_integrate(volume, aligner, trackers, pred, args.intrinsics,
                                                   pose if posed else last, sparse, rgb, loop)
            if failure is not None and args.place_recognition:
                failure, pose, _ = relocalise_and_integrate(volume, aligner, trackers, loop, pred, args.intrinsics,
                                                            sparse, rgb)
                if failure is None:
                    relocalised.append(p.name)
        else:
            pose = last if pose is None else pose
            rec, _ = align_and_integrate(volume, aligner, pred, args.intrinsics, pose, sparse, rgb, loop)
            failure = None if int(rec[1]) == 0 else STATUS[int(rec[1])]
        if failure is None:
            used.append(p)
            used_poses.append(pose)
            last = pose
            if args.pose_out is not None and loop is None:
                np.savetxt(Path(args.pose_out) / (p.stem + ".txt"), pose)
        else:
            skipped.append({"frame": p.name, "status": failure})
    if args.pose_out is not None and loop is not None:
        for p, pose in zip(used, loop.poses):                     # the final poses, after the last closure
            np.savetxt(Path(args.pose_out) / (p.stem + ".txt"), pose)
    vertices, faces, colors = volume.extract_mesh()
    write_ply(args.out, vertices, faces, colors)
    result = {"frames": len(images), "frames_used": len(used), "frames_skipped": skipped,
              "vertices": int(vertices.shape[0]), "faces": int(faces.shape[0])}
    if args.dims is None:
        bounds = volume.bounds()
        result.update(blocks=volume.blocks, bounds=None if bounds is None else [list(bounds[0]), list(bounds[1])])
    else:
        result["dims"] = list(args.dims)
    result.update(voxel=args.voxel, out=str(args.out), seconds=round(time.perf_counter() - t0, 3))
    if loop is not None:
        result.update(keyframes=len(loop.keyframes), loops=[list(pair) for pair in loop.loops],
                      refusions=loop.refusions)
        if args.place_recognition:
            result["relocalised"] = relocalised
        result["seconds"] = round(time.perf_counter() - t0, 3)
    if args.gt_mesh is not None:
        # every used frame is stored in the loop closure, whose poses are the final ones
        final = None if not used else loop.poses if loop is not None else np.stack(used_poses)
        result["mesh_metrics"] = evaluate_mesh(args, vertices, faces, final, tuple(pred.shape[-2:]))
        result["seconds"] = round(time.perf_counter() - t0, 3)
    return result


def evaluate_mesh(args, vertices, faces, poses, size) -> dict:
    """MeshMetrics of the extracted mesh against --gt_mesh; with --gt_cull both sides are culled to the frustums of
    the used frames' final poses (host float64 [F,4,4], None when no frame was used: then nothing is culled) at the
    prediction's size and intrinsics."""
    from omnidata_b200.metrics import MeshMetrics
    from omnidata_b200.volume import read_ply
    gv, gf, _ = read_ply(args.gt_mesh)
    dev = vertices.device
    metric = MeshMetrics(thresholds=args.eval_thresholds, density=args.eval_density)
    views = (args.intrinsics, size, poses) if args.gt_cull and poses is not None else None
    metric.update(vertices, faces, torch.from_numpy(gv).to(dev), torch.from_numpy(gf).to(dev), views=views)
    return metric.compute()


def main(argv=None) -> dict:
    args = parse_args(argv)
    if not torch.cuda.is_available():
        print("reconstruct.py: a CUDA (sm_90a) device is required; this implementation has no CPU path")
        sys.exit(1)
    result = reconstruct(args)
    print(json.dumps(result))
    return result


if __name__ == "__main__":
    main()
