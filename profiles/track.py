"""FrameTracker on the analytic sphere-in-a-room scene (oracle/volume_oracle.py, oracle/track_oracle.py): a volume fused
from 8 exact orbit frames, a frame 3 cm and 2 degrees from the reference pose with its depth scaled and shifted.  At
640x480 and 1296x968 into 256^3 and 512^3 grids: ms of one tracking call alone (depth_normals and the tracking
launches) at the default 20-iteration cap and at the iteration count where the frame stops, and ms of the whole
per-frame step (raycast, depth_normals, the initial scale and shift fit, tracking, apply and integrate; reconstruct.py's
step without its host reads of the statuses).  Also the launches per tracking call.  CUDA events, warmed up, mean of
repeated calls.  Prints one JSON line with the card's name and power limit (`--out FILE` also writes it).

--photometric LAMBDA measures the photometric term instead: a colour volume fused from the same frames with the solid
texture of color_volume_oracle.sphere_room_rgb, ms of a tracking call with and without the term (20-iteration cap, the
reference's coloured raycast as ref_rgb) and of a coloured raycast against a depth-only one at both sizes, and the
sweep that chose lambda: the largest rotation error of the chained 48-frame path against exact depth and colour
(tests/test_track_rgbd_gpu.py test_weak_views_of_the_chained_path) for lambda = 0 and 1e-6 .. 1e-1."""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle import color_volume_oracle as CO  # noqa: E402
from oracle import track_oracle as TO  # noqa: E402
from oracle import volume_oracle as VO  # noqa: E402
from profiles.volume import CENTER, LO, HI, RADIUS, _card, _time  # noqa: E402


def main():
    import reconstruct
    from omnidata_b200 import _capi
    from omnidata_b200.sparse import SparseDepthAligner
    from omnidata_b200.track import FrameTracker
    from omnidata_b200.volume import TSDFVolume
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--photometric", type=float, default=None, metavar="LAMBDA")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/track.py measures on the GPU"
    name, power, clock = _card()
    res = {"card": name, "power_limit": power, "max_sm_clock": clock, "runs": []}
    if args.photometric is not None:
        res.update(photometric(args.photometric))
        line = json.dumps(res)
        print(line)
        if args.out:
            Path(args.out).write_text(line + "\n")
        return
    rng = np.random.default_rng(0)
    for size in ((480, 640), (968, 1296)):
        h, w = size
        f = 0.8 * w
        K = (f, f, (w - 1) / 2, (h - 1) / 2)
        T = VO.orbit_poses(8, 1.2, CENTER)
        fused = torch.from_numpy(np.stack([VO.sphere_room_depth(K, t, size, CENTER, RADIUS, LO, HI)
                                           for t in T]).astype(np.float32)).cuda()
        ref = TO.camera_path(1, CENTER)[0]
        truth = TO.perturb(ref, 0.03, np.radians(2.0), rng)
        d = VO.sphere_room_depth(K, truth, size, CENTER, RADIUS, LO, HI)
        pred = torch.from_numpy((1.4 * d - 0.1).astype(np.float32)).cuda().unsqueeze(0)
        for n in (256, 512):
            vol = TSDFVolume((-1.6, -1.6, -1.6), 3.2 / (n - 1), (n, n, n))
            vol.integrate(fused, K, T)
            base = vol._data.clone()
            aligner = SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST)
            ref_depth = vol.raycast(K, ref, size)
            nodes0 = aligner.fit(pred, ref_depth.unsqueeze(0))[0].clone()
            tr = FrameTracker()
            _, _, rec = tr.track(pred, ref_depth, K, ref, init_nodes=nodes0)
            rec = rec.cpu().numpy()
            stop = int(rec[4])
            l0 = _capi.launch_count()
            tr.track(pred, ref_depth, K, ref, init_nodes=nodes0)
            launches = _capi.launch_count() - l0
            ms_cap = _time(lambda: tr.track(pred, ref_depth, K, ref, init_nodes=nodes0), 20)
            tr_stop = FrameTracker(iterations=stop)
            ms_stop = _time(lambda: tr_stop.track(pred, ref_depth, K, ref, init_nodes=nodes0), 20)

            def frame_step():
                r = vol.raycast(K, ref, size)
                n0, _ = aligner.fit(pred, r.unsqueeze(0))
                _, nodes, _ = tr.track(pred, r, K, ref, init_nodes=n0)
                vol.integrate(aligner.apply(pred, nodes), K, ref)

            ms_step = _time(frame_step, 10)
            vol._data.copy_(base)
            dp, dr = TO.pose_error(tr.track(pred, ref_depth, K, ref, init_nodes=nodes0)[0].cpu().numpy(), truth)
            res["runs"].append({"size": [h, w], "grid": n, "status": int(rec[1]), "iterations_to_stop": stop,
                                "correspondences": int(rec[0]), "launches_per_track": launches,
                                "track_ms_20_iterations": ms_cap, f"track_ms_{stop}_iterations": ms_stop,
                                "frame_step_ms_20_iterations": ms_step, "position_error_mm": dp * 1e3,
                                "rotation_error_deg": float(np.degrees(dr))})
            del vol
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


def photometric(lam):
    import reconstruct
    from omnidata_b200.sparse import SparseDepthAligner
    from omnidata_b200.track import FrameTracker
    from omnidata_b200.volume import TSDFVolume
    rng = np.random.default_rng(0)
    runs = []
    for size in ((480, 640), (968, 1296)):
        h, w = size
        f = 0.8 * w
        K = (f, f, (w - 1) / 2, (h - 1) / 2)
        T = VO.orbit_poses(8, 1.2, CENTER)
        scene = lambda t: (VO.sphere_room_depth(K, t, size, CENTER, RADIUS, LO, HI),
                           CO.sphere_room_rgb(K, t, size, CENTER, RADIUS, LO, HI))
        frames = [scene(t) for t in T]
        depth = torch.from_numpy(np.stack([d for d, _ in frames]).astype(np.float32)).cuda()
        colour = torch.from_numpy(np.stack([c for _, c in frames]).astype(np.float32)).cuda()
        ref = TO.camera_path(1, CENTER)[0]
        truth = TO.perturb(ref, 0.03, np.radians(2.0), rng)
        d, c = scene(truth)
        pred = torch.from_numpy((1.4 * d - 0.1).astype(np.float32)).cuda().unsqueeze(0)
        rgb = torch.from_numpy(c.astype(np.float32)).cuda()
        n = 512
        vol = TSDFVolume((-1.6, -1.6, -1.6), 3.2 / (n - 1), (n, n, n), color=True)
        vol.integrate(depth, K, T, colour)
        ref_depth, ref_rgb = vol.raycast(K, ref, size, color=True)
        nodes0 = SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST).fit(pred, ref_depth.unsqueeze(0))[0].clone()
        geo, photo = FrameTracker(), FrameTracker(photometric=lam)
        run = {"size": [h, w], "grid": n}
        for key, tr, kw in (("geometric", geo, {}), ("photometric", photo, dict(rgb=rgb, ref_rgb=ref_rgb))):
            pose, _, rec = tr.track(pred, ref_depth, K, ref, init_nodes=nodes0, **kw)
            dp, dr = TO.pose_error(pose.cpu().numpy(), truth)
            run[key] = {"track_ms_20_iterations": _time(lambda: tr.track(pred, ref_depth, K, ref, init_nodes=nodes0,
                                                                          **kw), 20),
                        "status": int(rec[1]), "iterations": int(rec[4]), "position_error_mm": dp * 1e3,
                        "rotation_error_deg": float(np.degrees(dr))}
        run["raycast_ms"] = _time(lambda: vol.raycast(K, ref, size), 20)
        run["raycast_color_ms"] = _time(lambda: vol.raycast(K, ref, size, color=True), 20)
        runs.append(run)
        del vol
        torch.cuda.empty_cache()
    return {"photometric": lam, "photometric_runs": runs, "sweep": sweep()}


def sweep():
    """{lambda: (largest rotation error in degrees, its frame)} over the chained path against exact depth and colour."""
    import reconstruct
    from omnidata_b200.sparse import SparseDepthAligner
    from omnidata_b200.track import FrameTracker
    size, f = (120, 160), 150.0
    K = (f, f, (size[1] - 1) / 2, (size[0] - 1) / 2)
    path = TO.camera_path(48, CENTER, seed=3)
    out = {}
    for lam in (0.0, 1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 1e-1):
        rng = np.random.default_rng(17)
        aligner, tr = SparseDepthAligner(grid=(1, 1), robust=reconstruct.ROBUST), FrameTracker(photometric=lam)
        last, errs = path[0], []
        for T in path[1:]:
            s1, t1 = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
            cam = lambda p, fn: torch.from_numpy(fn(K, p, size, CENTER, RADIUS, LO, HI).astype(np.float32)).cuda()
            pred = (s1 * cam(T, VO.sphere_room_depth) + t1).unsqueeze(0)
            ref = cam(last, VO.sphere_room_depth)
            n0, _ = aligner.fit(pred, ref.unsqueeze(0))
            kw = dict(rgb=cam(T, CO.sphere_room_rgb), ref_rgb=cam(last, CO.sphere_room_rgb)) if lam > 0 else {}
            pose, _, rec = tr.track(pred, ref, K, last, init_nodes=n0.clone(), **kw)
            if int(rec[1]) != 0:
                errs.append((float("nan"), float("nan")))
                continue
            last = pose.cpu().numpy()
            errs.append(TO.pose_error(last, T))
        e = np.array(errs)
        out[str(lam)] = {"rotation_max_deg": float(np.degrees(np.nanmax(e[:, 1]))),
                         "rotation_median_deg": float(np.degrees(np.nanmedian(e[:, 1]))),
                         "position_max_mm": float(np.nanmax(e[:, 0]) * 1e3), "frame": int(np.nanargmax(e[:, 1])) + 1,
                         "failed": int(np.isnan(e[:, 0]).sum())}
    return out


if __name__ == "__main__":
    main()
