"""TSDFVolume on the analytic sphere-in-a-room scene (oracle/volume_oracle.py): integrate ms per frame at 640x480 and
1920x1440 into 256^3 and 512^3 grids, with and without colour, with achieved GB/s against the bytes the definition needs
(F, W and colour read at every point and written where observed, plus one depth (and RGB) read per observation) and its
share of 3.35 TB/s; raycast ms at both sizes; mesh count and emit ms at 256^3 and 512^3.  CUDA events, warmed up, mean
of repeated calls.  Prints one JSON line with the card's name and power limit (`--out FILE` also writes it)."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle import volume_oracle as VO  # noqa: E402

PEAK_GBS = 3350.0
CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
LO, HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)
FRAMES = 8


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in q.split(",")]
    except Exception as e:  # the measurement stands without it, but says so
        return [torch.cuda.get_device_name(0), f"unknown ({e})", "unknown"]


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def _frames(size, n):
    h, w = size
    f = 0.8 * w
    K = (f, f, (w - 1) / 2, (h - 1) / 2)
    T = VO.orbit_poses(n, 1.2, CENTER)
    d = np.stack([VO.sphere_room_depth(K, t, size, CENTER, RADIUS, LO, HI) for t in T]).astype(np.float32)
    rgb = np.random.default_rng(0).random((n, 3, h, w), dtype=np.float32)
    return K, T, torch.from_numpy(d).cuda(), torch.from_numpy(rgb).cuda()


def main():
    from omnidata_b200.volume import TSDFVolume
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/volume.py measures on the GPU"
    name, power, clock = _card()
    res = {"card": name, "power_limit": power, "max_sm_clock": clock, "frames_per_call": FRAMES,
           "integrate": [], "raycast": [], "mesh": []}
    frames = {s: _frames(s, FRAMES) for s in ((480, 640), (1440, 1920))}
    for n in (256, 512):
        voxel = 3.2 / (n - 1)
        for color in (False, True):
            vol = TSDFVolume((-1.6, -1.6, -1.6), voxel, (n, n, n), color=color)
            for size, (K, T, d, rgb) in frames.items():
                vol.reset()
                w0 = vol.weight.clone()
                vol.integrate(d, K, T, rgb if color else None)
                obs = float((vol.weight - w0).sum())                 # observations over the 8 frames
                pts = float((vol.weight > w0).sum())                  # points written
                ms = _time(lambda: vol.integrate(d, K, T, rgb if color else None), 5)
                per_point = 20 if color else 8
                nbytes = per_point * n ** 3 + per_point * pts + (16 if color else 4) * obs
                gbs = nbytes / (ms * 1e-3) / 1e9
                res["integrate"].append({"grid": n, "color": color, "size": list(size), "ms_per_frame": ms / FRAMES,
                                         "ms_per_call": ms, "bytes_per_call": nbytes, "GBps": gbs,
                                         "share_of_3350GBps": gbs / PEAK_GBS, "points_written": pts,
                                         "observations": obs})
            if not color:
                for size, (K, T, _, _) in frames.items():
                    ms = _time(lambda: vol.raycast(K, T[1], size), 10)
                    res["raycast"].append({"grid": n, "size": list(size), "ms": ms})
                from omnidata_b200 import ops
                ws = torch.empty(-(-ops.tsdf_mesh_workspace_bytes(vol.dims) // 8), dtype=torch.float64,
                                 device="cuda")
                counts = torch.empty(2, dtype=torch.int64, device="cuda")
                count_ms = _time(lambda: ops.tsdf_mesh_count(vol.tsdf, vol.weight, vol.dims, ws, counts), 10)
                nv, nf = counts.tolist()
                v = torch.empty(nv, 3, device="cuda")
                f = torch.empty(nf, 3, dtype=torch.int32, device="cuda")
                emit_ms = _time(lambda: ops.tsdf_mesh_emit(vol.tsdf, vol.weight, None, vol.dims, vol.origin,
                                                           vol.voxel, ws, v, f, None), 10)
                res["mesh"].append({"grid": n, "count_ms": count_ms, "emit_ms": emit_ms, "vertices": nv, "faces": nf})
            del vol
            torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
