"""SparseTSDFVolume against TSDFVolume on the analytic sphere-in-a-room scene (oracle/volume_oracle.py), at the voxels of
256^3 and 512^3 dense grids over the 3.2 m room: integrate ms per frame (8 frames per call) and raycast ms (depth and
colour) at 640x480 and 1296x968, mesh extraction ms, the blocks allocated and the bytes used against the dense grid's,
and re-fusion of 240 frames at 640x480 (one call after reset, as LoopClosure.refuse does).  The sparse volume is timed
in steady state (every block already allocated, so each call reads the new-block count and allocates nothing).  CUDA
events, warmed up, mean of repeated calls.  Prints one JSON line with the card's name and power limit (`--out FILE`
also writes it)."""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from oracle import volume_oracle as VO  # noqa: E402
from volume import CENTER, FRAMES, HI, LO, RADIUS, _card, _time  # noqa: E402


def _frames(size, n, orbit=1.2):
    h, w = size
    f = 0.8 * w
    K = (f, f, (w - 1) / 2, (h - 1) / 2)
    T = VO.orbit_poses(n, orbit, CENTER)
    d = np.stack([VO.sphere_room_depth(K, t, size, CENTER, RADIUS, LO, HI) for t in T]).astype(np.float32)
    rgb = np.random.default_rng(0).random((n, 3, h, w), dtype=np.float32)
    return K, T, torch.from_numpy(d).cuda(), torch.from_numpy(rgb).cuda()


def main():
    from omnidata_b200.volume import SparseTSDFVolume, TSDFVolume
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/sparse_volume.py measures on the GPU"
    name, power, clock = _card()
    res = {"card": name, "power_limit": power, "max_sm_clock": clock, "frames_per_call": FRAMES, "runs": [],
           "refusion": []}
    sizes = ((480, 640), (968, 1296))
    frames = {s: _frames(s, FRAMES) for s in sizes}
    for n in (256, 512):
        voxel = 3.2 / (n - 1)
        for color in (False, True):
            dense = TSDFVolume((-1.6, -1.6, -1.6), voxel, (n, n, n), color=color)
            sparse = SparseTSDFVolume(voxel, color=color, origin=(-1.6, -1.6, -1.6))
            for size in sizes:
                K, T, d, rgb = frames[size]
                c = rgb if color else None
                for vol in (dense, sparse):
                    vol.reset()
                    vol.integrate(d, K, T, c)
                row = {"grid": n, "voxel": voxel, "color": color, "size": list(size), "blocks": sparse.blocks,
                       "sparse_bytes": sparse.blocks * 512 * 4 * (5 if color else 2),
                       "dense_bytes": n ** 3 * 4 * (5 if color else 2)}
                for what, vol in (("dense", dense), ("sparse", sparse)):
                    row[f"{what}_integrate_ms_per_frame"] = _time(lambda: vol.integrate(d, K, T, c), 5) / FRAMES
                    row[f"{what}_raycast_ms"] = _time(lambda: vol.raycast(K, T[1], size), 10)
                    if color:
                        row[f"{what}_raycast_color_ms"] = _time(lambda: vol.raycast(K, T[1], size, color=True), 10)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(3):
                        vol.extract_mesh()
                    torch.cuda.synchronize()
                    row[f"{what}_extract_ms"] = (time.perf_counter() - t0) / 3 * 1e3
                z0, z1 = dense.raycast(K, T[1], size), sparse.raycast(K, T[1], size)
                row["raycast_hits_equal"] = bool(torch.equal(z0 > 0, z1 > 0))
                res["runs"].append(row)
                print(json.dumps(row), file=sys.stderr)
            del dense, sparse
            torch.cuda.empty_cache()
    K, T, d, _ = _frames((480, 640), 240)
    for n in (256, 512):
        voxel = 3.2 / (n - 1)
        dense = TSDFVolume((-1.6, -1.6, -1.6), voxel, (n, n, n))
        sparse = SparseTSDFVolume(voxel, origin=(-1.6, -1.6, -1.6))
        row = {"grid": n, "frames": 240, "size": [480, 640]}
        for what, vol in (("dense", dense), ("sparse", sparse)):
            def refuse():
                vol.reset()
                vol.integrate(d, K, T)
            row[f"{what}_ms"] = _time(refuse, 3)
        row["blocks"] = sparse.blocks
        res["refusion"].append(row)
        print(json.dumps(row), file=sys.stderr)
        del dense, sparse
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
