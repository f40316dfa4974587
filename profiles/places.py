"""Place recognition costs and the dissimilarity curve (csrc/places.cu, omnidata_b200/places.py, omnidata_b200/loop.py).

- Encode: one frame at 480x640 and 968x1296 (device ms per call, 20 calls replayed from a CUDA graph, CUDA events).
- Query: one code against 10^3, 10^4 and 10^5 stored keyframes of 500 ferns, k = 3 (the same way).
- The added cost per keyframe of LoopClosure(places=True) on the closed 240-frame orbit of the analytic scene at
  160x120 (true metres and images at the true poses, photometric 1e-2): wall seconds of the whole feed with and without
  places, synchronised, over the keyframes.
- Dissimilarity against the angle between views on that orbit (1.5 degrees per frame): per separation the mean, min
  and max over the frames, and between each frame's metres and a relative prediction (a * d + b) of it.

Prints one JSON line with the card's name, power limit and max SM clock (`--out FILE` also writes it)."""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle import color_volume_oracle as CO  # noqa: E402
from oracle import track_oracle as TO  # noqa: E402
from oracle import volume_oracle as VO  # noqa: E402
from profiles.volume import _card  # noqa: E402

CENTER, RADIUS = (0.03, -0.02, 0.01), 0.5
ROOM_LO, ROOM_HI = (-1.5, -1.5, -1.5), (1.5, 1.5, 1.5)
SIZE = (120, 160)
K = (150.0, 150.0, (SIZE[1] - 1) / 2, (SIZE[0] - 1) / 2)
dev = torch.device("cuda:0")


def _graph_ms(fn, reps=20, windows=3):
    """Device ms per call of fn, `reps` calls captured in one CUDA graph, the best of `windows` replays."""
    fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
        for _ in range(reps):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) / reps)
    return best


def encode(size):
    from omnidata_b200.places import FernDatabase
    h, w = size
    db = FernDatabase(size, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    depth = torch.rand((h, w), generator=g, device=dev) + 0.5
    rgb = torch.rand((3, h, w), generator=g, device=dev)
    return _graph_ms(lambda: db.encode(depth, rgb))


def query(n):
    from omnidata_b200.places import FernDatabase
    db = FernDatabase((60, 80), device=dev)
    g = torch.Generator(device=dev).manual_seed(1)
    db.add(torch.randint(0, 16, (n, db.ferns), generator=g, device=dev, dtype=torch.uint8))
    code = db.codes[n // 2].clone()
    return _graph_ms(lambda: db.query(code, 3))


def _scene(path):
    depth = [torch.from_numpy(VO.sphere_room_depth(K, T, SIZE, CENTER, RADIUS, ROOM_LO, ROOM_HI).astype(np.float32))
             .to(dev) for T in path]
    rgb = [torch.from_numpy(CO.sphere_room_rgb(K, T, SIZE, CENTER, RADIUS, ROOM_LO, ROOM_HI).astype(np.float32))
           .to(dev) for T in path]
    return depth, rgb


def per_keyframe(path, depth, rgb):
    from omnidata_b200.loop import LoopClosure
    out = {}
    for places in (False, True, False, True):               # alternated; the second of each is kept
        loop = LoopClosure(K, SIZE, photometric=1e-2, places=places)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for T, d, c in zip(path, depth, rgb):
            loop.add(d, T, c)
        torch.cuda.synchronize()
        out[places] = (time.perf_counter() - t0, len(loop.keyframes), loop.loops)
    (t0, k0, l0), (t1, k1, l1) = out[False], out[True]
    return {"seconds_without": round(t0, 3), "seconds_with": round(t1, 3), "keyframes": k1,
            "added_ms_per_keyframe": round((t1 - t0) / k1 * 1e3, 3), "loops_without": l0, "loops_with": l1}


def curve(path, depth, rgb):
    from omnidata_b200.places import FernDatabase
    db = FernDatabase(SIZE, device=dev)
    codes = db.encode(torch.stack(depth), torch.stack(rgb)).clone()
    n = len(path)
    rows = []
    for sep in (0, 1, 2, 4, 8, 16, 30, 60, 120):
        d = (codes[: n - sep] != codes[sep:]).sum(1).double() / db.ferns
        angles = [np.degrees(TO.pose_error(path[q], path[q + sep])[1]) for q in range(0, n - sep, 8)]
        rows.append({"frames_apart": sep, "angle_deg": round(float(np.mean(angles)), 2),
                     "mean": round(float(d.mean()), 4), "min": round(float(d.min()), 4),
                     "max": round(float(d.max()), 4)})
    rng = np.random.default_rng(0)
    rel = []
    for q in range(0, n, 8):
        a, b = rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)
        c = db.encode((a * depth[q] + b).contiguous(), rgb[q])[0]
        rel.append(float((c != codes[q]).sum()) / db.ferns)
    return {"separation": rows, "relative_prediction_vs_metres": {"mean": round(float(np.mean(rel)), 4),
                                                                   "max": round(float(np.max(rel)), 4)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from omnidata_b200 import build
    build.build_library()
    path = TO.camera_path(240, CENTER, step_deg=1.5, seed=3)
    depth, rgb = _scene(path)
    res = {"card": _card(),
           "encode_ms": {f"{h}x{w}": round(encode((h, w)), 4) for h, w in ((480, 640), (968, 1296))},
           "query_ms": {str(n): round(query(n), 4) for n in (1000, 10000, 100000)},
           "loop_closure_orbit": per_keyframe(path, depth, rgb),
           "dissimilarity": curve(path, depth, rgb)}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
