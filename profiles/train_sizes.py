"""Train step time at 320x480 and 384x384 (batch 16, bf16, full loss mix, CUDA-graph replay as bench.py --config 4) and
the pos-embed resize backward kernel alone (odb_pos_embed_resize_bwd, 20x30 -> 24x24, D 768), CUDA events, with the
card's name and power limit.  The two sizes are timed alternately; the step's arithmetic does not depend on the values.
python profiles/train_sizes.py [batch] [--out FILE]   (prints one JSON line; --out also writes it to FILE)"""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from omnidata_b200 import bwd, synthetic  # noqa: E402
from omnidata_b200.model import DPTDepthModel  # noqa: E402
from omnidata_b200.train import DepthTrainStep  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def time_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps


def main():
    argv = sys.argv[1:]
    out_file = None
    if "--out" in argv:
        i = argv.index("--out")
        out_file = argv[i + 1]
        del argv[i:i + 2]
    B = int(argv[0]) if argv else 16
    if not torch.cuda.is_available():
        raise SystemExit("profiles/train_sizes.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"batch": B, "dtype": "bf16", "gpu": gpu_info()}

    # ---- the kernel alone
    g = torch.Generator().manual_seed(0)
    dgrid = torch.randn(20 * 30, 768, generator=g).to(dev)
    dpos = torch.empty(24 * 24, 768, device=dev)
    run = lambda: bwd.pos_embed_resize_bwd(dgrid, 20, 30, dpos)
    time_ms(run, 50)
    t = min(time_ms(run, 1000) for _ in range(3))
    res["pos_embed_resize_bwd_us"] = round(t * 1e3, 2)
    res["pos_embed_resize_bwd_gbytes_per_s"] = round((dgrid.numel() + dpos.numel()) * 4 / (t * 1e-3) / 1e9, 1)

    # ---- the train step at two sizes
    steps = {}
    for h, w in ((384, 384), (320, 480)):
        model = DPTDepthModel()
        model.load_state_dict(synthetic.make_state_dict(0, 1))
        st = DepthTrainStep(model.to(dev).train(), lr=1e-6, clip=10.0, precision="bf16", input_size=(h, w))
        st.use_cuda_graph = True
        rgb = (torch.rand(B, 3, h, w, generator=g) * 2 - 1).to(dev)
        gt = torch.rand(B, 1, h, w, generator=g).to(dev)
        mask = (torch.rand(B, 1, h, w, generator=g) > 0.1).float().to(dev)
        np.random.seed(1)
        pts = st.loss.vnl.select_index()
        fn = lambda st=st, b=(rgb, gt, mask), p=pts: st.step(*b, points=p, full_mix=True)
        for _ in range(3):
            fn()
        steps[(h, w)] = fn
    times = {k: [] for k in steps}
    for _ in range(5):
        for k, fn in steps.items():
            times[k].append(time_ms(fn, 10))
    for (h, w), ts in times.items():
        ts.sort()
        res[f"step_ms_{h}x{w}"] = {"median": round(ts[len(ts) // 2], 3), "min": round(ts[0], 3), "max": round(ts[-1], 3)}
        res[f"images_per_s_{h}x{w}"] = round(B / (ts[len(ts) // 2] * 1e-3), 1)
    line = json.dumps(res)
    print(line)
    if out_file:
        Path(out_file).parent.mkdir(parents=True, exist_ok=True)
        Path(out_file).write_text(line + "\n")


if __name__ == "__main__":
    main()
