"""Train step of the surface-normal DPT-Hybrid next to the depth one: batch 16, bf16, 384x384, both replayed as one CUDA
graph per step and alternated over rounds in one process (CUDA events; medians over rounds).
  * NormalTrainStep and DepthTrainStep (full loss mix: MiDaS + gradient matching + virtual normal): ms / step, images/s;
  * NormalStepLoss alone (make_valid_mask + loss forward + loss backward over [16,3,384,384]): ms / call over many calls;
  * the kernel launches of one eager step of each (odb_launch_count);
  * the card's name, power limit and maximum SM clock, read in the same run.
python profiles/normal_train.py [batch] [--out FILE] (one JSON line)."""
import gc
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from omnidata_b200 import _capi, synthetic  # noqa: E402
from omnidata_b200.losses import NormalStepLoss  # noqa: E402
from omnidata_b200.model import DPTDepthModel  # noqa: E402
from omnidata_b200.train import DepthTrainStep, NormalTrainStep  # noqa: E402


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


def launches(fn):
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    fn()
    torch.cuda.synchronize()
    return _capi.launch_count() - n0


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def main():
    argv = sys.argv[1:]
    out_file = None
    if "--out" in argv:
        i = argv.index("--out")
        out_file = argv[i + 1]
        del argv[i:i + 2]
    B = int(argv[0]) if argv else 16
    if not torch.cuda.is_available():
        raise SystemExit("profiles/normal_train.py needs a CUDA device")
    dev = torch.device("cuda:0")
    H = W = 384
    res = {"batch": B, "size": [H, W], "dtype": "bf16", "gpu": gpu_info()}
    g = torch.Generator().manual_seed(0)
    rgb = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(dev)
    mask = (torch.rand(B, 1, H, W, generator=g) > 0.1).float().to(dev)
    targets = {"normal": torch.rand(B, 3, H, W, generator=g).to(dev), "depth": torch.rand(B, 1, H, W, generator=g).to(dev)}
    classes = {"normal": (NormalTrainStep, 3), "depth": (DepthTrainStep, 1)}

    def make(task):
        cls, c = classes[task]
        m = DPTDepthModel(num_channels=c)
        m.load_state_dict(synthetic.make_state_dict(0, c))
        return cls(m.to(dev).train(), lr=1e-6, clip=10.0)

    def run(task, step):
        return step.step(rgb, targets[task], mask) if task == "normal" else step.step(rgb, targets[task], mask,
                                                                                       full_mix=True)

    # ---- the two captured steps, alternated over rounds (a fresh step per round: capture, warm-up, timed replays)
    times = {k: [] for k in classes}
    counts = {}
    for rnd in range(4):
        for task in classes:
            step = make(task)
            np.random.seed(11)
            if rnd == 0:
                counts[task] = launches(lambda: run(task, step))
            step.use_cuda_graph = True
            for _ in range(3):
                run(task, step)
            times[task].append(time_ms(lambda: run(task, step), 10))
            del step
            gc.collect()
            torch.cuda.empty_cache()
    ms = {k: median(v) for k, v in times.items()}
    res["train_step_graph"] = {"ms_median": ms, "ms_min": {k: min(v) for k, v in times.items()},
                               "ms_rounds": times, "images_per_s": {k: B * 1000.0 / v for k, v in ms.items()},
                               "normal_over_depth": ms["normal"] / ms["depth"], "launches_eager": counts}

    # ---- NormalStepLoss alone on a network-shaped prediction
    pred = (targets["normal"] + 0.25 * torch.randn(B, 3, H, W, generator=g).to(dev)) * 1.2 - 0.1
    fn = NormalStepLoss()
    res["normal_step_loss"] = {"launches": launches(lambda: fn(pred, targets["normal"], mask))}
    for _ in range(20):
        fn(pred, targets["normal"], mask)
    loss_ms = [time_ms(lambda: fn(pred, targets["normal"], mask), 200) for _ in range(5)]
    res["normal_step_loss"].update(ms_median=median(loss_ms), ms_min=min(loss_ms),
                                   share_of_normal_step=median(loss_ms) / ms["normal"])
    line = json.dumps(res)
    print(line)
    if out_file:
        Path(out_file).parent.mkdir(parents=True, exist_ok=True)
        Path(out_file).write_text(line + "\n")


if __name__ == "__main__":
    main()
