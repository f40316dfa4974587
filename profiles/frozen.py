"""Cost of a partly or fully frozen DPT-Hybrid at batch 16, bf16, 384x384, CUDA events (medians over alternated runs):
  (a) forward + backward for x.grad through autograd, every parameter frozen vs every parameter requiring grad;
  (b) the captured DepthTrainStep with every parameter trainable, with the encoder (pretrained.*) frozen and with the
      ResNetV2 frozen.
Launch counts are those of one eager call.  python profiles/frozen.py [batch] [--out FILE] (one JSON line)."""
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
from omnidata_b200.model import DPTDepthModel  # noqa: E402
from omnidata_b200.train import DepthTrainStep  # noqa: E402

BB = "pretrained.model.patch_embed.backbone."
STEP_VARIANTS = {"all_trainable": lambda n: True, "encoder_frozen": lambda n: n.startswith("scratch."),
                 "resnet_frozen": lambda n: not n.startswith(BB)}


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


def model(dev, trainable=lambda n: True):
    m = DPTDepthModel()
    m.load_state_dict(synthetic.make_state_dict(0, 1))
    m = m.to(dev).train()
    for n, p in m.named_parameters():
        p.requires_grad_(trainable(n))
    return m


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
        raise SystemExit("profiles/frozen.py needs a CUDA device")
    dev = torch.device("cuda:0")
    H = W = 384
    res = {"batch": B, "size": [H, W], "dtype": "bf16", "gpu": gpu_info()}
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(dev)
    R = torch.randn(B, H, W, generator=g).to(dev)

    # ---- (a) x.grad of sum(model(x) * R): all frozen (eval) vs all requiring grad (train), alternated
    m = model(dev)

    def input_grad(frozen):
        m.eval() if frozen else m.train()
        m.requires_grad_(not frozen)
        for p in m.parameters():
            p.grad = None
        xi = x.clone().requires_grad_(True)
        (m(xi) * R).sum().backward()

    counts = {k: launches(lambda: input_grad(k == "frozen")) for k in ("trainable", "frozen")}
    t = {"trainable": [], "frozen": []}
    for _ in range(2):
        input_grad(False); input_grad(True)
    for _ in range(7):
        for k in ("trainable", "frozen"):
            t[k].append(time_ms(lambda: input_grad(k == "frozen"), 1))
    res["input_grad"] = {"ms_median": {k: median(v) for k, v in t.items()}, "ms_min": {k: min(v) for k, v in t.items()},
                         "launches": counts}
    del m
    gc.collect()
    torch.cuda.empty_cache()

    # ---- (b) the captured train step per trainable set, the variants alternated over rounds
    rgb = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(dev)
    gt = torch.rand(B, 1, H, W, generator=g).to(dev)
    mask = (torch.rand(B, 1, H, W, generator=g) > 0.1).float().to(dev)
    times = {k: [] for k in STEP_VARIANTS}
    counts = {}
    for rnd in range(3):
        for name, pred in STEP_VARIANTS.items():
            step = DepthTrainStep(model(dev, pred), lr=1e-6, clip=10.0)
            np.random.seed(11)
            if rnd == 0:
                counts[name] = launches(lambda: step.step(rgb, gt, mask, full_mix=False))
            step.use_cuda_graph = True
            for _ in range(3):
                step.step(rgb, gt, mask, full_mix=False)
            times[name].append(time_ms(lambda: step.step(rgb, gt, mask, full_mix=False), 10))
            del step
            gc.collect()
            torch.cuda.empty_cache()
    res["train_step_graph"] = {"ms_median": {k: median(v) for k, v in times.items()},
                               "ms_min": {k: min(v) for k, v in times.items()}, "launches_eager": counts}
    line = json.dumps(res)
    print(line)
    if out_file:
        Path(out_file).parent.mkdir(parents=True, exist_ok=True)
        Path(out_file).write_text(line + "\n")


if __name__ == "__main__":
    main()
