"""Cost of the input-image gradient (odb_stem_input_grad) at batch 16, bf16, 384x384, CUDA events:
  * the kernel alone over many launches, its FLOP/s and share of the FP32 data-sheet rate;
  * TrainEngine.backward with and without dx (alternated, same saved forward).
python profiles/input_grad.py [batch] [--out FILE]   (prints one JSON line; --out also writes it to FILE)"""
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from omnidata_b200 import bwd, synthetic  # noqa: E402
from omnidata_b200.model import DPTDepthModel  # noqa: E402
from omnidata_b200.train import TrainEngine  # noqa: E402

FP32_PEAK = 67e12          # H100 SXM data sheet, dense FP32 (700 W)


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
        raise SystemExit("profiles/input_grad.py needs a CUDA device")
    dev = torch.device("cuda:0")
    H = W = 384
    res = {"batch": B, "size": [H, W], "dtype": "bf16", "gpu": gpu_info()}

    # ---- the kernel alone
    g = torch.Generator().manual_seed(0)
    ds0 = torch.randn(B, H // 2, W // 2, 64, generator=g).to(dev, torch.bfloat16)
    wp = torch.zeros(64, 160)
    wp[:, :147] = torch.randn(64, 147, generator=g)
    wp = wp.to(dev, torch.bfloat16)
    dx = torch.empty(B, 3, H, W, device=dev)
    run = lambda: bwd.stem_input_grad(ds0, wp, dx)
    time_ms(run, 20)
    t_kernel = min(time_ms(run, 200) for _ in range(3))
    flops = 2.0 * B * (H // 2) * (W // 2) * 64 * 147
    res["kernel_ms"] = t_kernel
    res["kernel_tflops"] = flops / (t_kernel * 1e-3) / 1e12
    res["kernel_share_of_fp32_datasheet"] = flops / (t_kernel * 1e-3) / FP32_PEAK
    res["kernel_gbytes_per_s"] = (ds0.numel() * 2 + dx.numel() * 4) / (t_kernel * 1e-3) / 1e9

    # ---- the engine's backward with and without dx
    model = DPTDepthModel()
    model.load_state_dict(synthetic.make_state_dict(0, 1))
    model = model.to(dev).train()
    eng = TrainEngine(model, precision="bf16")
    x = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(dev)
    dout = torch.randn(B, 1, H, W, generator=g).to(dev)
    eng.forward(x)
    without = lambda: eng.backward(dout)
    with_dx = lambda: eng.backward(dout, dx=dx)
    for _ in range(3):
        without(); with_dx()
    t0, t1 = [], []
    for _ in range(8):
        t0.append(time_ms(without, 2))
        t1.append(time_ms(with_dx, 2))
    t0.sort(); t1.sort()
    res["backward_ms"] = {"without_dx_median": t0[len(t0) // 2], "with_dx_median": t1[len(t1) // 2],
                          "without_dx_min": t0[0], "with_dx_min": t1[0]}
    line = json.dumps(res)
    print(line)
    if out_file:
        Path(out_file).parent.mkdir(parents=True, exist_ok=True)
        Path(out_file).write_text(line + "\n")


if __name__ == "__main__":
    main()
