"""Train step of the plain-ViT DPTs (DPT-Large `vitl16_384`, plain ViT-B `vitb16_384`): batch 16, bf16, 384x384.
For each backbone:
  * the captured DepthTrainStep (one CUDA graph per step, CUDA events, median over rounds): ms / step, images/s;
  * the kernel launches of one eager step (odb_launch_count);
  * executed GFLOP per image of one eager step, counted as profiles/large.py counts them (2 m n k of every GEMM launch,
    weight gradients included, plus the attention kernels' own counts);
  * odb_patch_input_grad alone (CUDA events over many launches) as GB/s of the bytes it moves, against the 3.35 TB/s
    HBM3 data-sheet bandwidth of the H100 SXM;
  * the yardstick: a stock torch.autocast(bfloat16) eager train step of the oracle network
    (oracle/plain_vit_oracle.py, torch autograd, clip_grad_norm_, torch.optim.Adam) on the same GPU, weights and
    batch, with a masked L1 loss in place of the depth loss mix (cheaper than the mix, so the comparison favours the
    yardstick).
The card's name, power limit and maximum SM clock are read in the same run.
python profiles/plain_vit_train.py [batch] [--out FILE] (one JSON line)."""
import gc
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from omnidata_b200 import _capi, bwd, ops, synthetic  # noqa: E402
from omnidata_b200.model import DPTDepthModel, state_dict_spec  # noqa: E402
from omnidata_b200.train import DepthTrainStep  # noqa: E402
from oracle import plain_vit_oracle  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


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
        raise SystemExit("profiles/plain_vit_train.py needs a CUDA device")
    dev = torch.device("cuda:0")
    H = W = 384
    res = {"batch": B, "size": [H, W], "dtype": "bf16", "gpu": gpu_info()}
    g = torch.Generator().manual_seed(0)
    rgb = (torch.rand(B, 3, H, W, generator=g) * 2 - 1).to(dev)
    gt = torch.rand(B, 1, H, W, generator=g).to(dev)
    mask = (torch.rand(B, 1, H, W, generator=g) > 0.1).float().to(dev)
    for backbone in ("vitl16_384", "vitb16_384"):
        sd = synthetic.make_state_dict(0, 1, spec=state_dict_spec(1, backbone=backbone))

        def make():
            m = DPTDepthModel(backbone=backbone)
            m.load_state_dict(sd)
            return DepthTrainStep(m.to(dev).train(), lr=1e-6, clip=10.0)

        r = {}
        # ---- one eager step: launches and executed GEMM / attention FLOP
        step = make()
        np.random.seed(11)
        step.step(rgb, gt, mask, full_mix=True)
        torch.cuda.synchronize()
        n0 = _capi.launch_count()
        with ops.LaunchTimer() as lt:
            step.step(rgb, gt, mask, full_mix=True)
        recs = lt.results()
        r["launches_eager"] = _capi.launch_count() - n0
        flops = 0.0
        for name, info, _ in recs:
            if name in ("odb_conv_gemm", "odb_conv_wgrad"):
                flops += 2.0 * info["m"] * info["n"] * info["k"]
            flops += info.get("flops", 0.0)
        r["gflop_per_image"] = flops / B / 1e9
        del step, lt, recs
        gc.collect()
        torch.cuda.empty_cache()
        # ---- the captured step, a fresh step per round
        times = []
        for _ in range(3):
            step = make()
            step.use_cuda_graph = True
            np.random.seed(11)
            for _ in range(3):
                step.step(rgb, gt, mask, full_mix=True)
            times.append(time_ms(lambda: step.step(rgb, gt, mask, full_mix=True), 10))
            del step
            gc.collect()
            torch.cuda.empty_cache()
        ms = median(times)
        r.update(step_ms_median=ms, step_ms_rounds=times, images_per_s=B * 1000.0 / ms,
                 executed_tflop_per_s=r["gflop_per_image"] * B / ms)
        # ---- the patch-embedding input gradient alone
        gh, gw = H // 16, W // 16
        dcols = torch.randn(B * gh * gw, 768, device=dev).to(torch.bfloat16)
        dx = torch.empty(B, 3, H, W, device=dev)
        run = lambda: bwd.patch_input_grad(dcols, dx)
        for _ in range(20):
            run()
        pig = median([time_ms(run, 200) for _ in range(3)])
        nbytes = dcols.numel() * 2 + dx.numel() * 4
        r["patch_input_grad"] = {"ms": pig, "bytes": nbytes, "GB_per_s": nbytes / pig / 1e6,
                                 "share_of_hbm_datasheet": nbytes / (pig * 1e-3) / HBM_BYTES_PER_S}
        del dcols, dx
        # ---- yardstick: stock autocast(bf16) eager train step of the oracle network
        leaves = {k: v.to(dev).float().requires_grad_(True) for k, v in sd.items()}
        opt = torch.optim.Adam(list(leaves.values()), lr=1e-6)
        target = gt[:, 0]

        def stock_step():
            opt.zero_grad(set_to_none=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                y = plain_vit_oracle.forward_fp32(leaves, rgb)
            loss = ((y.float() - target).abs() * mask[:, 0]).mean()
            loss.backward()
            torch.nn.utils.clip_grad_norm_(list(leaves.values()), 10.0)
            opt.step()
        for _ in range(2):
            stock_step()
        stock = median([time_ms(stock_step, 3) for _ in range(3)])
        r["stock_autocast_eager"] = {"step_ms": stock, "images_per_s": B * 1000.0 / stock,
                                     "speedup_of_captured_step": stock / ms}
        del leaves, opt
        gc.collect()
        torch.cuda.empty_cache()
        res[backbone] = r
        print(backbone, json.dumps(r), flush=True)
    line = json.dumps(res)
    print(line)
    if out_file:
        Path(out_file).parent.mkdir(parents=True, exist_ok=True)
        Path(out_file).write_text(line + "\n")


if __name__ == "__main__":
    main()
