"""High-resolution inference on one GPU: for the three backbones at 384^2, 512^2, 768^2 and 1024^2, batch 8 and 1,
  * images/s of the captured bf16 forward (CUDA graph, CUDA events around 10 replays after 3 warm-up calls);
  * the attention kernel's time per forward and its share of the summed launch times of one eager forward
    (ops.LaunchTimer: CUDA events around every launch), and its TFLOP/s counted as 4 T^2 64 heads per block and
    image (the pass-1 recompute of S excluded);
  * at 512^2 and 1024^2, stock torch.autocast(bfloat16) eager of the oracle network (oracle/dpt_oracle.py,
    oracle/plain_vit_oracle.py) as the yardstick.
The card's name and power limit are printed first.    python profiles/highres.py > highres.txt"""
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from omnidata_b200 import ops, synthetic  # noqa: E402
from omnidata_b200.model import DPTDepthModel, state_dict_spec  # noqa: E402
from oracle import dpt_oracle, plain_vit_oracle  # noqa: E402

BACKBONES = ("vitb_rn50_384", "vitl16_384", "vitb16_384")
SIZES = (384, 512, 768, 1024)
BATCHES = (8, 1)


def _timed(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    print(f"device: {torch.cuda.get_device_name(0)}; nvidia-smi name, power limit, max SM clock: {q}")
    for backbone in BACKBONES:
        sd = synthetic.make_state_dict(0, 1, spec=state_dict_spec(1, backbone=backbone))
        model = DPTDepthModel(backbone=backbone)
        model.load_state_dict(sd)
        model = model.cuda().eval()
        sdg = {k: v.cuda() for k, v in sd.items()}
        oracle = dpt_oracle.forward_fp32 if backbone == "vitb_rn50_384" else plain_vit_oracle.forward_fp32
        for size in SIZES:
            for batch in BATCHES:
                x = torch.rand(batch, 3, size, size, device="cuda") * 2 - 1
                with torch.no_grad():
                    model.use_cuda_graph = True
                    ms = _timed(lambda: model(x))
                    model.use_cuda_graph = False
                    model(x)
                    with ops.LaunchTimer() as lt:
                        model(x)
                    recs = lt.results()
                tot = sum(t for _, _, t in recs)
                att = [(info, t) for name, info, t in recs if name == "odb_attention"]
                att_ms = sum(t for _, t in att)
                att_flop = sum(info["flops"] for info, _ in att)
                line = (f"{backbone} {size}x{size} batch {batch}: {ms:.3f} ms = {batch / ms * 1e3:.1f} images/s (graph); "
                        f"attention {len(att)} launches {att_ms:.3f} ms = {100 * att_ms / tot:.1f} % of {tot:.3f} ms "
                        f"launch time, {att_flop / att_ms / 1e9:.0f} TFLOP/s")
                if size in (512, 1024):
                    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                        ams = _timed(lambda: oracle(sdg, x), iters=3, warmup=1)
                    line += f"; stock autocast eager {ams:.3f} ms = {batch / ams * 1e3:.1f} images/s"
                print(line, flush=True)
                model._workspaces.clear()
                model._graphs.clear()
                del x
                torch.cuda.empty_cache()
        del model, sdg
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
