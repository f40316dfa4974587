"""Cost of one DepthMetrics / NormalMetrics update (omnidata_b200/metrics.py) at 384x384 batch 32 and at 4032x3024
batch 1, with a uint8 mask: device time per update (the update captured in a CUDA graph and replayed, CUDA events), the
bytes it must move, the achieved GB/s against the 3.35 TB/s HBM3 data-sheet figure, and its share of the bf16
CUDA-graph forward of the same batch (model(x) at 384x384; TiledPredictor, tile 384 overlap 64, at 4032x3024).  The
card's name and power limit are read in the same run.

    python profiles/metrics.py [--iters 50] [--out FILE]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from omnidata_b200.metrics import DepthMetrics, NormalMetrics      # noqa: E402
from omnidata_b200.model import DPTDepthModel                      # noqa: E402
from omnidata_b200.tiled import TiledPredictor                     # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SIZES = [(32, 384, 384), (1, 3024, 4032)]


def device_ms(fn, iters):
    """Mean device time of fn() over `iters` calls, after warm-up."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def graphed(fn):
    fn()                                               # first call at the shape allocates
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st), torch.cuda.graph(g, stream=st):
        fn()
    torch.cuda.current_stream().wait_stream(st)
    return g.replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--fwd_iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profiles/metrics.py measures on a CUDA device; none found")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    torch.manual_seed(0)
    rows = []
    for task, c in (("depth", 1), ("normal", 3)):
        model = DPTDepthModel(backbone="vitb_rn50_384", num_channels=c).cuda().eval()
        model.use_cuda_graph = True
        for b, h, w in SIZES:
            px = b * h * w
            mask = (torch.rand(b, h, w, device="cuda") > 0.1).to(torch.uint8)
            if task == "depth":
                pred, gt = torch.rand(b, h, w, device="cuda"), torch.rand(b, h, w, device="cuda") * 10 + 0.5
                metric = DepthMetrics(space="disparity", max_depth=10.0)
                nbytes = 2 * px * (4 + 4 + 1)                  # prediction, ground truth and mask, read in both passes
            else:
                pred, gt = torch.rand(b, 3, h, w, device="cuda"), torch.rand(b, 3, h, w, device="cuda")
                metric = NormalMetrics()
                nbytes = px * (12 + 12 + 1)                    # one pass; histogram increments not counted
            upd = device_ms(graphed(lambda: metric.update(pred, gt, mask)), a.iters)
            x = torch.rand(b, 3, h, w, device="cuda")
            with torch.no_grad():
                if h * w <= 4096 * 256:
                    fwd = device_ms(lambda: model(x), a.fwd_iters)
                else:
                    tp = TiledPredictor(model, tile=(384, 384), overlap=64, max_batch=32)
                    fwd = device_ms(lambda: tp(x), max(1, a.fwd_iters // 3))
            r = {"task": task, "batch": b, "size": f"{w}x{h}", "update_us": round(upd * 1000, 1),
                 "bytes_MB": round(nbytes / 1e6, 1), "GBps": round(nbytes / (upd * 1e-3) / 1e9, 1),
                 "share_of_hbm": round(nbytes / (upd * 1e-3) / HBM_BYTES_PER_S, 3),
                 "forward_ms": round(fwd, 2), "share_of_forward": round(upd / fwd, 5)}
            print(json.dumps(r), flush=True)
            rows.append(r)
        del model
        torch.cuda.empty_cache()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps({"card": card, "results": rows}, indent=1))


if __name__ == "__main__":
    main()
