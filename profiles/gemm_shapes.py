"""Per-shape times of the wgmma GEMM (`conv_gemm_kernel`) in the batch-32 DPT-Hybrid forward, single CTAs against
CTA pairs, and the in-kernel timeline of the four ViT-block shapes.  Prints one JSON line.

- shapes: every odb_conv_gemm launch of one eager forward is intercepted where the forward makes it (all its tensors
  live) and re-launched back to back, `reps` times as planned (`cta_pair` 0) and `reps` times as a CTA pair where
  the plan allows one (`cta_pair` 1), with CUDA events around each run; launches of one shape are aggregated.  The
  repeated launches write the layer's output (and an in-place residual) again: the forward's result is meaningless
  and only the times are kept.
- vit_trace: the %globaltimer stamps of odb_debug_conv_trace on the four ViT shapes (qkv, proj, fc1, fc2 with the
  fp32 residual stream the forward uses): per tile, the K-loop window (MMA start -> accumulator complete) and the
  epilogue window, median over all tiles of all CTAs, and the epilogue's share of the tile.

  python profiles/gemm_shapes.py [batch] [reps]
"""
import ctypes as C
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from omnidata_b200 import _capi, ops, synthetic  # noqa: E402
from omnidata_b200.model import DPTDepthModel  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power, clk = [s.strip() for s in out.strip().split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clk}
    except Exception as e:  # the measurement stands without it, but says so
        return {"name": torch.cuda.get_device_name(), "power_limit": f"not read ({type(e).__name__})"}


def sm_clock():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return out.strip()
    except Exception:
        return None


def epilogue_kind(d):
    if d.out_dtype == ops.DTYPE_F32:
        return "bias+res_f32"
    if d.head_out:
        return "head"
    if d.out2.ptr:
        return "generic(out2)"
    if d.gn_partial:
        return "gn"
    s = "bias" if d.bias else "nobias"
    if d.residual.ptr:
        s += "+res"
    return s + {ops.ACT_NONE: "", ops.ACT_RELU: "+relu", ops.ACT_GELU: "+gelu"}.get(d.act, "+act")


def time_launch(fn, args, stream, reps):
    for _ in range(2):
        _capi.check(fn(*args, stream), "odb_conv_gemm")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    rcs = [fn(*args, stream) for _ in range(reps)]
    e1.record()
    torch.cuda.synchronize()
    for rc in rcs:
        _capi.check(rc, "odb_conv_gemm")
    return e0.elapsed_time(e1) * 1e3 / reps       # us per launch


def shapes(batch, reps):
    lib = _capi.lib()
    model = DPTDepthModel()
    model.load_state_dict(synthetic.make_state_dict(0, 1))
    model = model.cuda().eval()
    model.use_cuda_graph = False
    x = torch.rand(batch, 3, 384, 384, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0)) * 2 - 1
    agg = {}
    orig = ops._call

    def intercept(name, info, fn, dev, *args):
        r = orig(name, info, fn, dev, *args)
        if name != "odb_conv_gemm" or info.get("f32"):
            return r
        d = args[0]._obj
        stream = torch.cuda.current_stream(dev).cuda_stream
        plan = (C.c_int32 * 4)()
        _capi.check(lib.odb_conv_gemm_plan(C.byref(d), plan), "plan")
        key = (epilogue_kind(d), info["m"], info["n"], info["k"], info["taps"], info["w"], info["h"])
        a = agg.setdefault(key, {"launches": 0, "block_n": plan[2], "tile": [plan[0], plan[1]],
                                 "single_us": [], "pair_us": []})
        a["launches"] += 1
        saved = d.cta_pair
        d.cta_pair = 0
        a["single_us"].append(time_launch(fn, args, stream, reps))
        d.cta_pair = 1
        if lib.odb_conv_gemm_plan(C.byref(d), plan) == 0:
            a["pair_us"].append(time_launch(fn, args, stream, reps))
        d.cta_pair = saved
        return r

    with torch.no_grad():
        model(x)
        torch.cuda.synchronize()
        ops._call = intercept
        try:
            model(x)
        finally:
            ops._call = orig
        torch.cuda.synchronize()
    rows, tot_single, tot_best = [], 0.0, 0.0
    for (kind, m, n, k, taps, w, h), a in sorted(agg.items(), key=lambda kv: -sum(kv[1]["single_us"])):
        s = sum(a["single_us"]) / len(a["single_us"])
        p = sum(a["pair_us"]) / len(a["pair_us"]) if a["pair_us"] else None
        fl = 2.0 * m * n * k
        tot_single += s * a["launches"]
        tot_best += min(s, p if p is not None else s) * a["launches"]
        rows.append({"epilogue": kind, "m": m, "n": n, "k": k, "taps": taps, "out_wh": [w, h], "tile": a["tile"],
                     "block_n": a["block_n"], "m_tiles": -(-m // 128), "k_blocks": -(-k // 64),
                     "launches_per_forward": a["launches"],
                     "single_us": round(s, 1), "single_tflops": round(fl / s / 1e6, 1),
                     "pair_us": round(p, 1) if p is not None else None,
                     "pair_tflops": round(fl / p / 1e6, 1) if p is not None else None,
                     "pair_over_single": round(s / p, 3) if p is not None else None})
    return {"per_shape": rows, "forward_gemm_ms_single": round(tot_single / 1e3, 3),
            "forward_gemm_ms_best_of_both": round(tot_best / 1e3, 3)}


def vit_trace(batch):
    dev = torch.device("cuda")
    rows = batch * 577
    g = torch.Generator().manual_seed(0)

    def rnd(*s, scale=1.0, dtype=torch.bfloat16):
        return (torch.randn(*s, generator=g) * scale).to(dev).to(dtype)

    x768, x3072 = rnd(rows, 768), rnd(rows, 3072)
    res32 = rnd(rows, 768, dtype=torch.float32)
    cases = {
        "qkv": (x768, 2304, torch.bfloat16, {}),
        "proj": (x768, 768, torch.float32, {"residual": res32}),
        "fc1": (x768, 3072, torch.bfloat16, {"act": ops.ACT_GELU}),
        "fc2": (x3072, 768, torch.float32, {"residual": res32}),
    }
    lib = _capi.lib()
    slots = lib.odb_debug_conv_trace(None)
    ctas = 2 * torch.cuda.get_device_properties(0).multi_processor_count
    trace = torch.zeros(ctas * slots, dtype=torch.int64, device=dev)
    res = {}
    for name, (xin, n, odt, kw) in cases.items():
        k = xin.shape[1]
        w = rnd(n, k, scale=0.03)
        bias = rnd(n, dtype=torch.float32)
        out = torch.empty(rows, n, device=dev, dtype=odt)
        for _ in range(3):
            ops.linear(xin, w, out, bias=bias, **kw)
        torch.cuda.synchronize()
        trace.zero_()
        lib.odb_debug_conv_trace(trace.data_ptr())
        ops.linear(xin, w, out, bias=bias, **kw)
        torch.cuda.synchronize()
        lib.odb_debug_conv_trace(None)
        t = trace.view(ctas, slots).cpu()
        t = t[t[:, 0] > 0]
        kloop, epi = [], []
        for r in t:
            for i in range(24):
                ev = [int(v) for v in r[8 + 5 * i: 8 + 5 * i + 5]]
                if ev[0] == 0 or ev[4] == 0:
                    break
                kloop.append((ev[2] - ev[0]) / 1e3)
                epi.append((ev[4] - ev[3]) / 1e3)
        kl, ep = torch.tensor(kloop).median().item(), torch.tensor(epi).median().item()
        span = (int(t[:, 2].max()) - int(t[:, 0].min())) / 1e3
        res[name] = {"n": n, "k": k, "tiles": len(kloop), "kloop_us_median": round(kl, 2),
                     "epilogue_us_median": round(ep, 2), "epilogue_share": round(ep / (kl + ep), 3),
                     "kernel_span_us": round(span, 1), "tflops_traced": round(2.0 * rows * n * k / span / 1e6, 1)}
    return res


def main():
    batch = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    if not torch.cuda.is_available():
        raise SystemExit("gemm_shapes.py: no CUDA device")
    info = card()
    out = {"card": info, "batch": batch, "reps": reps}
    out.update(shapes(batch, reps))
    out["sm_clock_after_shapes"] = sm_clock()
    out["vit_trace"] = vit_trace(batch)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
