"""Data-parallel plumbing for batched inference: one process per GPU (torch.distributed, NCCL on
GPUs / gloo in CPU tests).  Images are independent units, so the data path has NO collective:
the batch is split into contiguous per-rank slices, weights are broadcast once from rank 0, and
only scalars (timings, counts) are reduced.  The reference has no multi-GPU inference at all
(demo.py:41-42 uses cuda:0); its training path is PL DDP (train_depth.py:424-426).
"""
from __future__ import annotations

import os
from typing import Dict, Tuple

import torch
import torch.distributed as dist


def init_from_env(backend: str | None = None) -> Tuple[int, int, int]:
    """(rank, world_size, local_rank); initialises the default process group when WORLD_SIZE > 1."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        import datetime
        # a mismatched collective must fail fast (the default watchdog timeout is ten minutes of a hung GPU box)
        tmo = datetime.timedelta(seconds=int(os.environ.get("ODB_DIST_TIMEOUT_S", "180")))
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, rank=rank, world_size=world, device_id=torch.device("cuda", local), timeout=tmo)
        else:
            dist.init_process_group(backend, rank=rank, world_size=world, timeout=tmo)
    return rank, world, local


def shard_range(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous, balanced [start, end) slice of `n_items` for `rank` (first ranks take the remainder)."""
    base, rem = divmod(n_items, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def broadcast_state_dict(module: torch.nn.Module, src: int = 0, bucket_bytes: int = 64 << 20) -> int:
    """Broadcast every parameter / buffer of `module` from `src` in flat buckets; returns bytes sent."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return 0
    tensors = [t for t in module.state_dict().values() if torch.is_tensor(t)]
    total = 0
    bucket, size = [], 0

    def flush():
        nonlocal bucket, size, total
        if not bucket:
            return
        flat = torch.cat([t.reshape(-1).to(torch.float32) for t in bucket])
        dist.broadcast(flat, src=src)
        off = 0
        for t in bucket:
            n = t.numel()
            t.copy_(flat[off:off + n].view_as(t).to(t.dtype))
            off += n
        total += flat.numel() * 4
        bucket, size = [], 0

    with torch.no_grad():
        for t in tensors:
            bucket.append(t)
            size += t.numel() * 4
            if size >= bucket_bytes:
                flush()
        flush()
    return total


def _packed_tensors(pk):
    """Deterministic (name, tensor) walk of a packed operand table (schema: model.dpt_forward): pos_embed, then the
    GEMM operands and the fp32 vectors in key order.  The pos_cache derived from pos_embed is left out."""
    yield "pos", pk["pos"]
    for table in ("gemm", "vec"):
        for k in sorted(pk[table]):
            yield f"{table}.{k}", pk[table][k]


def broadcast_packed_weights(model, device, src: int = 0) -> int:
    """Inference weight distribution (SURVEY.md 8e): rank `src` packs its checkpoint into the layout the kernels
    consume (bf16 GEMM / conv operands, weight-standardised ResNetV2 filters, fp32 biases and norm affines) and that
    PACKED form — about 246 MB for DPT-Hybrid instead of the 493 MB fp32 state_dict — is broadcast, one flat buffer per
    storage type.  The other ranks never build the fp32 -> packed conversion of real weights; their nn.Parameters keep
    whatever they were initialised with and are not used by the inference path.  Returns the bytes sent."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return 0
    sig = model._weights_signature()
    if model._packed is None or model._packed_sig != sig:
        model._invalidate()
        model._packed = model._prepack(device)
        model._packed_sig = sig
    items = list(_packed_tensors(model._packed))
    total = 0
    with torch.no_grad():
        # precision "fp8": the e4m3 operands travel as their bytes (uint8 views)
        for dtype in (torch.bfloat16, torch.float32, torch.float8_e4m3fn):
            group = [t if dtype != torch.float8_e4m3fn else t.view(torch.uint8) for _, t in items if t.dtype == dtype]
            if not group:
                continue
            flat = torch.cat([t.reshape(-1) for t in group])
            dist.broadcast(flat, src=src)
            off = 0
            for t in group:
                n = t.numel()
                t.copy_(flat[off:off + n].view_as(t))
                off += n
            total += flat.numel() * flat.element_size()
    model._packed["pos_cache"] = {}
    model._graphs.clear()
    model._packed_sig = model._weights_signature()      # the received operands are current: the next forward must not re-pack
    return total


def packed_weights_identical(model, device) -> bool:
    """True when every rank holds bit-identical packed operands (checked after broadcast_packed_weights): per-tensor
    float64 checksums, MAX- and MIN-reduced."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return True
    sums = torch.stack([t.double().abs().sum() + t.double().sum() * 0.5 for _, t in _packed_tensors(model._packed)]).to(device)
    hi, lo = sums.clone(), sums.clone()
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    return bool(torch.equal(hi, lo))


def reduce_max(value: float, device) -> float:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def reduce_sum(value: float, device) -> float:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


def barrier():
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()
