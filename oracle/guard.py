"""Guarded launches for kernel tests: every tensor a launch touches lives in a buffer with >= 64 KiB guard bands on
both sides, filled with a seeded random pattern.  `checked_launch` runs a launch, verifies that it wrote every output
element and nothing else (inputs and guard bands stay bit-identical), and that a second run from the same state is
bit-identical."""
from __future__ import annotations

from typing import Callable, Sequence

import torch

GUARD_BYTES = 64 * 1024
_INT = {torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}


def bits(t: torch.Tensor) -> torch.Tensor:
    """The tensor's storage as integers: equality that also holds for NaN and tells -0 from 0."""
    return t.view(_INT[t.dtype])


class Guarded:
    """One allocation: guard band, `n` elements for the tensors under test, guard band.  Every element starts as a
    seeded N(0, 1) sample, so a window's neighbours hold non-zero values."""

    def __init__(self, n: int, dtype, gen: torch.Generator, device="cuda"):
        self.pad = GUARD_BYTES // torch.tensor([], dtype=dtype).element_size()
        self.t = torch.randn(n + 2 * self.pad, generator=gen, device=device).to(dtype)

    def view(self, shape, stride, offset: int = 0) -> torch.Tensor:
        return self.t.as_strided(tuple(shape), tuple(stride), self.pad + offset)

    def contiguous(self, *shape) -> torch.Tensor:
        strides, s = [], 1
        for d in reversed(shape):
            strides.insert(0, s)
            s *= d
        return self.view(shape, strides)

    def owns(self, v: torch.Tensor) -> bool:
        return v.untyped_storage().data_ptr() == self.t.untyped_storage().data_ptr()

    def mask(self, outs: Sequence[torch.Tensor]) -> torch.Tensor:
        m = torch.zeros(self.t.shape, dtype=torch.bool, device=self.t.device)
        for o in outs:
            if self.owns(o):
                m.as_strided(o.shape, o.stride(), o.storage_offset()).fill_(True)
        return m


def checked_launch(bufs: Sequence[Guarded], outs: Sequence[torch.Tensor], launch: Callable[[], None],
                   prefill_nan: bool = True):
    """Runs `launch` once (outputs prefilled with NaN when they neither accumulate nor alias an input) and checks that
    every output element is finite, that nothing outside the output elements changed, and that a second run from the
    same starting state writes bit-identical outputs.  Returns copies of the outputs."""
    if prefill_nan:
        for o in outs:
            o.fill_(float("nan"))
    snaps = [b.t.clone() for b in bufs]
    masks = [b.mask(outs) for b in bufs]
    launch()
    torch.cuda.synchronize()
    for i, (b, s, m) in enumerate(zip(bufs, snaps, masks)):
        changed = bits(b.t) != bits(s)
        assert not bool((changed & ~m).any()), f"buffer {i}: {int((changed & ~m).sum())} elements outside the output changed"
    for o in outs:
        assert bool(torch.isfinite(o).all()), f"{int((~torch.isfinite(o)).sum())} output elements not written / not finite"
    first = [o.clone() for o in outs]
    for b, s in zip(bufs, snaps):
        b.t.copy_(s)
    launch()
    torch.cuda.synchronize()
    for o, f in zip(outs, first):
        assert torch.equal(bits(o), bits(f)), "a second run is not bit-identical"
    return first


def _extent(t: torch.Tensor) -> int:
    return 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride())) if t.numel() else 0


def geometry(tensors: dict):
    """Tensors of one launch (name -> tensor or None) -> (groups, specs), hashable: one group per storage, spanning only
    what the tensors cover (plus the base's offset within 256 bytes, so alignment is kept); each tensor as (group,
    shape, stride, element offset in the group).  Aliasing between the tensors (in-place outputs, views of one
    buffer) is part of the geometry."""
    by_storage = {}
    for t in tensors.values():
        if t is not None:
            by_storage.setdefault(t.untyped_storage().data_ptr(), []).append(t)
    groups, where = [], {}
    for key, ts in by_storage.items():
        assert len({t.dtype for t in ts}) == 1
        es, base = ts[0].element_size(), min(t.data_ptr() for t in ts)
        lead = (base % 256) // es
        where[key] = (len(groups), base, lead, es)
        groups.append((max(lead + (t.data_ptr() - base) // es + _extent(t) for t in ts), ts[0].dtype))
    specs = []
    for name, t in tensors.items():
        if t is None:
            specs.append((name, None))
            continue
        gi, base, lead, es = where[t.untyped_storage().data_ptr()]
        specs.append((name, (gi, tuple(t.shape), tuple(t.stride()), lead + (t.data_ptr() - base) // es)))
    return tuple(groups), tuple(specs)


def materialize(geom, gen: torch.Generator):
    """A geometry -> (Guarded buffers, name -> tensor), every tensor at its recorded place in a fresh guarded buffer
    of seeded random values, so that the tensors alias each other exactly as they did when recorded."""
    groups, specs = geom
    bufs = [Guarded(n, dtype, gen) for n, dtype in groups]
    return bufs, {name: None if s is None else bufs[s[0]].view(s[1], s[2], s[3]) for name, s in specs}


def same_storage(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a is not None and b is not None and a.untyped_storage().data_ptr() == b.untyped_storage().data_ptr()


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values at |x| (8 significant bits), for |x| in the normal range; float64."""
    _, e = torch.frexp(x.double().abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), e - 8)
