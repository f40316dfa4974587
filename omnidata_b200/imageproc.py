"""Device-side image pre- / post-processing of the demo path (SURVEY.md 8(f) rank 1).

Reference (omnidata_tools/torch/demo.py):
  :74-76, :92-95   trans_totensor = Resize(384, BILINEAR) -> CenterCrop(384) -> ToTensor [-> Normalize(0.5, 0.5)]
  :137-138         a single-channel image is repeated to three channels
  :140-145         depth: clamp(0,1) -> F.interpolate((512,512), 'bicubic') -> clamp(0,1) -> 1 - x
  :150             normal: ToPILImage (x * 255 truncated to uint8, HWC)

`Resize` on a PIL image is Pillow's ImagingResample: antialiased, two passes, 8-bit fixed point.  The host
part below restates Pillow's coefficient generation (src/libImaging/Resample.c: precompute_coeffs,
normalize_coeffs_8bpc; bilinear_filter, support 1.0) in the same double-precision arithmetic; the
kernels (csrc/imageproc.cu) do the per-pixel integer work.  Result: the network input is bit-identical
to the reference's, with the decoded image uploaded once as uint8 (3 bytes / pixel) instead of a float
tensor prepared on the CPU.
"""
from __future__ import annotations

import ctypes as C
import math
from functools import lru_cache
from typing import Optional, Tuple

import numpy as np
import torch

from . import _capi
from ._capi import check, lib

PRECISION_BITS = 32 - 8 - 2          # Pillow Resample.c


def resized_size(w: int, h: int, size: int) -> Tuple[int, int]:
    """torchvision.transforms.Resize(size) for an int size: the shorter edge becomes `size`."""
    if w <= h:
        return size, int(size * h / w)
    return int(size * w / h), size


def center_crop_offset(full: int, crop: int) -> int:
    """torchvision center_crop: int(round((full - crop) / 2.0))."""
    return int(round((full - crop) / 2.0))


@lru_cache(maxsize=256)
def bilinear_aa_weights(in_size: int, out_size: int):
    """Pillow precompute_coeffs for the BILINEAR filter over the full axis, before the 8-bit step: a triangle filter
    whose support scales with the downsampling factor, each output's taps normalised to sum 1 in double precision.
    It is also torch's F.interpolate(mode="bilinear", align_corners=False, antialias=True) coefficient rule.
    Returns (bounds int32 [out_size, 2] = (xmin, count), weights float64 [out_size, ksize], ksize)."""
    in0, in1 = 0.0, float(in_size)
    scale = (in1 - in0) / out_size
    filterscale = scale if scale >= 1.0 else 1.0
    support = 1.0 * filterscale                      # bilinear: filter support 1.0
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    weights = np.zeros((out_size, ksize), dtype=np.float64)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = in0 + (xx + 0.5) * scale
        xmin = int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        xmax -= xmin
        ws = []
        ww = 0.0
        for x in range(xmax):
            a = (x + xmin - center + 0.5) * ss
            if a < 0.0:
                a = -a
            w = 1.0 - a if a < 1.0 else 0.0          # bilinear_filter
            ws.append(w)
            ww += w
        for x in range(xmax):
            w = ws[x]
            if ww != 0.0:
                w /= ww
            weights[xx, x] = w
        bounds[xx, 0] = xmin
        bounds[xx, 1] = xmax
    return bounds, weights, ksize


@lru_cache(maxsize=256)
def pil_bilinear_coeffs(in_size: int, out_size: int):
    """Pillow precompute_coeffs + normalize_coeffs_8bpc for the BILINEAR filter over the full axis.
    Returns (bounds int32 [out_size, 2] = (xmin, count), kk int32 [out_size, ksize], ksize)."""
    bounds, weights, ksize = bilinear_aa_weights(in_size, out_size)
    kk = np.zeros((out_size, ksize), dtype=np.int32)
    for xx in range(out_size):
        for x in range(int(bounds[xx, 1])):
            w = float(weights[xx, x])
            v = w * (1 << PRECISION_BITS)
            kk[xx, x] = int(-0.5 + v) if w < 0 else int(0.5 + v)
    return bounds, kk, ksize


@lru_cache(maxsize=64)
def resample_tables(in_size: int, out_size: int, device: torch.device):
    """bilinear_aa_weights resident on `device`: (bounds int32 [out_size, 2], weights fp32 [out_size, ksize], ksize),
    cached per (size, device) as the preprocessing plans are."""
    bounds, weights, ksize = bilinear_aa_weights(in_size, out_size)
    return (torch.from_numpy(bounds).to(device), torch.from_numpy(weights.astype(np.float32)).to(device), ksize)


class _Plan:
    """Coefficient tables of one (source size -> size, crop) geometry, resident on the device."""

    def __init__(self, src_w: int, src_h: int, size: int, device):
        nw, nh = resized_size(src_w, src_h, size)
        left, top = center_crop_offset(nw, size), center_crop_offset(nh, size)
        if left < 0 or top < 0:
            raise _capi.OdbError("imageproc: image smaller than the crop after Resize — not produced by Resize(size)")
        bh, kh, self.ksize_h = pil_bilinear_coeffs(src_w, nw)
        bv, kv, self.ksize_v = pil_bilinear_coeffs(src_h, nh)
        bh, kh = bh[left:left + size], kh[left:left + size]
        bv, kv = bv[top:top + size], kv[top:top + size]
        self.row0 = int(bv[:, 0].min())
        self.nrows = int((bv[:, 0] + bv[:, 1]).max()) - self.row0
        self.size = size
        self.bounds_h = torch.from_numpy(np.ascontiguousarray(bh)).to(device)
        self.kk_h = torch.from_numpy(np.ascontiguousarray(kh)).to(device)
        self.bounds_v = torch.from_numpy(np.ascontiguousarray(bv)).to(device)
        self.kk_v = torch.from_numpy(np.ascontiguousarray(kv)).to(device)


class DevicePreprocessor:
    """demo.py's `trans_totensor` for 8-bit images, on the device.

        pre = DevicePreprocessor(task='depth')            # or 'normal'
        x = pre(img_u8)                                     # uint8 [H, W, 3] / [H, W] (host or device) -> fp32 [3,384,384]

    `task='depth'` applies Normalize(mean=0.5, std=0.5) (demo.py:92-95); 'normal' stops after ToTensor."""

    def __init__(self, task: str = "depth", size: int = 384, device="cuda:0"):
        if task not in ("depth", "normal"):
            raise ValueError("task should be one of the following: normal, depth")
        self.normalize = task == "depth"
        self.size = size
        self.device = torch.device(device)
        self._plans = {}

    def _plan(self, w: int, h: int) -> _Plan:
        key = (w, h)
        if key not in self._plans:
            self._plans[key] = _Plan(w, h, self.size, self.device)
        return self._plans[key]

    @_capi.on_tensor_device
    def __call__(self, img, out: Optional[torch.Tensor] = None, out_u8: Optional[torch.Tensor] = None) -> torch.Tensor:
        if not isinstance(img, torch.Tensor):
            img = torch.from_numpy(np.array(img))              # (copy: PIL buffers are read-only)
        if img.dtype != torch.uint8 or img.dim() not in (2, 3):
            raise _capi.OdbError("imageproc: expected a uint8 image [H, W] or [H, W, C]")
        if img.dim() == 2:
            img = img.unsqueeze(-1)
        if img.shape[2] == 4:
            raise _capi.OdbError("imageproc: RGBA is resized premultiplied by Pillow — convert on the host first")
        if img.shape[2] not in (1, 3):
            raise _capi.OdbError("imageproc: 1 or 3 channels")
        if not img.is_cuda:
            img = img.to(self.device, non_blocking=True)      # 1 or 3 bytes per pixel over PCIe
        img = img.contiguous()
        h, w, c = img.shape
        plan = self._plan(w, h)
        s = self.size
        if out is None:
            out = torch.empty(3, s, s, device=self.device, dtype=torch.float32)
        tmp = torch.empty(plan.nrows * s * c, device=self.device, dtype=torch.uint8)
        check(lib().odb_pil_resize_crop_to_tensor(
            img.data_ptr(), h, w, c, w * c, plan.bounds_h.data_ptr(), plan.kk_h.data_ptr(), plan.ksize_h,
            plan.bounds_v.data_ptr(), plan.kk_v.data_ptr(), plan.ksize_v, plan.row0, plan.nrows, s, s,
            1 if self.normalize else 0, 0.5, 0.5, tmp.data_ptr(), out.data_ptr(),
            None if out_u8 is None else out_u8.data_ptr(), torch.cuda.current_stream().cuda_stream),
            "odb_pil_resize_crop_to_tensor")
        return out


@_capi.on_tensor_device
def bicubic_resize(x: torch.Tensor, size: Tuple[int, int], *, clamp_in: bool = False, clamp_out: bool = False,
                   invert: bool = False) -> torch.Tensor:
    """F.interpolate(x, size, mode='bicubic') for fp32 [..., h, w] with demo.py's clamps / 1 - x fused."""
    if not x.is_cuda or x.dtype != torch.float32:
        raise _capi.OdbError("bicubic_resize: fp32 CUDA tensor expected (no CPU path exists)")
    x = x.contiguous()
    ih, iw = x.shape[-2:]
    planes = x.numel() // (ih * iw)
    out = torch.empty(*x.shape[:-2], size[0], size[1], device=x.device, dtype=torch.float32)
    flags = (1 if clamp_in else 0) | (2 if clamp_out else 0) | (4 if invert else 0)
    check(lib().odb_bicubic_resize_f32(x.data_ptr(), planes, ih, iw, size[0], size[1], flags, out.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "odb_bicubic_resize_f32")
    return out


@_capi.on_tensor_device
def to_uint8_hwc(x: torch.Tensor, clamp01: bool = True) -> torch.Tensor:
    """transforms.ToPILImage() arithmetic for a float [C, H, W] tensor: uint8 [H, W, C] = trunc(x * 255)."""
    if not x.is_cuda or x.dtype != torch.float32 or x.dim() != 3:
        raise _capi.OdbError("to_uint8_hwc: fp32 CUDA tensor [C, H, W] expected")
    x = x.contiguous()
    c, h, w = x.shape
    out = torch.empty(h, w, c, device=x.device, dtype=torch.uint8)
    check(lib().odb_f32_chw_to_u8_hwc(x.data_ptr(), c, h, w, 1 if clamp01 else 0, out.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream), "odb_f32_chw_to_u8_hwc")
    return out
