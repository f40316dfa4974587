"""Depth-training losses of omnidata_tools/torch, forward pass on the GPU (C ABI, csrc/loss.cu).

Same constructor / call signatures as the reference modules (losses/midas_loss.py:137-157,
losses/virtual_normal_loss.py:7-27,151-194) and the loss mix of train_depth.py:261-279.  MidasLoss and VNL_Loss
are differentiable with respect to the prediction (odb_midas_loss_bwd / odb_vnl_loss_bwd behind torch.autograd), so
`depth_step_losses(...)["depth_loss"].backward()` yields d(loss)/d(depth_preds) — the first step of the train
step's backward pass; so is the normal-training pair (odb_normal_loss_bwd).  DepthStepLoss and NormalStepLoss are the
same arithmetic as one fixed, sync-free launch sequence that also returns d(loss)/d(prediction): the train steps' loss.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _capi
from ._capi import check, lib


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _capi.OdbError(f"{name}: CUDA tensor required (no CPU path)")
    return t.detach().float().contiguous()


@_capi.on_tensor_device
def make_valid_mask(mask_float: torch.Tensor, max_pool_size: int = 4) -> torch.Tensor:
    """train_depth.py:215-242 (the 4-D [B,1,H,W] case): bool mask of pixels whose 4x4 cell is fully valid."""
    if mask_float.dim() == 3:
        mask_float = mask_float.unsqueeze(0)
    elif mask_float.dim() == 2:
        mask_float = mask_float.unsqueeze(0).unsqueeze(0)
    m = _f32(mask_float, "mask_float")
    b, c, h, w = m.shape
    out = torch.empty((b, c, h, w), dtype=torch.uint8, device=m.device)
    check(lib().odb_make_valid_mask(m.data_ptr(), out.data_ptr(), b * c, h, w, max_pool_size, _stream()),
          "odb_make_valid_mask")
    return out.bool()


class MidasLoss(torch.nn.Module):
    def __init__(self, alpha: float = 0.1, scales: int = 4, reduction: str = "image-based"):
        super().__init__()
        if reduction != "image-based":
            raise NotImplementedError("only reduction='image-based' (what train_depth.py uses)")
        self.alpha, self.scales = float(alpha), int(scales)

    def forward(self, prediction, target, mask):
        """-> (total, ssi, reg).  Differentiable with respect to `prediction` (odb_midas_loss_bwd)."""
        if not prediction.is_cuda:
            raise _capi.OdbError("prediction: CUDA tensor required (no CPU path)")
        out = _MidasFn.apply(prediction, target, mask, self.alpha, self.scales)
        return out[0], out[1], out[2]


class _MidasFn(torch.autograd.Function):
    """MidasLoss forward / backward kernels behind torch.autograd (gradient with respect to the prediction only, as
    in the train step: target and mask are data)."""

    @staticmethod
    @_capi.on_tensor_device
    def forward(ctx, prediction, target, mask, alpha, scales):
        p, g = _f32(prediction, "prediction"), _f32(target, "target")
        b = p.shape[0]
        h, w = p.shape[-2:]
        m = mask.detach().to(torch.uint8).contiguous()
        ws_bytes = int(lib().odb_midas_loss_workspace_bytes(b))
        ws = torch.empty(ws_bytes + 256, dtype=torch.uint8, device=p.device)
        off = (-ws.data_ptr()) % 256
        out = torch.empty(3, dtype=torch.float32, device=p.device)
        check(lib().odb_midas_loss_fwd(p.data_ptr(), g.data_ptr(), m.data_ptr(), b, h, w, alpha, scales,
                                       out.data_ptr(), ws.data_ptr() + off, ws_bytes, _stream()), "odb_midas_loss_fwd")
        ctx.save_for_backward(p, g, m, ws)
        ctx.meta = (b, h, w, alpha, scales, off, prediction.shape, prediction.dtype)
        return out

    @staticmethod
    @_capi.on_tensor_device
    def backward(ctx, grad_out):
        p, g, m, ws = ctx.saved_tensors
        b, h, w, alpha, scales, off, shape, dtype = ctx.meta
        go = grad_out.detach().float().cpu()                       # (d/d total, d/d ssi, d/d reg)
        w_ssi = float(go[0] + go[1])
        w_reg = float(alpha * go[0] + go[2])
        bws = torch.empty(int(lib().odb_midas_loss_bwd_workspace_bytes(b)) // 8, dtype=torch.float64, device=p.device)
        gbuf = torch.empty(b * h * w, dtype=torch.float32, device=p.device)
        grad = torch.empty(b * h * w, dtype=torch.float32, device=p.device)
        check(lib().odb_midas_loss_bwd(p.data_ptr(), g.data_ptr(), m.data_ptr(), b, h, w, scales, w_ssi, w_reg,
                                       ws.data_ptr() + off, bws.data_ptr(), gbuf.data_ptr(), grad.data_ptr(),
                                       _stream()), "odb_midas_loss_bwd")
        return grad.view(shape).to(dtype), None, None, None, None


class VNL_Loss(torch.nn.Module):
    def __init__(self, focal_x, focal_y, input_size, delta_cos=0.867, delta_diff_x=0.01, delta_diff_y=0.01,
                 delta_diff_z=0.01, delta_z=0.0001, sample_ratio=0.15):
        super().__init__()
        self.fx, self.fy = float(focal_x), float(focal_y)
        self.input_size = tuple(input_size)
        self.delta_z, self.sample_ratio = float(delta_z), float(sample_ratio)

    def select_index(self):
        """Same host NumPy RNG call sequence as the reference (virtual_normal_loss.py:52-72), so that
        np.random.seed(s) yields the same triplets on both sides; returns flat indices y*W + x."""
        num = self.input_size[1] * self.input_size[0]
        pts = []
        for _ in range(3):
            p = np.random.choice(num, int(num * self.sample_ratio), replace=True)
            np.random.shuffle(p)
            pts.append(p.astype(np.int32))
        return pts

    def forward(self, gt_depth, pred_depth, select=True, points=None):
        """Differentiable with respect to the FIRST argument (what train_depth.py:272 passes there: the prediction)."""
        if not gt_depth.is_cuda:
            raise _capi.OdbError("gt_depth: CUDA tensor required (no CPU path)")
        h, w = gt_depth.shape[-2:]
        if (h, w) != self.input_size:
            raise ValueError("input size differs from the one given at construction")
        p1, p2, p3 = points if points is not None else self.select_index()
        dev = gt_depth.device
        pts = tuple(torch.from_numpy(np.ascontiguousarray(p)).to(dev) for p in (p1, p2, p3))
        return _VnlFn.apply(gt_depth, pred_depth, pts, self.fx, self.fy, self.delta_z, bool(select))


class _VnlFn(torch.autograd.Function):
    @staticmethod
    @_capi.on_tensor_device
    def forward(ctx, first, second, pts, fx, fy, delta_z, select):
        a, d = _f32(first, "gt_depth"), _f32(second, "pred_depth")
        b = a.shape[0]
        h, w = a.shape[-2:]
        t1, t2, t3 = pts
        n = t1.numel()
        scratch = torch.empty(b * n, dtype=torch.float32, device=a.device)
        out = torch.empty(1, dtype=torch.float32, device=a.device)
        check(lib().odb_vnl_loss_fwd(a.data_ptr(), d.data_ptr(), t1.data_ptr(), t2.data_ptr(), t3.data_ptr(), n, b, h,
                                     w, fx, fy, delta_z, 1 if select else 0, out.data_ptr(),
                                     scratch.data_ptr(), _stream()), "odb_vnl_loss_fwd")
        ctx.save_for_backward(a, d, t1, t2, t3, scratch)
        ctx.meta = (b, h, w, n, fx, fy, select, first.shape, first.dtype)
        return out[0]

    @staticmethod
    @_capi.on_tensor_device
    def backward(ctx, grad_out):
        a, d, t1, t2, t3, scratch = ctx.saved_tensors
        b, h, w, n, fx, fy, select, shape, dtype = ctx.meta
        acc = torch.empty(b * h * w, dtype=torch.int64, device=a.device)
        sel = torch.empty(4, dtype=torch.float64, device=a.device)
        grad = torch.empty(b * h * w, dtype=torch.float32, device=a.device)
        check(lib().odb_vnl_loss_bwd(a.data_ptr(), d.data_ptr(), t1.data_ptr(), t2.data_ptr(), t3.data_ptr(), n, b, h, w,
                                     fx, fy, 1 if select else 0, scratch.data_ptr(), float(grad_out), acc.data_ptr(),
                                     sel.data_ptr(), grad.data_ptr(), _stream()), "odb_vnl_loss_bwd")
        return grad.view(shape).to(dtype), None, None, None, None, None, None


def depth_step_losses(depth_preds, depth_gt, mask_float, midas: MidasLoss, vnl: VNL_Loss, train: bool = True,
                      global_step: int = 10 ** 9):
    """The loss arithmetic of Depth._shared_step (train_depth.py:261-287); differentiable w.r.t. depth_preds."""
    depth_preds = torch.clamp(depth_preds, 0, 1)
    mask_valid = make_valid_mask(mask_float)
    _, ssi, reg = midas(depth_preds, depth_gt, mask_valid)
    vn = vnl(depth_preds, depth_gt)               # NB: reference passes (pred, gt) into (gt_depth, pred_depth)
    if train and global_step < 15000:
        return {"ssi_loss": ssi, "reg_loss": 0, "vn_loss": 0, "depth_loss": ssi}
    return {"ssi_loss": ssi, "reg_loss": reg, "vn_loss": vn, "depth_loss": ssi + 0.1 * reg + 10 * vn}


class _NormalLossFn(torch.autograd.Function):
    @staticmethod
    @_capi.on_tensor_device
    def forward(ctx, preds, gt, mask_u8, clamp_preds):
        p, g = _f32(preds, "normal_preds"), _f32(gt, "normal_gt")
        b, _, h, w = p.shape
        out = torch.empty(3, device=p.device, dtype=torch.float32)
        ws = torch.empty(3 * b, device=p.device, dtype=torch.float64)
        check(lib().odb_normal_loss_fwd(p.data_ptr(), g.data_ptr(), mask_u8.data_ptr(), b, h, w, 1 if clamp_preds else 0,
                                        out.data_ptr(), ws.data_ptr(), _stream()), "odb_normal_loss_fwd")
        ctx.save_for_backward(p, g, mask_u8, ws)
        ctx.meta = (b, h, w, clamp_preds, preds.dtype)
        return out

    @staticmethod
    @_capi.on_tensor_device
    def backward(ctx, grad_out):
        p, g, m, ws = ctx.saved_tensors
        b, h, w, clamp_preds, dtype = ctx.meta
        go = grad_out.detach().float().cpu()                          # (d/d total, d/d l1, d/d cos); total = cos + 10 l1
        w_l1, w_cos = float(10.0 * go[0] + go[1]), float(go[0] + go[2])
        grad = torch.empty_like(p)
        check(lib().odb_normal_loss_bwd(p.data_ptr(), g.data_ptr(), m.data_ptr(), b, h, w, 1 if clamp_preds else 0,
                                        w_l1, w_cos, ws.data_ptr(), grad.data_ptr(), _stream()), "odb_normal_loss_bwd")
        return grad.to(dtype), None, None, None


def normal_losses(normal_preds: torch.Tensor, normal_gt: torch.Tensor, mask_valid: torch.Tensor,
                  clamp_preds: bool = False):
    """masked_l1_loss + masked_cosine_angular_loss (losses/masked_losses.py:4-7,14-23) in one pass.
    normal_preds, normal_gt: [B,3,H,W]; mask_valid: bool/uint8 [B,1,H,W] or the reference's
    `.repeat_interleave(3, 1)` form [B,3,H,W] (its first channel is used, as masked_cosine_angular_loss does).
    Returns (cos + 10 * l1, l1, cos); differentiable with respect to normal_preds."""
    if not normal_preds.is_cuda or not mask_valid.is_cuda:
        raise _capi.OdbError("normal_losses: CUDA tensors required (no CPU path)")
    if normal_preds.dim() != 4 or normal_preds.shape[1] != 3 or normal_gt.shape != normal_preds.shape:
        raise _capi.OdbError("normal_losses: [B,3,H,W] tensors expected")
    m = mask_valid[:, 0].to(torch.uint8).contiguous()
    out = _NormalLossFn.apply(normal_preds, normal_gt, m, bool(clamp_preds))
    return out[0], out[1], out[2]


def normal_step_losses(normal_preds, normal_gt, mask_float):
    """The loss arithmetic of train_normal.py:247-265 (differentiable w.r.t. normal_preds): clamp, make_valid_mask repeated over
    the three channels, l1 + cosine losses, normal_loss = cos + 10 * l1."""
    mask_valid = make_valid_mask(mask_float)
    total, l1, cos = normal_losses(normal_preds, normal_gt, mask_valid, clamp_preds=True)
    return {"l1_loss": l1, "cos_loss": cos, "normal_loss": total}


def check_vnl_points(points, h: int, w: int):
    """The VNL kernels gather at the index arrays without bounds checks: host arrays must be three equally long arrays of
    flat indices in [0, h*w).  Device tensors (a captured step's copies of arrays checked here) are not read back."""
    if len(points) != 3:
        raise ValueError("points: three VNL index arrays expected")
    if len({int(q.numel()) if isinstance(q, torch.Tensor) else int(np.size(q)) for q in points}) != 1:
        raise ValueError("points: the three VNL index arrays must have the same length")
    for q in points:
        if isinstance(q, torch.Tensor) and q.is_cuda:
            continue
        a = np.asarray(q)
        if a.size and (int(a.min()) < 0 or int(a.max()) >= h * w):
            raise ValueError(f"points: VNL indices must lie in [0, {h * w}) for a {h}x{w} prediction")


class _StepBuffers:
    """Persistent device buffers of a train step's loss, allocated at the first call at a shape and reused after it (no
    allocation in a CUDA-graph capture or replay)."""

    def _buf(self, name, shape, dtype, device):
        t = self._bufs.get(name)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype or t.device != device:
            t = self._bufs[name] = torch.empty(tuple(shape), dtype=dtype, device=device)
        return t


class DepthStepLoss(_StepBuffers):
    """The loss arithmetic of Depth._shared_step (train_depth.py:261-279) AND its gradient with respect to the raw
    network output, as one fixed launch sequence with no host synchronisation and no autograd graph (the train step's
    hot path; `depth_step_losses` above is the autograd-facing equivalent):

        pc = clamp(pred, 0, 1); mask = make_valid_mask(mask_float); (ssi, reg) = MidasLoss(pc, gt, mask)
        vn = VNL_Loss(pc, gt)                     # (pred, gt) order as the reference calls it
        loss = ssi                                 if global_step < 15000 (train)
               ssi + 0.1 reg + 10 vn               otherwise
        d loss / d pred

    `points`: the three VNL index arrays (host NumPy RNG, reference call sequence); drawn with np.random if None."""

    def __init__(self, input_size=(384, 384), alpha: float = 0.1, scales: int = 4):
        self.midas = MidasLoss(alpha=alpha, scales=scales)
        self.vnl = VNL_Loss(1.0, 1.0, tuple(input_size))
        self._bufs = {}

    @_capi.on_tensor_device
    @torch.no_grad()
    def __call__(self, pred: torch.Tensor, depth_gt: torch.Tensor, mask_float: torch.Tensor, full_mix: bool = True,
                 points=None):
        """pred, depth_gt, mask_float: [B,1,H,W] fp32 CUDA.  Returns (losses fp32 [4] = (loss, ssi, reg, vn), dpred)."""
        h, w = pred.shape[-2], pred.shape[-1]
        if (h, w) != self.vnl.input_size:
            raise ValueError(f"DepthStepLoss: prediction is {h}x{w}, built for {self.vnl.input_size[0]}x{self.vnl.input_size[1]}")
        if full_mix and points is not None:
            check_vnl_points(points, h, w)
        p, g = _f32(pred, "pred"), _f32(depth_gt, "depth_gt")
        dev = p.device
        b = p.shape[0]
        n = b * h * w
        st = torch.cuda.current_stream(dev).cuda_stream
        pc = self._buf("pc", (b, 1, h, w), torch.float32, dev)
        check(lib().odb_clamp01(p.data_ptr(), pc.data_ptr(), n, st), "odb_clamp01")
        m = make_valid_mask(mask_float).to(torch.uint8)
        alpha, scales = self.midas.alpha, self.midas.scales
        ws_bytes = int(lib().odb_midas_loss_workspace_bytes(b))
        ws = self._buf("midas_ws", (ws_bytes + 256,), torch.uint8, dev)
        off = (-ws.data_ptr()) % 256
        out3 = self._buf("midas_out", (3,), torch.float32, dev)
        check(lib().odb_midas_loss_fwd(pc.data_ptr(), g.data_ptr(), m.data_ptr(), b, h, w, alpha, scales, out3.data_ptr(),
                                       ws.data_ptr() + off, ws_bytes, st), "odb_midas_loss_fwd")
        bws = self._buf("midas_bws", (int(lib().odb_midas_loss_bwd_workspace_bytes(b)) // 8,), torch.float64, dev)
        gbuf = self._buf("midas_gbuf", (n,), torch.float32, dev)
        gm = self._buf("midas_grad", (n,), torch.float32, dev)
        check(lib().odb_midas_loss_bwd(pc.data_ptr(), g.data_ptr(), m.data_ptr(), b, h, w, scales, 1.0,
                                       alpha if full_mix else 0.0, ws.data_ptr() + off, bws.data_ptr(), gbuf.data_ptr(),
                                       gm.data_ptr(), st), "odb_midas_loss_bwd")
        losses = self._buf("losses", (4,), torch.float32, dev)
        gv = None
        if full_mix:
            p1, p2, p3 = points if points is not None else self.vnl.select_index()
            # int32 index arrays: host NumPy (copied here) or already on the device (a captured step's static buffers)
            t1, t2, t3 = (q if isinstance(q, torch.Tensor) and q.is_cuda else
                          torch.from_numpy(np.ascontiguousarray(q)).to(dev, non_blocking=True) for q in (p1, p2, p3))
            if any(t.dtype != torch.int32 or not t.is_contiguous() for t in (t1, t2, t3)):
                raise _capi.OdbError("DepthStepLoss: VNL index arrays must be contiguous int32")
            npts = t1.numel()
            scratch = self._buf("vnl_scratch", (b * npts,), torch.float32, dev)
            vout = self._buf("vnl_out", (1,), torch.float32, dev)
            check(lib().odb_vnl_loss_fwd(pc.data_ptr(), g.data_ptr(), t1.data_ptr(), t2.data_ptr(), t3.data_ptr(), npts, b, h,
                                         w, self.vnl.fx, self.vnl.fy, self.vnl.delta_z, 1, vout.data_ptr(),
                                         scratch.data_ptr(), st), "odb_vnl_loss_fwd")
            acc = self._buf("vnl_acc", (n,), torch.int64, dev)
            sel = self._buf("vnl_sel", (4,), torch.float64, dev)
            gv = self._buf("vnl_grad", (n,), torch.float32, dev)
            check(lib().odb_vnl_loss_bwd(pc.data_ptr(), g.data_ptr(), t1.data_ptr(), t2.data_ptr(), t3.data_ptr(), npts, b, h,
                                         w, self.vnl.fx, self.vnl.fy, 1, scratch.data_ptr(), 10.0, acc.data_ptr(),
                                         sel.data_ptr(), gv.data_ptr(), st), "odb_vnl_loss_bwd")
            losses[1:3].copy_(out3[1:3])
            losses[3:4].copy_(vout)
            torch.add(out3[1] + alpha * out3[2], vout[0], alpha=10.0, out=losses[0])
        else:
            losses.zero_()
            losses[0:2].copy_(out3[1:2].expand(2))
        dpred = self._buf("dpred", (b, 1, h, w), torch.float32, dev)
        check(lib().odb_clamp01_bwd(p.data_ptr(), gm.data_ptr(), None if gv is None else gv.data_ptr(), dpred.data_ptr(), n,
                                    st), "odb_clamp01_bwd")
        return losses, dpred


class NormalStepLoss(_StepBuffers):
    """The loss arithmetic of the normal model's _shared_step (train_normal.py:247-265) AND its gradient with respect to
    the raw network output, as one fixed launch sequence with no host synchronisation, no autograd graph and no
    allocation after the first call at a shape (the normal train step's hot path; `normal_step_losses` above is the
    autograd-facing equivalent):

        pc = clamp(pred, 0, 1); mask = make_valid_mask(mask_float) repeated over the 3 channels
        l1 = masked_l1_loss(pc, gt, mask); cos = masked_cosine_angular_loss(pc, gt, mask)
        loss = cos + 10 l1
        d loss / d pred                           (through the clamp)"""

    def __init__(self):
        self._bufs = {}

    @_capi.on_tensor_device
    @torch.no_grad()
    def __call__(self, pred: torch.Tensor, normal_gt: torch.Tensor, mask_float: torch.Tensor):
        """pred, normal_gt: [B,3,H,W]; mask_float: [B,1,H,W]; fp32 CUDA.  Returns (losses fp32 [3] = (loss, l1, cos),
        dpred [B,3,H,W])."""
        if pred.dim() != 4 or pred.shape[1] != 3:
            raise ValueError(f"NormalStepLoss: prediction must be [B,3,H,W], got {tuple(pred.shape)}")
        b, _, h, w = pred.shape
        if tuple(normal_gt.shape) != (b, 3, h, w):
            raise ValueError(f"NormalStepLoss: normal_gt must be [{b},3,{h},{w}], got {tuple(normal_gt.shape)}")
        if tuple(mask_float.shape) != (b, 1, h, w):
            raise ValueError(f"NormalStepLoss: mask_float must be [{b},1,{h},{w}], got {tuple(mask_float.shape)}")
        p, g, mf = _f32(pred, "pred"), _f32(normal_gt, "normal_gt"), _f32(mask_float, "mask_float")
        dev = p.device
        st = torch.cuda.current_stream(dev).cuda_stream
        m = self._buf("mask", (b, h, w), torch.uint8, dev)
        check(lib().odb_make_valid_mask(mf.data_ptr(), m.data_ptr(), b, h, w, 4, st), "odb_make_valid_mask")
        losses = self._buf("losses", (3,), torch.float32, dev)
        ws = self._buf("ws", (3 * b,), torch.float64, dev)
        check(lib().odb_normal_loss_fwd(p.data_ptr(), g.data_ptr(), m.data_ptr(), b, h, w, 1, losses.data_ptr(),
                                        ws.data_ptr(), st), "odb_normal_loss_fwd")
        dpred = self._buf("dpred", (b, 3, h, w), torch.float32, dev)
        check(lib().odb_normal_loss_bwd(p.data_ptr(), g.data_ptr(), m.data_ptr(), b, h, w, 1, 10.0, 1.0, ws.data_ptr(),
                                        dpred.data_ptr(), st), "odb_normal_loss_bwd")
        return losses, dpred
