"""Track the camera through unposed frames: one frame's pose (and the scale and shift of its depth) solved against a
model depth map rendered at a reference pose, by point-to-plane ICP with projective association (KinectFusion,
Newcombe et al. 2011), optionally with a photometric term, on the device (csrc/track.cu).

    from omnidata_b200.track import FrameTracker
    tracker = FrameTracker(affine=True, iterations=20, tol=1e-6, robust=0.02, max_dist=0.1, min_overlap=0.1,
                           photometric=0.0, photometric_robust=0.1)
    ref = volume.raycast((fx, fy, cx, cy), ref_pose, (h, w))            # the model's z-depth at ref_pose
    nodes0, _ = SparseDepthAligner(grid=(1, 1), robust=0.05).fit(pred, ref.unsqueeze(0))
    pose, nodes, record = tracker.track(pred, ref, (fx, fy, cx, cy), ref_pose, init_pose=None, init_nodes=nodes0)
    metres = aligner.apply(pred, nodes)                                  # then volume.integrate(metres, K, pose)

pred fp32 [H,W] or [1,H,W] is the frame's depth: the clamped relative prediction with affine=True (its scale s and
shift t are solved with the pose, starting from init_nodes), or metres with affine=False (s = 1, t = 0 fixed, a 6-DoF
solve).  ref_depth fp32 [H,W] is the model's depth at ref_pose with the same intrinsics, 0 where there is no surface.
Poses are host 4 x 4 camera-to-world matrices; init_pose defaults to ref_pose.  The model's normals are
`depth_normals(ref_depth, K, axes=(1, 1, 1), mask=ref_depth > 0)`, computed here into buffers the tracker keeps.

Outputs on the device: pose fp64 [4,4], nodes fp64 [1,1,1,2] in `SparseDepthAligner`'s layout (so `apply(pred, nodes)`
gives the aligned metres), record fp64 [8] = (correspondences in the last iteration, status, weighted RMS of the
point-to-plane residual in metres, fraction of correspondences the Huber weight reduced, iterations run, s, t, valid
frame pixels); status indexes STATUS.  A failed frame (no_overlap: fewer than min_overlap of its valid pixels found a
correspondence, also for an empty model; degenerate: the scene does not fix every unknown, as with a single plane;
nonfinite: NaN in init_nodes or the update) returns init_pose and init_nodes unchanged.

The defaults max_dist = 0.1 m, robust = 0.02 m, min_overlap = 0.1, the pivot threshold 1e-6 and iterations = 20 are
not tuned.  Tracking is frame-to-model: drift is bounded by the model and not corrected here; LoopClosure
(omnidata_b200/loop.py) corrects it when the camera revisits a place, from the information matrices below.
Photometric term (RGB-D odometry, Whelan et al. 2013; the joint cost of ElasticFusion): with `photometric` = lambda > 0
each geometric correspondence also asks the reference image's luminance at the frame point's projection to equal the
frame's, which fixes the motions that geometry alone leaves free (a textured wall).  Then
`track(..., rgb=image, ref_rgb=model_colour)` is required: rgb fp32 [3,H,W] or [1,3,H,W] the frame's image in [0, 1],
ref_rgb the model's colour at ref_pose, normally `volume.raycast(K, ref_pose, (h, w), color=True)[1]` (NaN: no
colour).  lambda is in m^2 per squared intensity step; photometric_robust is the Huber threshold of the intensity
residual.  The record then has 11 columns: the 8 above, then (photometric terms in the last iteration, weighted RMS of
the intensity residual, fraction of them the Huber weight reduced).  The reference's luminance and Sobel gradient go to
a buffer the tracker keeps; a call is one launch longer.  There is no exposure or brightness compensation between
frames: real video will need it.  lambda = 1e-2 is what the sweep on the analytic scene chose (DESIGN.md §6); it is not
tuned on real data.  photometric = 0 (the default) is the geometric tracker unchanged.

`information()` after a call returns the normal matrix sum w J J^T of that call's last Gauss-Newton step, fp64 [n,n]
on the device (n = 8 with affine, else 6; the photometric terms included, unscaled, in the tracker's (v, omega[, s,
t]) increment coordinates): the information of the solved pose, as a pose-graph edge needs it.  It is meaningful only
when that call's status is ok, and it reads the workspace of the last `track` call, so call it before the next one.

Definition: DESIGN.md §3 "Camera tracking" and include/omnidata_b200.h; oracle/track_oracle.py restates it in float64,
and oracle/photometric_oracle.py the photometric term.
Bit-reproducible; after the first call at a shape a call neither synchronises nor allocates beyond its outputs, so it
can be captured in a CUDA graph.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _capi, ops
from .fusion import _check_jump
from .losses import _StepBuffers

STATUS = ("ok", "no_overlap", "degenerate", "nonfinite")     # record column 1
NORMAL_AXES = (1, 1, 1)          # the model normals are decoded as n = 2 c - 1 in the reference camera frame
NORMAL_JUMP = 0.02               # depth_normals' default depth-step threshold (fraction of the depth range)


def _value_error(fn, *args):
    try:
        return fn(*args)
    except _capi.OdbError as e:
        raise ValueError(str(e)) from None


class FrameTracker(_StepBuffers):
    """Solves a frame's camera pose against a model depth map (module docstring)."""

    def __init__(self, affine: bool = True, iterations: int = 20, tol: float = 1e-6, robust: float = 0.02,
                 max_dist: float = 0.1, min_overlap: float = 0.1, photometric: float = 0.0,
                 photometric_robust: float = 0.1):
        _value_error(ops.check_track_params, "FrameTracker", affine, iterations, tol, robust, max_dist, min_overlap)
        _value_error(ops.check_photometric, "FrameTracker", photometric, photometric_robust)
        self.photometric, self.photometric_robust = float(photometric), float(photometric_robust)
        self.affine, self.iterations = affine, int(iterations)
        self.tol, self.robust, self.max_dist, self.min_overlap = float(tol), float(robust), float(max_dist), \
            float(min_overlap)
        self._jump = _check_jump(NORMAL_JUMP)
        self._bufs = {}
        self._last_hw = None

    @_capi.on_tensor_device
    @torch.no_grad()
    def track(self, pred: torch.Tensor, ref_depth: torch.Tensor, intrinsics, ref_pose, init_pose=None,
              init_nodes: Optional[torch.Tensor] = None, rgb: Optional[torch.Tensor] = None,
              ref_rgb: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """(pose fp64 [4,4], nodes fp64 [1,1,1,2], record fp64 [8], or [11] with the photometric term) on pred's
        device; kept for the next call at this shape, which overwrites them.  rgb and ref_rgb (fp32 [3,H,W] or
        [1,3,H,W]) exactly when photometric > 0."""
        name = "FrameTracker.track"
        photo = self.photometric > 0
        if (rgb is None) == photo or (ref_rgb is None) == photo:
            raise ValueError(f"{name}: rgb and ref_rgb are required exactly when photometric > 0 "
                             f"(photometric={self.photometric})")
        if pred.dim() == 3 and pred.shape[0] == 1:
            pred = pred[0]
        if pred.dim() != 2:
            raise ValueError(f"{name}: pred must be [H,W] or [1,H,W], got {tuple(pred.shape)}")
        h, w = pred.shape
        if tuple(ref_depth.shape) != (h, w):
            raise ValueError(f"{name}: ref_depth must be [{h}, {w}] like pred, got {tuple(ref_depth.shape)}")
        tensors = [("pred", pred), ("ref_depth", ref_depth)]
        if photo:
            rgb, ref_rgb = (t[0] if t.dim() == 4 and t.shape[0] == 1 else t for t in (rgb, ref_rgb))
            for what, t in (("rgb", rgb), ("ref_rgb", ref_rgb)):
                if tuple(t.shape) != (3, h, w):
                    raise ValueError(f"{name}: {what} must be [3, {h}, {w}] or [1, 3, {h}, {w}] like pred, got "
                                     f"{tuple(t.shape)}")
            tensors += [("rgb", rgb), ("ref_rgb", ref_rgb)]
        for what, t in tensors:
            if not t.is_cuda or t.dtype != torch.float32:
                raise ValueError(f"{name}: {what} must be fp32 on a CUDA device, got {t.dtype} on {t.device}")
            if t.device != pred.device:
                raise ValueError(f"{name}: pred and {what} live on different devices")
            if not t.is_contiguous():
                raise ValueError(f"{name}: {what} must be contiguous (a copy would allocate on every call)")
        if self.affine != (init_nodes is not None):
            raise ValueError(f"{name}: init_nodes (the initial (s, t), e.g. SparseDepthAligner(grid=(1, 1)).fit) is "
                             f"required exactly when affine (affine={self.affine})")
        k = _value_error(ops.check_intrinsics, name, intrinsics)
        ref_pose = _value_error(ops.check_poses, name, ref_pose)
        init_pose = ref_pose if init_pose is None else _value_error(ops.check_poses, name, init_pose)
        for what, T in (("ref_pose", ref_pose), ("init_pose", init_pose)):
            if T.shape[0] != 1:
                raise ValueError(f"{name}: {what} must be one [4,4] pose, got {T.shape[0]}")
        _value_error(ops._check_planes, name, 1, h, w)
        dev = pred.device
        if init_nodes is not None and (tuple(init_nodes.shape) != (1, 1, 1, 2) or init_nodes.dtype != torch.float64
                                       or init_nodes.device != dev):
            raise ValueError(f"{name}: init_nodes must be fp64 [1, 1, 1, 2] on {dev}, got {init_nodes.dtype} "
                             f"{tuple(init_nodes.shape)} on {init_nodes.device}")
        mask = self._buf("mask", (1, h, w), torch.bool, dev)
        torch.gt(ref_depth.unsqueeze(0), 0.0, out=mask)
        nws = self._buf("normals_ws", (-(-ops.depth_normals_workspace_bytes(1, h, w) // 8),), torch.float64, dev)
        normals = self._buf("normals", (1, 3, h, w), torch.float32, dev)
        ws = self._buf("workspace", (-(-ops.track_workspace_bytes(h, w) // 8),), torch.float64, dev)
        pose = self._buf("pose", (4, 4), torch.float64, dev)
        nodes = self._buf("nodes", (1, 1, 1, 2), torch.float64, dev)
        rec = self._buf("record", (_capi.TRACK_RGBD_RECORD if photo else _capi.TRACK_RECORD,), torch.float64, dev)
        intensity = self._buf("intensity", (3, h, w), torch.float32, dev) if photo else None
        ops.depth_normals(ref_depth.unsqueeze(0), mask, k, NORMAL_AXES, self._jump, nws, normals)
        ops.track_frame(pred, ref_depth, normals, k, ref_pose.reshape(4, 4), init_pose.reshape(4, 4), init_nodes,
                        self.affine, self.iterations, self.tol, self.robust, self.max_dist, self.min_overlap, ws,
                        pose, nodes, rec, rgb, ref_rgb, intensity, self.photometric, self.photometric_robust)
        self._last_hw = (h, w)
        return pose, nodes, rec

    @torch.no_grad()
    def information(self) -> torch.Tensor:
        """fp64 [n,n] on the device (n = 8 with affine, else 6): sum w J J^T of the last Gauss-Newton step of the last
        `track` call, meaningful when its status is ok (module docstring).  Kept for the next call, which overwrites
        it."""
        if self._last_hw is None:
            raise ValueError("FrameTracker.information: no track call yet")
        h, w = self._last_hw
        ws = self._bufs["workspace"]
        n = 8 if self.affine else 6
        info = self._buf("information", (n, n), torch.float64, ws.device)
        with torch.cuda.device(ws.device):
            ops.track_information(ws, h, w, n, info)
        return info
