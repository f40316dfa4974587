"""Correct tracking drift when the camera revisits a place: keyframes, loop detection by pose proximity (and, with
places=True, by appearance), verification by tracking, an SE(3) pose-graph solve (omnidata_b200/posegraph.py) and
re-fusion of the TSDF volume at the corrected poses.  Host orchestration over the existing kernels.

    from omnidata_b200.loop import LoopClosure
    loop = LoopClosure((fx, fy, cx, cy), (h, w))
    # after each frame is integrated at its tracked pose:
    if loop.add(metres, pose, rgb=None):      # True: a loop closed and every frame's pose changed
        loop.refuse(volume)                   # the volume again, from all stored frames at the new poses
        pose = loop.poses[-1]                 # track the next frame from the corrected last pose

Store.  `add` keeps every frame's aligned metres fp32 [H,W] (and rgb fp32 [3,H,W]) on the device in buffers of
[capacity,H,W] grown by doubling, so that re-fusion is one `integrate` call without a stacking copy: 4 H W bytes per
frame (16 H W with colour), 1.2 GB per 1000 frames at 640 x 480 without colour, plus up to as much again of unused
capacity.  It also keeps each frame's pose, the keyframe it is attached to and its pose relative to that keyframe.

Keyframes.  Frame 0 is keyframe 0 and the gauge of the graph.  A frame becomes a keyframe when it has moved at least
keyframe_dist metres or turned at least keyframe_angle degrees from the last keyframe.  Each new keyframe j gets an
odometry edge to keyframe j - 1: FrameTracker(affine=False, photometric=photometric) tracks its metres against
keyframe j - 1's stored metres (and, with photometric > 0, its image against keyframe j - 1's stored image; then every
frame needs rgb) with ref_pose T_{j-1} and init_pose T_j; Z = T_{j-1}^-1 T^_j and W = FrameTracker.information().  When that tracking fails,
the edge keeps the current relative pose with a fixed isotropic W (sigma 1 cm and 0.5 degrees), so that the graph stays
connected.

Loops.  Candidates for keyframe j are the keyframes i <= j - min_gap whose camera centre lies within `radius` metres
of keyframe j's and whose optical axis lies within `angle` degrees of its; the nearest `candidates` are verified by the
same tracking against keyframe i's stored metres.  An edge is accepted when the status is ok, the correspondences are
at least min_overlap of the valid pixels and the weighted RMS residual is at most max_rms metres.  When a step accepts a
loop edge, PoseGraph.optimize runs over all keyframes, every frame's pose becomes T_kf,new (T_kf,old^-1 T_frame,old),
and `add` returns True.  `refuse(volume)` then resets the volume and integrates all stored frames in order at the new
poses; integration loops over the frames in order at every point, so the result is bit-identical to a fresh volume
integrating the same frames at those poses.  When no loop is accepted nothing changes.

Place recognition (places=True; every frame then needs rgb).  Each new keyframe is encoded from its stored metres and
rgb into a randomized-fern code (omnidata_b200/places.py FernDatabase), so candidates no longer depend on poses that
may have drifted.  After the pose candidates, which are unchanged, up to `candidates` more come from the fern lookup
over the keyframes i <= j - min_gap whose dissimilarity (the fraction of ferns whose codes differ) is at most
max_dissimilarity, skipping those already proposed.  A fern candidate is verified by the same tracking but from init
pose T_i, keyframe i's own pose: the match says that the views are alike, the drifted pose says nothing.  The
acceptance rule, the solve and the re-posing are unchanged.

Relocalisation (places=True).  `relocalise(pred, rgb, sparse=None)` finds the pose of a frame whose tracking failed:
it encodes the frame and tries the nearest `candidates` keyframes under max_dissimilarity in order of distance,
tracking pred from keyframe i's pose T_i against its stored metres and rgb (with sparse depths: pred fitted to them,
then the metres with the metric tracker; without: FrameTracker(affine=True) from a SparseDepthAligner(grid=(1, 1),
robust=0.05) fit of pred to keyframe i's metres).  The first candidate that passes the loop-edge test gives the pose,
host [4,4]; None when none does.  The next `add` must then be of that frame: it always becomes a keyframe, and its
first edge goes to keyframe i with the relocalisation's Z = T_i^-1 T^ and W (with affine tracking the information of
the pose with the scale and shift marginalised out), not an odometry edge to keyframe j - 1, which it could not track
against; that keyframe is not proposed again as a loop candidate in the same `add`, so the one constraint is not
counted twice.  `cancel_relocalisation()` forgets a relocalisation whose frame is not added.  `relocalisations` lists
(keyframe frame index, frame index) pairs.  Relocalisation starts only from a failure status: a frame that tracks to
a wrong pose with status ok is not detected.

Every default (keyframe_dist = 0.1 m, keyframe_angle = 5 degrees, min_gap = 10 keyframes, radius = 0.3 m, angle = 30
degrees, candidates = 3, min_overlap = 0.3, max_rms = 0.01 m, the fallback sigmas, max_dissimilarity = MAX_DISSIMILARITY
from the analytic orbit, DESIGN.md §6) is untuned on real data.  Loop edges are not robust (one wrong accepted edge
bends the whole graph), the graph is SE(3) (no scale drift) and a closure re-fuses every frame instead of
de-integrating: DESIGN.md §8.

Use the photometric term (photometric = 1e-2, as the tracking): on the analytic scene's closed orbit, edges from
geometry alone leave rotations about weakly seen axes nearly free, and a closure then bends the graph along them and
makes the trajectory worse (DESIGN.md §6).
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import numpy as np
import torch

from . import ops
from .posegraph import PoseGraph
from .places import FernDatabase
from .sparse import SparseDepthAligner
from .track import FrameTracker, _value_error

FALLBACK_SIGMA = (0.01, math.radians(0.5))      # metres, radians: a failed odometry edge's information (untuned)
MAX_DISSIMILARITY = 0.6                         # fern candidates' largest dissimilarity (DESIGN.md §6; untuned)
RELOCALISE_ROBUST = 0.05                        # Huber threshold of relocalisation's scale-and-shift fit (untuned)


def _angle_deg(Ra, Rb):
    c = (np.trace(Ra.T @ Rb) - 1.0) / 2.0
    return math.degrees(math.acos(min(1.0, max(-1.0, c))))


def _axis_angle_deg(Ra, Rb):
    c = float(Ra[:, 2] @ Rb[:, 2])
    return math.degrees(math.acos(min(1.0, max(-1.0, c))))


class LoopClosure:
    """Keyframes, loop detection, pose-graph correction and re-fusion (module docstring)."""

    def __init__(self, intrinsics, size: Tuple[int, int], keyframe_dist: float = 0.1, keyframe_angle: float = 5.0,
                 min_gap: int = 10, radius: float = 0.3, angle: float = 30.0, candidates: int = 3,
                 min_overlap: float = 0.3, max_rms: float = 0.01, photometric: float = 0.0, places: bool = False,
                 max_dissimilarity: float = MAX_DISSIMILARITY, device=None):
        self.intrinsics = _value_error(ops.check_intrinsics, "LoopClosure", intrinsics)
        h, w = (int(v) for v in size)
        _value_error(ops._check_planes, "LoopClosure", 1, h, w)
        for what, v in (("keyframe_dist", keyframe_dist), ("keyframe_angle", keyframe_angle), ("radius", radius),
                        ("angle", angle), ("max_rms", max_rms)):
            if not (isinstance(v, (int, float)) and math.isfinite(v) and v > 0):
                raise ValueError(f"LoopClosure: {what} must be finite and > 0, got {v!r}")
        if not (isinstance(min_gap, int) and min_gap >= 1 and isinstance(candidates, int) and candidates >= 1):
            raise ValueError(f"LoopClosure: min_gap and candidates must be integers >= 1, got {min_gap!r}, "
                             f"{candidates!r}")
        if not 0 < min_overlap <= 1:
            raise ValueError(f"LoopClosure: min_overlap must lie in (0, 1], got {min_overlap!r}")
        if not isinstance(places, bool):
            raise ValueError(f"LoopClosure: places must be a bool, got {places!r}")
        if isinstance(max_dissimilarity, bool) or not (isinstance(max_dissimilarity, (int, float)) and
                                                       0 <= max_dissimilarity <= 1):
            raise ValueError(f"LoopClosure: max_dissimilarity must lie in [0, 1], got {max_dissimilarity!r}")
        self.size = (h, w)
        self.keyframe_dist, self.keyframe_angle = float(keyframe_dist), float(keyframe_angle)
        self.min_gap, self.radius, self.angle, self.candidates = min_gap, float(radius), float(angle), candidates
        self.min_overlap, self.max_rms = float(min_overlap), float(max_rms)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.tracker = FrameTracker(affine=False, photometric=photometric)
        self.photometric = float(photometric)
        self.graph = PoseGraph(device=self.device)
        self._metres: Optional[torch.Tensor] = None   # [capacity,H,W]
        self._rgb: Optional[torch.Tensor] = None      # [capacity,3,H,W]
        self._poses: List[np.ndarray] = []            # every frame's camera-to-world pose
        self._attach: List[Tuple[int, np.ndarray]] = []   # (keyframe index, T_kf^-1 T_frame) of every frame
        self.keyframes: List[int] = []                # frame index of each keyframe
        self._kf_poses: List[np.ndarray] = []
        self._edges: List[Tuple[int, int]] = []       # keyframe indices
        self._Z: List[np.ndarray] = []
        self._W: List[np.ndarray] = []
        self.loops: List[Tuple[int, int]] = []        # accepted loop edges as (frame i, frame j)
        self.refusions = 0
        self.closures = 0
        self.max_dissimilarity = float(max_dissimilarity)
        self.places: Optional[FernDatabase] = FernDatabase((h, w), device=self.device) if places else None
        self.relocalisations: List[Tuple[int, int]] = []   # (keyframe frame index, relocalised frame index)
        self._reloc = None                            # (keyframe index i, Z, W) of the pending relocalisation
        self._affine_tracker = FrameTracker(affine=True, photometric=photometric) if places else None
        self._aligner = SparseDepthAligner(grid=(1, 1), robust=RELOCALISE_ROBUST) if places else None

    @property
    def frames(self) -> int:
        return len(self._poses)

    @property
    def poses(self) -> np.ndarray:
        """Every stored frame's current camera-to-world pose, host float64 [F,4,4]."""
        return np.stack(self._poses)

    def _store(self, metres: torch.Tensor, rgb: Optional[torch.Tensor]):
        f = self.frames
        if self._metres is None or f == self._metres.shape[0]:
            cap = 16 if self._metres is None else 2 * self._metres.shape[0]
            grown = torch.empty((cap, *self.size), dtype=torch.float32, device=self.device)
            grown_rgb = None if rgb is None else torch.empty((cap, 3, *self.size), dtype=torch.float32,
                                                             device=self.device)
            if f:
                grown[:f].copy_(self._metres[:f])
                if rgb is not None:
                    grown_rgb[:f].copy_(self._rgb[:f])
            self._metres, self._rgb = grown, grown_rgb
        self._metres[f].copy_(metres.reshape(self.size))
        if rgb is not None:
            self._rgb[f].copy_(rgb.reshape(3, *self.size))

    def _track(self, frame: int, ref_frame: int, ref_pose, init_pose):
        """(status ok, corrected pose, information, record) of stored frame `frame` tracked against `ref_frame`."""
        colour = dict(rgb=self._rgb[frame], ref_rgb=self._rgb[ref_frame]) if self.photometric > 0 else {}
        pose, _, rec = self.tracker.track(self._metres[frame], self._metres[ref_frame], self.intrinsics, ref_pose,
                                          init_pose, **colour)
        rec = rec.cpu().numpy()
        if int(rec[1]) != 0:
            return False, None, None, rec
        return True, pose.cpu().numpy(), self.tracker.information().cpu().numpy(), rec

    def _edge_ok(self, rec) -> bool:
        """The loop-edge test: status ok, correspondences >= min_overlap of the valid pixels, RMS <= max_rms."""
        return int(rec[1]) == 0 and rec[0] >= self.min_overlap * rec[7] and rec[2] <= self.max_rms

    def _fern_candidates(self, code: torch.Tensor, limit: int, count: int, skip=()) -> List[int]:
        """Up to `count` keyframe indices i < limit in order of fern distance to code, at most max_dissimilarity, not
        in skip."""
        if limit <= 0:
            return []
        idx, dist = self.places.query(code, min(count + len(skip), limit), limit=limit)
        out = []
        for i, d in zip(idx.cpu().tolist(), dist.cpu().tolist()):
            if i >= 0 and i not in skip and self.places.dissimilarity(d) <= self.max_dissimilarity:
                out.append(i)
        return out[:count]

    @torch.no_grad()
    def add(self, metres: torch.Tensor, pose, rgb: Optional[torch.Tensor] = None) -> bool:
        """Stores a frame integrated at pose (host [4,4]): metres fp32 [H,W] or [1,H,W] on the device, rgb fp32 [3,H,W]
        exactly when the volume keeps colour.  True when a loop closed and the stored poses changed."""
        name = "LoopClosure.add"
        h, w = self.size
        if metres.numel() != h * w or metres.dtype != torch.float32 or metres.device != self.device:
            raise ValueError(f"{name}: metres must be fp32 [{h}, {w}] on {self.device}, got {metres.dtype} "
                             f"{tuple(metres.shape)} on {metres.device}")
        if (self.frames and (rgb is None) != (self._rgb is None)) or \
                ((self.photometric > 0 or self.places is not None) and rgb is None):
            raise ValueError(f"{name}: pass rgb for every frame or for none, and for every frame when photometric > 0 "
                             f"or with places")
        if rgb is not None and (rgb.numel() != 3 * h * w or rgb.dtype != torch.float32 or rgb.device != self.device):
            raise ValueError(f"{name}: rgb must be fp32 [3, {h}, {w}] on {self.device}")
        T = _value_error(ops.check_poses, name, pose).reshape(-1, 4, 4)
        if T.shape[0] != 1:
            raise ValueError(f"{name}: one [4,4] pose, got {T.shape[0]}")
        T = T[0]
        f = self.frames
        self._store(metres, rgb)
        self._poses.append(T.copy())
        reloc, self._reloc = self._reloc, None
        new_kf = not self.keyframes or reloc is not None
        if not new_kf:
            last = self._kf_poses[-1]
            new_kf = np.linalg.norm(T[:3, 3] - last[:3, 3]) >= self.keyframe_dist or \
                _angle_deg(last[:3, :3], T[:3, :3]) >= self.keyframe_angle
        if not new_kf:
            self._attach.append((len(self.keyframes) - 1, np.linalg.inv(self._kf_poses[-1]) @ T))
            return False
        self.keyframes.append(f)
        self._kf_poses.append(T.copy())
        self._attach.append((len(self.keyframes) - 1, np.eye(4)))
        j = len(self.keyframes) - 1
        code = None
        if self.places is not None:
            code = self.places.encode(self._metres[f], self._rgb[f])[0]
            self.places.add(code)
        if j == 0:
            return False
        if reloc is not None:
            i, Z, W = reloc
            self._edges.append((i, j))
            self._Z.append(Z)
            self._W.append(W)
            self.relocalisations.append((self.keyframes[i], f))
        else:
            prev = self._kf_poses[j - 1]
            ok, That, W, _ = self._track(f, self.keyframes[j - 1], prev, T)
            if not ok:
                That, W = T, np.diag([FALLBACK_SIGMA[0] ** -2] * 3 + [FALLBACK_SIGMA[1] ** -2] * 3)
            self._edges.append((j - 1, j))
            self._Z.append(np.linalg.inv(prev) @ That)
            self._W.append(W)
        # a relocalised keyframe already has its edge to the keyframe it was found against: not proposed again
        skip = [] if reloc is None else [reloc[0]]
        accepted = []
        cands = []
        for i in range(0, j - self.min_gap + 1):
            if i in skip:
                continue
            Ti = self._kf_poses[i]
            d = float(np.linalg.norm(Ti[:3, 3] - T[:3, 3]))
            if d <= self.radius and _axis_angle_deg(Ti[:3, :3], T[:3, :3]) <= self.angle:
                cands.append((d, i))
        proposals = [(i, T) for _, i in sorted(cands)[:self.candidates]]
        if code is not None:
            # fern candidates, tracked from keyframe i's own pose
            near = [i for i, _ in proposals] + skip
            proposals += [(i, self._kf_poses[i]) for i in
                          self._fern_candidates(code, j - self.min_gap + 1, self.candidates, near)]
        for i, init in proposals:
            Ti = self._kf_poses[i]
            ok, That, W, rec = self._track(f, self.keyframes[i], Ti, init)
            if ok and self._edge_ok(rec):
                accepted.append((i, np.linalg.inv(Ti) @ That, W))
        if not accepted:
            return False
        edges = self._edges + [(i, j) for i, _, _ in accepted]
        Z = self._Z + [z for _, z, _ in accepted]
        Ws = self._W + [w_ for _, _, w_ in accepted]
        out, rec = self.graph.optimize(np.stack(self._kf_poses), np.array(edges), np.stack(Z), np.stack(Ws))
        if int(rec[0].item()) != 0:
            return False
        self._edges, self._Z, self._W = edges, Z, Ws
        self.loops += [(self.keyframes[i], f) for i, _, _ in accepted]
        self._kf_poses = list(out.cpu().numpy())
        self._poses = [self._kf_poses[k] @ rel for k, rel in self._attach]
        self.closures += 1
        return True

    @torch.no_grad()
    def relocalise(self, pred: torch.Tensor, rgb: torch.Tensor, sparse: Optional[torch.Tensor] = None):
        """The camera-to-world pose (host float64 [4,4]) of a lost frame found against the keyframes, or None: pred
        fp32 [H,W] or [1,H,W] (the relative prediction), rgb fp32 [3,H,W], sparse fp32 [1,H,W] metres (0: none) or
        None (module docstring).  The next `add` must be of this frame."""
        name = "LoopClosure.relocalise"
        if self.places is None:
            raise ValueError(f"{name}: needs places=True")
        h, w = self.size
        if pred.numel() != h * w or pred.dtype != torch.float32 or pred.device != self.device:
            raise ValueError(f"{name}: pred must be fp32 [{h}, {w}] on {self.device}")
        if rgb is None or rgb.numel() != 3 * h * w or rgb.dtype != torch.float32 or rgb.device != self.device:
            raise ValueError(f"{name}: rgb must be fp32 [3, {h}, {w}] on {self.device}")
        pred, rgb = pred.reshape(1, h, w), rgb.reshape(3, h, w)
        self._reloc = None
        if not self.keyframes:
            return None
        code = self.places.encode(pred[0], rgb)[0]
        cands = self._fern_candidates(code, len(self.keyframes), self.candidates)
        metres = None
        if sparse is not None:
            nodes, rec = self._aligner.fit(pred, sparse.reshape(1, h, w))
            if int(rec[0, 1].item()) != 0:
                return None
            metres = self._aligner.apply(pred, nodes)[0]
        for i in cands:
            Ti = self._kf_poses[i]
            kf = self.keyframes[i]
            colour = dict(rgb=rgb, ref_rgb=self._rgb[kf]) if self.photometric > 0 else {}
            if metres is not None:
                tracker = self.tracker
                pose, _, rec = tracker.track(metres, self._metres[kf], self.intrinsics, Ti, Ti, **colour)
            else:
                nodes, frec = self._aligner.fit(pred, self._metres[kf].unsqueeze(0))
                if int(frec[0, 1].item()) != 0:
                    continue
                tracker = self._affine_tracker
                pose, _, rec = tracker.track(pred[0], self._metres[kf], self.intrinsics, Ti, Ti,
                                             init_nodes=nodes, **colour)
            rec = rec.cpu().numpy()
            if not self._edge_ok(rec):
                continue
            W = tracker.information().cpu().numpy()
            if W.shape[0] == 8:                      # marginalise the scale and shift out of the pose's information
                W = W[:6, :6] - W[:6, 6:] @ np.linalg.solve(W[6:, 6:], W[6:, :6])
                W = (W + W.T) / 2
            pose = pose.cpu().numpy()
            self._reloc = (i, np.linalg.inv(Ti) @ pose, W)
            return pose
        return None

    def cancel_relocalisation(self):
        """Forgets the last relocalisation, for a frame that is not added after all."""
        self._reloc = None

    @torch.no_grad()
    def refuse(self, volume):
        """Resets volume and integrates every stored frame, in order, at its current pose (one integrate call)."""
        f = self.frames
        volume.reset()
        volume.integrate(self._metres[:f], self.intrinsics, self.poses, None if self._rgb is None else self._rgb[:f])
        self.refusions += 1
