"""Multi-object tracking from scene flow: the rigidly moving objects that pvraft_b200.rigid_objects finds on each pair of a scan
sequence are associated with the objects of the previous pair on the device, so that each keeps one identity over its life
and carries its rigid motion since it was born (csrc/tracks.cu; the rule is stated in include/pvraft_b200.h,
pvraft_track_objects_fwd).  Nothing synchronises with the host."""
import math
from typing import NamedTuple

import torch

from . import ops
from ._lib import PvraftError
from .rigid import RigidMotion, RigidObjects, rigid_flow


class ObjectTracks(NamedTuple):
    track_id: torch.Tensor      # [B,O] int32: the track of each object slot, -1 for an empty slot
    labels: torch.Tensor        # [B,N] int32: each point's track id, -1 for none
    matched: torch.Tensor       # [B,O] int32: the previous step's object slot, -1 for a new track or an empty slot
    age: torch.Tensor           # [B,O] int32: steps since the track was born (0 at birth), -1 for an empty slot
    rotation: torch.Tensor      # [B,O,3,3] f32 and
    translation: torch.Tensor   # [B,O,3] f32: the object's motion from the scan it was born on to this scan (x R^T + t)


def _check_params(gate, min_overlap):
    if isinstance(gate, bool) or not isinstance(gate, (int, float)) or not math.isfinite(gate) or not gate > 0:
        raise ValueError(f'ObjectTracker: gate={gate!r} must be a finite number > 0')
    if float(gate) ** 2 >= 3.4e38:
        raise ValueError(f'ObjectTracker: gate={gate!r}: its square is beyond fp32 range')
    if isinstance(min_overlap, bool) or not isinstance(min_overlap, (int, float)) or \
            not ops.TRACK_MIN_OVERLAP <= min_overlap <= 1:
        raise ValueError(f'ObjectTracker: min_overlap={min_overlap!r} must be a number in [1/16, 1]')


class ObjectTracker:
    """Tracks the objects of a scan sequence, one pair at a time.

    step(xyz1 [B,N,3], flow [B,N,3], objects, ego=None) takes the first cloud of a pair, its flow, the pair's
    `rigid_objects(xyz1, flow, ...)` and optionally its ego-motion `rigid_motion(xyz1, flow, ...)`, and returns
    ObjectTracks for the slots of `objects`.  The previous step's cloud X is moved by its rigid flow G = rigid_flow(X, flow,
    objects, ego) (the static scene by the ego fit, each object's inliers by their object's fit, every other point by its
    own flow); each point of xyz1 votes, through the nearest moved point W_i = X_i + G_i within `gate` metres
    (ops.flow_propagate with k = 1), for that point's previous object.  A current object and a previous one whose shared
    votes are at least `min_overlap` of the current object's points may match; the pairs are matched greedily, largest
    overlap first.  A matched object keeps its track id and composes its previous fit after its pose; an unmatched one is
    a new track (fresh ids, never reused) with the identity pose.  A track without a match in a step ends.

    N and the slot count O may change from step to step; the batch size and device may not (reset() starts a new
    sequence).  Nothing reads a device value on the host, so a step never synchronises.  The outputs carry no gradient:
    the tracker keeps detached copies of what it needs as state.  gate = 0.5 m and min_overlap = 0.5 have not been
    checked against real scans."""

    def __init__(self, gate=0.5, min_overlap=0.5):
        _check_params(gate, min_overlap)
        self.gate, self.min_overlap = gate, min_overlap
        self.reset()

    def reset(self):
        """Forget the sequence: the next step is a first step, and track ids start again at 0."""
        self._prev = None      # (X, G, labels, track, age, pose, R, t) of the previous step, for ops.track_objects
        self._next_id = None   # [B] int32 on the device: the next fresh track id of each sample

    def step(self, xyz1, flow, objects, ego=None):
        _check_params(self.gate, self.min_overlap)
        for name, v in (('xyz1', xyz1), ('flow', flow)):
            if not torch.is_tensor(v) or v.dim() != 3 or v.shape[-1] != 3 or not v.is_floating_point() or v.shape[0] < 1 or v.shape[1] < 1:
                raise ValueError(f'ObjectTracker.step: expected {name} [B,N,3] floating point with B, N >= 1, got '
                                 f'{tuple(v.shape) if torch.is_tensor(v) else type(v)}')
        if flow.shape != xyz1.shape:
            raise ValueError(f'ObjectTracker.step: flow {tuple(flow.shape)} does not match xyz1 {tuple(xyz1.shape)}')
        if not isinstance(objects, RigidObjects):
            raise ValueError(f'ObjectTracker.step: objects must be a RigidObjects, got {type(objects)}')
        if ego is not None and not isinstance(ego, RigidMotion):
            raise ValueError(f'ObjectTracker.step: ego must be a RigidMotion or None, got {type(ego)}')
        b, n = int(xyz1.shape[0]), int(xyz1.shape[1])
        o = int(objects.rotation.shape[1]) if objects.rotation.dim() == 4 else -1
        if tuple(objects.labels.shape) != (b, n) or tuple(objects.num_objects.shape) != (b,) or \
                tuple(objects.rotation.shape) != (b, o, 3, 3) or tuple(objects.translation.shape) != (b, o, 3) or \
                not 1 <= o <= ops.RIGID_MAX_OBJECTS or objects.labels.dtype != torch.int32 or objects.num_objects.dtype != torch.int32:
            raise ValueError(f'ObjectTracker.step: objects (labels {tuple(objects.labels.shape)}, num_objects '
                             f'{tuple(objects.num_objects.shape)}, rotation {tuple(objects.rotation.shape)}, translation '
                             f'{tuple(objects.translation.shape)}) do not fit xyz1 {tuple(xyz1.shape)} with 1..'
                             f'{ops.RIGID_MAX_OBJECTS} int32-labelled slots')
        if ego is not None and tuple(ego.inliers.shape) != (b, n):
            raise ValueError(f'ObjectTracker.step: ego inliers {tuple(ego.inliers.shape)} do not match xyz1 {tuple(xyz1.shape)}')
        if self._prev is not None:
            x_prev = self._prev[0]
            if x_prev.shape[0] != b:
                raise ValueError(f'ObjectTracker.step: batch size {b} differs from the previous step\'s {x_prev.shape[0]} '
                                 '(reset() starts a new sequence)')
            if xyz1.device != x_prev.device:
                raise ValueError(f'ObjectTracker.step: xyz1 on {xyz1.device}, the previous step on {x_prev.device} '
                                 '(reset() starts a new sequence)')
        for v in (xyz1, flow, objects.labels, objects.num_objects, objects.rotation, objects.translation):
            if not v.is_cuda:
                raise PvraftError('pvraft_b200 kernels need CUDA tensors (no CPU fallback exists)')

        with torch.no_grad():
            x = xyz1.detach().float().contiguous()
            labels = objects.labels.contiguous()
            num = objects.num_objects.contiguous()
            if self._next_id is None:
                self._next_id = torch.zeros(b, dtype=torch.int32, device=x.device)
            nn = None
            if self._prev is not None:
                nn = ops.flow_propagate(self._prev[0], self._prev[1], x, k=1, want_idx=True)[1].view(b, n)
            _, _, match, track, age, pose = ops.track_objects(self._prev, x, labels, num, o, nn, self.gate, self.min_overlap,
                                                              self._next_id)
            lab = labels.long()
            inside = (lab >= 0) & (lab < o)
            point_track = torch.where(inside, torch.gather(track, 1, lab.clamp(0, o - 1)), -1).to(torch.int32)
            g = rigid_flow(x, flow.detach().float(), objects, ego).contiguous()   # a new tensor (torch.where)
            # the state is the tracker's own copy: the caller may reuse or change its tensors, and those returned
            self._prev = (x.clone(), g, labels.clone(), track.clone(), age.clone(), pose,
                          objects.rotation.detach().float().contiguous().clone(), objects.translation.detach().float().contiguous().clone())
        return ObjectTracks(track, point_track, match, age, pose[..., :9].float().reshape(b, o, 3, 3), pose[..., 9:].float())
