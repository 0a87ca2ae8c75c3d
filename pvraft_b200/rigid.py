"""The rigid motion behind a scene flow: which points move with the sensor (the static scene), and the rotation and translation
that carries them, fitted on the device without a host synchronisation (csrc/rigid_motion.cu; the algorithm is stated in
include/pvraft_b200.h, pvraft_rigid_objects_fwd); the rigidly moving objects among the other points, by Euclidean clustering
(csrc/clusters.cu) and one such fit per object; and the flow those fits imply.  Both fits are one operation: O segments per
sample, given by labels, and the ego-motion is the case O = 1."""
import math
from typing import NamedTuple

import torch

from . import _lib, ops


class RigidMotion(NamedTuple):
    rotation: torch.Tensor      # [B,3,3] f32: xyz1 @ R^T + t ~ xyz1 + flow on the inliers
    translation: torch.Tensor   # [B,3] f32
    inliers: torch.Tensor       # bool [B,N]: the points (R, t) was fitted to -- the static points, for ego-motion
    count: torch.Tensor         # [B] int32: their number
    degenerate: torch.Tensor    # bool [B]: no proper fit existed; then R = I and t = mean(y) - mean(x) over the inliers


class RigidObjectsFn(torch.autograd.Function):
    """xyz1, flow [B,N,3], labels [B,N] (or None with objects = 1: every point in segment 0) -> R [B,O,3,3], t [B,O,3]
    (differentiable; labels and inlier sets held fixed in the backward, as the neighbours are in the consistency and
    Laplacian terms), inliers [B,N] uint8, count [B,O], degenerate [B,O] uint8."""

    @staticmethod
    def forward(ctx, x, f, labels, objects, threshold, hypotheses, rounds, seed):
        x, f = x.contiguous(), f.contiguous()
        R, t, inl, count, degen, state = ops.rigid_objects(x, f, labels, objects, threshold, hypotheses, rounds, seed)
        ctx.save_for_backward(x, f, labels, inl, state)
        ctx.mark_non_differentiable(inl, count, degen)
        return R, t, inl, count, degen

    @staticmethod
    def backward(ctx, dR, dt, *_):
        x, f, labels, inl, state = ctx.saved_tensors
        b, o = state.shape[0], state.shape[1]
        dR = torch.zeros(b, o, 3, 3, dtype=torch.float32, device=x.device) if dR is None else dR.float().contiguous()
        dt = torch.zeros(b, o, 3, dtype=torch.float32, device=x.device) if dt is None else dt.float().contiguous()
        d_x, d_f = ops.rigid_objects_bwd(x, f, labels, inl, state, dR, dt)
        return d_x, d_f, None, None, None, None, None, None


def _is_int(v):
    return isinstance(v, int) and not isinstance(v, bool)


def _positive(name, arg, v):
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or not v > 0:
        raise ValueError(f'{name}: {arg}={v!r} must be a finite number > 0')
    if float(v) ** 2 >= 3.4e38:
        raise ValueError(f'{name}: {arg}={v!r}: its square is beyond fp32 range')


def _check_fit(name, xyz1, flow, mask, threshold, hypotheses, rounds, seed):
    """The argument checks rigid_motion and rigid_objects share, with the caller's name in the messages -> (B, N)."""
    for arg, v in (('xyz1', xyz1), ('flow', flow)):
        if not torch.is_tensor(v) or v.dim() != 3 or v.shape[-1] != 3 or not v.is_floating_point():
            raise ValueError(f'{name}: expected {arg} [B,N,3] floating point, got '
                             f'{tuple(v.shape) if torch.is_tensor(v) else type(v)}')
    if flow.shape != xyz1.shape:
        raise ValueError(f'{name}: flow {tuple(flow.shape)} does not match xyz1 {tuple(xyz1.shape)}')
    b, n = int(xyz1.shape[0]), int(xyz1.shape[1])
    if mask is not None and (not torch.is_tensor(mask) or mask.dtype != torch.bool or tuple(mask.shape) != (b, n)):
        raise ValueError(f'{name}: mask must be bool [{b},{n}], got '
                         f'{(tuple(mask.shape), mask.dtype) if torch.is_tensor(mask) else type(mask)}')
    _positive(name, 'threshold', threshold)
    if not _is_int(hypotheses) or not 1 <= hypotheses <= ops.RIGID_MAX_HYPOTHESES:
        raise ValueError(f'{name}: hypotheses={hypotheses!r} must be an integer in 1..{ops.RIGID_MAX_HYPOTHESES}')
    if not _is_int(rounds) or not 1 <= rounds <= ops.RIGID_MAX_ROUNDS:
        raise ValueError(f'{name}: rounds={rounds!r} must be an integer in 1..{ops.RIGID_MAX_ROUNDS}')
    if not _is_int(seed) or not 0 <= seed < 2 ** 31:
        raise ValueError(f'{name}: seed={seed!r} must be an integer in 0..2^31-1')
    return b, n


def _need_cuda(*ts):
    for v in ts:
        if v is not None and not v.is_cuda:
            raise _lib.PvraftError('pvraft_b200 kernels need CUDA tensors (no CPU fallback exists)')


def rigid_motion(xyz1, flow, mask=None, threshold=0.1, hypotheses=256, rounds=2, seed=0):
    """The rigid motion (R, t) that the most points of xyz1 [B,N,3] follow under flow [B,N,3]: RANSAC over `hypotheses`
    minimal samples of three points (counter-based: hypothesis h of a given seed draws the same points in any batch), scored
    by the number of points within `threshold` (metres) of each, then `rounds` unweighted Horn/Kabsch refits on the points
    within the threshold of the previous model.  For a LiDAR pair the inliers are the static scene and (R, t) the sensor's
    ego-motion.  mask (bool [B,N], e.g. flow_consistency(...).consistent_12) lists the points that may take part; the others
    are never sampled, counted or fitted.  -> RigidMotion.  rotation and translation carry gradients to xyz1 and flow
    (RigidObjectsFn with one segment per sample).  Nothing synchronises with the host, so the call can be captured in a CUDA
    graph; a sample without a proper fit is reported in `degenerate` on the device.
    threshold = 0.1 m has not been checked against real scans."""
    b, n = _check_fit('rigid_motion', xyz1, flow, mask, threshold, hypotheses, rounds, seed)
    if b < 1 or n < 3:
        raise ValueError(f'rigid_motion: need B >= 1 and at least 3 points, got {tuple(xyz1.shape)}')
    _need_cuda(xyz1, flow, mask)
    labels = None
    if mask is not None:   # where(mask, 0, -1): segment 0 is the masked-in points, built in one elementwise launch
        labels = torch.empty(b, n, dtype=torch.int32, device=mask.device)
        torch.add(mask, -1, out=labels)
    R, t, inl, count, degen = RigidObjectsFn.apply(xyz1.float(), flow.float(), labels, 1, float(threshold), hypotheses, rounds, seed)
    return RigidMotion(R.view(b, 3, 3), t.view(b, 3), inl.bool(), count.view(b), degen.view(b).bool())


class RigidObjects(NamedTuple):
    labels: torch.Tensor        # [B,N] int32: the object of each point, -1 for none
    num_objects: torch.Tensor   # [B] int32: objects 0 .. num_objects - 1 exist
    rotation: torch.Tensor      # [B,O,3,3] f32 (O = max_objects): xyz1 @ R^T + t ~ xyz1 + flow on the object's inliers
    translation: torch.Tensor   # [B,O,3] f32
    count: torch.Tensor         # [B,O] int32: the number of inliers of each object's fit (0 for an empty slot)
    degenerate: torch.Tensor    # bool [B,O]: no proper fit (always for an empty slot: R = I, t = 0)
    inliers: torch.Tensor       # bool [B,N]: an inlier of its own object's fit


def rigid_objects(xyz1, flow, mask=None, radius=0.5, min_points=10, max_objects=64, flow_radius=None, threshold=0.1, hypotheses=256,
                  rounds=2, seed=0):
    """The rigidly moving objects of a scene flow and the motion of each: the points allowed by mask (bool [B,N]; all with
    None; typically consistent & ~ego.inliers, the points that do not move with the sensor) are clustered by single linkage --
    two points are adjacent within `radius` (metres; with flow_radius, their flows must also lie within flow_radius, which
    separates touching objects that move differently) -- and the components of at least `min_points` points, largest first
    (smallest point id on ties), become objects 0 .. num_objects - 1, at most `max_objects`.  Each object then gets exactly
    the fit rigid_motion(xyz1[b:b+1], flow[b:b+1], mask=labels[b:b+1] == o, threshold, hypotheses, rounds, seed) would give
    it.  -> RigidObjects with static shapes (O = max_objects slots); rotation and translation carry gradients to xyz1 and
    flow (RigidObjectsFn).  Nothing synchronises with the host, so the call can be captured in a CUDA graph.
    radius = 0.5 m and min_points = 10 have not been checked against real scans."""
    b, n = _check_fit('rigid_objects', xyz1, flow, mask, threshold, hypotheses, rounds, seed)
    if b < 1 or n < 1:
        raise ValueError(f'rigid_objects: need B >= 1 and N >= 1, got {tuple(xyz1.shape)}')
    if b * n >= 2 ** 31:
        raise ValueError(f'rigid_objects: B N = {b * n} points (at most 2^31 - 1)')
    _positive('rigid_objects', 'radius', radius)
    if flow_radius is not None:
        _positive('rigid_objects', 'flow_radius', flow_radius)
    if not _is_int(min_points) or min_points < 1:
        raise ValueError(f'rigid_objects: min_points={min_points!r} must be an integer >= 1')
    if not _is_int(max_objects) or not 1 <= max_objects <= ops.RIGID_MAX_OBJECTS:
        raise ValueError(f'rigid_objects: max_objects={max_objects!r} must be an integer in 1..{ops.RIGID_MAX_OBJECTS}')
    _need_cuda(xyz1, flow, mask)
    x, f = xyz1.float().contiguous(), flow.float().contiguous()
    m = None if mask is None else mask.contiguous().view(torch.uint8)
    labels, num, _ = ops.euclidean_clusters(x, f if flow_radius is not None else None, m, float(radius),
                                            None if flow_radius is None else float(flow_radius), min_points, max_objects)
    R, t, inl, count, degen = RigidObjectsFn.apply(x, f, labels, max_objects, float(threshold), hypotheses, rounds, seed)
    return RigidObjects(labels, num, R, t, count, degen.bool(), inl.bool())


def rigid_flow(xyz1, flow, objects, ego=None):
    """The flow the rigid fits imply, [B,N,3]: an inlier of a non-degenerate object o gets x R_o^T + t_o - x; otherwise an
    inlier of a non-degenerate `ego` (a RigidMotion, e.g. rigid_motion's ego-motion) gets x R_e^T + t_e - x; every other
    point keeps `flow`.  Differentiable (ATen), through the fits' rotation and translation and through flow."""
    if not isinstance(objects, RigidObjects):
        raise ValueError(f'rigid_flow: objects must be a RigidObjects, got {type(objects)}')
    if ego is not None and not isinstance(ego, RigidMotion):
        raise ValueError(f'rigid_flow: ego must be a RigidMotion or None, got {type(ego)}')
    for name, v in (('xyz1', xyz1), ('flow', flow)):
        if not torch.is_tensor(v) or v.dim() != 3 or v.shape[-1] != 3 or not v.is_floating_point():
            raise ValueError(f'rigid_flow: expected {name} [B,N,3] floating point, got '
                             f'{tuple(v.shape) if torch.is_tensor(v) else type(v)}')
    if flow.shape != xyz1.shape or tuple(objects.labels.shape) != tuple(xyz1.shape[:2]) or \
            (ego is not None and tuple(ego.inliers.shape) != tuple(xyz1.shape[:2])):
        raise ValueError(f'rigid_flow: xyz1 {tuple(xyz1.shape)}, flow {tuple(flow.shape)}, labels {tuple(objects.labels.shape)}'
                         f'{"" if ego is None else f", ego inliers {tuple(ego.inliers.shape)}"} do not agree')
    out = flow
    if ego is not None:
        moved = torch.einsum('bnk,bjk->bnj', xyz1, ego.rotation) + ego.translation[:, None, :] - xyz1
        use = ego.inliers & ~ego.degenerate[:, None]
        out = torch.where(use[..., None], moved, out)
    lab = objects.labels.long()
    idx = lab.clamp_min(0)
    R = torch.gather(objects.rotation, 1, idx[..., None, None].expand(-1, -1, 3, 3))
    t = torch.gather(objects.translation, 1, idx[..., None].expand(-1, -1, 3))
    moved = torch.einsum('bnjk,bnk->bnj', R, xyz1) + t - xyz1
    use = objects.inliers & (lab >= 0) & ~torch.gather(objects.degenerate, 1, idx)
    return torch.where(use[..., None], moved, out)
