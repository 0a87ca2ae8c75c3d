"""The rigid motion behind a scene flow: which points move with the sensor (the static scene), and the rotation and translation
that carries them, fitted on the device without a host synchronisation (csrc/rigid_motion.cu; the algorithm is stated in
include/pvraft_b200.h, pvraft_rigid_motion_fwd)."""
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


class RigidFitFn(torch.autograd.Function):
    """xyz1, flow [B,N,3] -> R [B,3,3], t [B,3] (differentiable; the inlier set is held fixed in the backward, as the
    neighbours are in the consistency and Laplacian terms), inliers [B,N] uint8, count [B], degenerate [B] uint8."""

    @staticmethod
    def forward(ctx, x, f, mask, threshold, hypotheses, rounds, seed):
        x, f = x.contiguous(), f.contiguous()
        R, t, inl, count, degen, state = ops.rigid_motion(x, f, mask, threshold, hypotheses, rounds, seed)
        ctx.save_for_backward(x, f, inl, state)
        ctx.mark_non_differentiable(inl, count, degen)
        return R, t, inl, count, degen

    @staticmethod
    def backward(ctx, dR, dt, *_):
        x, f, inl, state = ctx.saved_tensors
        dR = torch.zeros(x.shape[0], 3, 3, dtype=torch.float32, device=x.device) if dR is None else dR.float().contiguous()
        dt = torch.zeros(x.shape[0], 3, dtype=torch.float32, device=x.device) if dt is None else dt.float().contiguous()
        d_x, d_f = ops.rigid_motion_bwd(x, f, inl, state, dR, dt)
        return d_x, d_f, None, None, None, None, None


def _is_int(v):
    return isinstance(v, int) and not isinstance(v, bool)


def rigid_motion(xyz1, flow, mask=None, threshold=0.1, hypotheses=256, rounds=2, seed=0):
    """The rigid motion (R, t) that the most points of xyz1 [B,N,3] follow under flow [B,N,3]: RANSAC over `hypotheses`
    minimal samples of three points (counter-based: hypothesis h of a given seed draws the same points in any batch), scored
    by the number of points within `threshold` (metres) of each, then `rounds` unweighted Horn/Kabsch refits on the points
    within the threshold of the previous model.  For a LiDAR pair the inliers are the static scene and (R, t) the sensor's
    ego-motion.  mask (bool [B,N], e.g. flow_consistency(...).consistent_12) lists the points that may take part; the others
    are never sampled, counted or fitted.  -> RigidMotion.  rotation and translation carry gradients to xyz1 and flow
    (RigidFitFn).  Nothing synchronises with the host, so the call can be captured in a CUDA graph; a sample without a
    proper fit is reported in `degenerate` on the device.
    threshold = 0.1 m has not been checked against real scans."""
    for name, v in (('xyz1', xyz1), ('flow', flow)):
        if not torch.is_tensor(v) or v.dim() != 3 or v.shape[-1] != 3 or not v.is_floating_point():
            raise ValueError(f'rigid_motion: expected {name} [B,N,3] floating point, got '
                             f'{tuple(v.shape) if torch.is_tensor(v) else type(v)}')
    if flow.shape != xyz1.shape:
        raise ValueError(f'rigid_motion: flow {tuple(flow.shape)} does not match xyz1 {tuple(xyz1.shape)}')
    b, n = int(xyz1.shape[0]), int(xyz1.shape[1])
    if b < 1 or n < 3:
        raise ValueError(f'rigid_motion: need B >= 1 and at least 3 points, got {tuple(xyz1.shape)}')
    if mask is not None and (not torch.is_tensor(mask) or mask.dtype != torch.bool or tuple(mask.shape) != (b, n)):
        raise ValueError(f'rigid_motion: mask must be bool [{b},{n}], got '
                         f'{(tuple(mask.shape), mask.dtype) if torch.is_tensor(mask) else type(mask)}')
    if isinstance(threshold, bool) or not isinstance(threshold, (int, float)) or not math.isfinite(threshold) or not threshold > 0:
        raise ValueError(f'rigid_motion: threshold={threshold!r} must be a finite number > 0')
    if not _is_int(hypotheses) or not 1 <= hypotheses <= ops.RIGID_MAX_HYPOTHESES:
        raise ValueError(f'rigid_motion: hypotheses={hypotheses!r} must be an integer in 1..{ops.RIGID_MAX_HYPOTHESES}')
    if not _is_int(rounds) or not 1 <= rounds <= ops.RIGID_MAX_ROUNDS:
        raise ValueError(f'rigid_motion: rounds={rounds!r} must be an integer in 1..{ops.RIGID_MAX_ROUNDS}')
    if not _is_int(seed) or not 0 <= seed < 2 ** 31:
        raise ValueError(f'rigid_motion: seed={seed!r} must be an integer in 0..2^31-1')
    if float(threshold) ** 2 >= 3.4e38:
        raise ValueError(f'rigid_motion: threshold={threshold!r}: its square is beyond fp32 range')
    for v in (xyz1, flow) + (() if mask is None else (mask,)):
        if not v.is_cuda:
            raise _lib.PvraftError('pvraft_b200 kernels need CUDA tensors (no CPU fallback exists)')
    m = None if mask is None else mask.contiguous().view(torch.uint8)
    R, t, inl, count, degen = RigidFitFn.apply(xyz1.float(), flow.float(), m, float(threshold), hypotheses, rounds, seed)
    return RigidMotion(R, t, inl.bool(), count, degen.bool())
