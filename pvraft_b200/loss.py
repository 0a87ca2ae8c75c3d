"""Device-side loss and metrics -- mirrors of tools/loss.py:4-40 and tools/metric.py:6-79 with the same signatures
(`batch["ground_truth"] = [mask [B,N,1], flow [B,N,3]]`), one kernel pass per prediction and no host synchronisation
inside a training step (the reference indexes `error[mask > 0]`, a host-synchronising boolean gather, per prediction).
`tools/loss.py` and `tools/metric.py` of this repository re-export them under the reference's import paths."""
from typing import NamedTuple

import torch

from . import ops
from ._lib import lib


def _gt(batch):
    mask, flow = batch['ground_truth'][0], batch['ground_truth'][1]
    return mask[..., 0].contiguous().float(), flow.contiguous().float()


def _metrics(est, gt, mask):
    acc = torch.zeros(8, dtype=torch.float64, device=est.device)
    ws = ops._det_workspace(lib().pvraft_flow_metrics_det_workspace_bytes, device=est.device)
    ops._count(lib().pvraft_flow_metrics_fwd(ops._p(est), ops._p(gt), ops._p(mask), est.numel() // 3, acc.data_ptr(), ops._p(ws, torch.uint8),
                                             ops._stream()), 'flow_metrics')
    return acc


class MaskedL1Fn(torch.autograd.Function):
    """weight * mean over the valid points and their 3 components of |est - gt| (tools/loss.py:34-38)."""

    @staticmethod
    def forward(ctx, est, gt, mask, weight):
        est = est.contiguous()
        acc = _metrics(est, gt, mask)
        ctx.save_for_backward(est, gt, mask, acc)
        ctx.weight = float(weight)
        return (acc[0] / (3.0 * acc[1])).float() * ctx.weight

    @staticmethod
    def backward(ctx, g):
        est, gt, mask, acc = ctx.saved_tensors
        d = torch.empty_like(est)
        ops._count(lib().pvraft_flow_l1_bwd(ops._p(est), ops._p(gt), ops._p(mask), est.numel() // 3, acc.data_ptr(),
                                            ops._p(g.contiguous().float().reshape(1)), ctx.weight, ops._p(d), ops._stream()), 'flow_l1_bwd')
        return d, None, None, None


def compute_loss(est_flow, batch):
    """tools/loss.py:16-40."""
    mask, flow = _gt(batch)
    return MaskedL1Fn.apply(est_flow.float(), flow, mask, 1.0)


def sequence_loss(est_flow, batch, gamma=0.8):
    """tools/loss.py:4-13: sum_i gamma^(n-i-1) * compute_loss(est_flow[i], batch)."""
    mask, flow = _gt(batch)
    n = len(est_flow)
    total = 0
    for i in range(n):
        total = total + MaskedL1Fn.apply(est_flow[i].float(), flow, mask, gamma ** (n - i - 1))
    return total


# ---- self-supervised losses (no ground truth: only batch['sequence'] is read) ------------------------------------------------
class ChamferFn(torch.autograd.Function):
    """W [S,N,3], P2 [B,M,3] -> [S]: C_s = mean_i min_j ||W_i - P2_j||^2 + mean_j min_i ||W_i - P2_j||^2, sample s against
    P2[s % B].  The nearest-neighbour indices are saved; they carry no gradient."""

    @staticmethod
    def forward(ctx, w, p2):
        w, p2 = w.contiguous(), p2.contiguous()
        acc, nn_ab, nn_ba = ops.chamfer(w, p2)
        ctx.save_for_backward(w, p2, nn_ab, nn_ba)
        return (acc[:, 0] / w.shape[1] + acc[:, 1] / p2.shape[1]).float()

    @staticmethod
    def backward(ctx, g):
        w, p2, nn_ab, nn_ba = ctx.saved_tensors
        d_w, d_p2 = ops.chamfer_bwd(w, p2, nn_ab, nn_ba, g.contiguous().float(), want_db=ctx.needs_input_grad[1])
        return d_w, d_p2


class SmoothFn(torch.autograd.Function):
    """f [S,N,3], nbr [B,N,k] int32 -> [S]: S_s = mean over the points and their k neighbours of ||f_j - f_i||."""

    @staticmethod
    def forward(ctx, f, nbr):
        f = f.contiguous()
        acc = ops.flow_smooth(f, nbr)
        ctx.save_for_backward(f, nbr)
        return (acc / (f.shape[1] * nbr.shape[2])).float()

    @staticmethod
    def backward(ctx, g):
        f, nbr = ctx.saved_tensors
        return ops.flow_smooth_bwd(f, nbr, g.contiguous().float()), None


class LaplacianFn(torch.autograd.Function):
    """W [S,N,3], P2 [B,M,3], g1 [B,N,k_lap], g2 [B,M,k_lap] int32 -> [S]: R_s = mean_i ||Lhat_i - L(W)_i||^2, with L(W) the
    Laplacian of W over P1's graph g1 and Lhat_i the Laplacian of P2 over g2 interpolated at W_i from its k_int nearest points
    of P2[s % B] (weights 1 / (d^2 + 1e-8)).  The interpolation neighbours are saved; they and the graphs carry no gradient."""

    @staticmethod
    def forward(ctx, w, p2, g1, g2, k_int):
        w, p2 = w.contiguous(), p2.contiguous()
        l2 = ops.cloud_laplacian(p2, g2)
        acc, nn_idx, res = ops.laplacian(w, p2, l2, g1, k_int)
        ctx.save_for_backward(w, p2, l2, g1, g2, nn_idx, res)
        return (acc / w.shape[1]).float()

    @staticmethod
    def backward(ctx, g):
        w, p2, l2, g1, g2, nn_idx, res = ctx.saved_tensors
        d_w, d_p2, d_l2 = ops.laplacian_bwd(w, p2, l2, g1, nn_idx, res, g.contiguous().float(), want_dp2=ctx.needs_input_grad[1])
        if d_p2 is not None:
            ops.cloud_laplacian_bwd(d_l2, g2, d_p2)
        return d_w, d_p2, None, None, None


class ConsistencyFn(torch.autograd.Function):
    """W [S,N,3] (P1 + f12), f12 [S,N,3], P2 [B,M,3], f21 [S,M,3] -> [S]: F_s = mean_i ||f12_i + bhat_i||^2, with bhat_i the
    reverse flow f21 interpolated at W_i from its k nearest points of P2[s % B] (weights 1 / (d^2 + 1e-8), the Laplacian
    term's).  The neighbours are saved; they carry no gradient."""

    @staticmethod
    def forward(ctx, w, f12, p2, f21, k):
        w, f12, p2, f21 = w.contiguous(), f12.contiguous(), p2.contiguous(), f21.contiguous()
        acc, nn_idx, res, _ = ops.flow_consistency(w, f12, p2, f21, k, 0.0, 0.0)
        ctx.save_for_backward(w, p2, f21, nn_idx, res)
        return (acc / w.shape[1]).float()

    @staticmethod
    def backward(ctx, g):
        w, p2, f21, nn_idx, res = ctx.saved_tensors
        d_w, d_f12, d_p2, d_f21 = ops.flow_consistency_bwd(w, p2, f21, nn_idx, res, g.contiguous().float(),
                                                           want_dp2=ctx.needs_input_grad[2])
        return d_w, d_f12, d_p2, d_f21, None


def _laplacian_checks(w_laplacian, k_lap, k_int, npts, m):
    if isinstance(k_lap, bool) or not isinstance(k_lap, int) or not 2 <= k_lap <= ops.KNN:
        raise ValueError(f'k_lap={k_lap!r}: the Laplacian graphs take 2 to {ops.KNN} neighbours')
    if isinstance(k_int, bool) or not isinstance(k_int, int) or not 1 <= k_int <= ops.LAPLACIAN_MAX_K_INT:
        raise ValueError(f'k_int={k_int!r}: the Laplacian is interpolated from 1 to {ops.LAPLACIAN_MAX_K_INT} neighbours')
    if w_laplacian != 0 and (k_lap > npts or k_lap > m or k_int > m):
        raise ValueError(f'k_lap={k_lap}, k_int={k_int}: the clouds have {npts} and {m} points')


def _self_supervised(flows, batch, k, w_chamfer, w_smooth, w_laplacian=0.0, k_lap=10, k_int=5):
    """flows [n,B,N,3] -> [n]: mean over the batch of w_chamfer * C + w_smooth * S (+ w_laplacian * R when it is not 0), one
    launch per term and direction."""
    p1, p2 = batch['sequence'][0], batch['sequence'][1]
    n, b, npts = flows.shape[0], flows.shape[1], flows.shape[2]
    if not 1 <= k <= ops.KNN:
        raise ValueError(f'k={k}: the smoothness graph takes 1 to {ops.KNN} neighbours')
    if p1.dim() != 3 or p2.dim() != 3 or p1.shape[-1] != 3 or p2.shape[-1] != 3 or p2.shape[0] != p1.shape[0]:
        raise ValueError(f"batch['sequence'] must be [P1 [B,N,3], P2 [B,M,3]], got {tuple(p1.shape)} and {tuple(p2.shape)}")
    if tuple(flows.shape[1:]) != tuple(p1.shape):
        raise ValueError(f'flow {tuple(flows.shape[1:])} does not match the first cloud {tuple(p1.shape)}')
    if k > npts:
        raise ValueError(f'k={k} exceeds the {npts} points of the first cloud')
    _laplacian_checks(w_laplacian, k_lap, k_int, npts, p2.shape[1])
    p1f = p1.float()
    nbr = ops.knn(p1f.detach().contiguous(), p1f.detach().contiguous(), k, mode=0)
    w = (flows + p1f).reshape(n * b, npts, 3)
    p2f = p2.float()
    per = w_chamfer * ChamferFn.apply(w, p2f) + w_smooth * SmoothFn.apply(flows.reshape(n * b, npts, 3), nbr)
    if w_laplacian != 0:
        g1 = ops.knn(p1f.detach().contiguous(), p1f.detach().contiguous(), k_lap, mode=0)
        g2 = ops.knn(p2f.detach().contiguous(), p2f.detach().contiguous(), k_lap, mode=0)
        per = per + w_laplacian * LaplacianFn.apply(w, p2f, g1, g2, k_int)
    return per.view(n, b).mean(1)


def _check_k_cons(k_cons):
    if isinstance(k_cons, bool) or not isinstance(k_cons, int) or not 1 <= k_cons <= ops.CONSISTENCY_MAX_K:
        raise ValueError(f'k_cons={k_cons!r}: the reverse flow is interpolated from 1 to {ops.CONSISTENCY_MAX_K} neighbours')


def _is_pair(est_flow, sequence):
    """True for the (forward, backward) pair that model(p, n, bidirectional=True) returns."""
    if not isinstance(est_flow, tuple) or len(est_flow) != 2:
        return False
    if sequence:
        return all(isinstance(e, (list, tuple)) for e in est_flow)
    return all(torch.is_tensor(e) for e in est_flow)


def _pair_loss(pair, batch, k_cons, w_consistency, one):
    """The loss of a bidirectional forward: one(flows [n,B,N,3], batch) per direction, the reverse one with P1 and P2 swapped,
    each plus w_consistency * F of its direction (ConsistencyFn, launched only when w_consistency != 0) -> [n], the mean of the
    two directions."""
    p1, p2 = batch['sequence'][0], batch['sequence'][1]
    f12, f21 = pair
    if w_consistency != 0 and k_cons > min(p1.shape[1], p2.shape[1]):
        raise ValueError(f'k_cons={k_cons}: the clouds have {p1.shape[1]} and {p2.shape[1]} points')
    back = dict(batch, sequence=[p2, p1])
    per12, per21 = one(f12, batch), one(f21, back)
    if w_consistency != 0:
        n, b = f12.shape[0], f12.shape[1]
        p1f, p2f = p1.float(), p2.float()
        a = f12.reshape(n * b, -1, 3)
        r = f21.reshape(n * b, -1, 3)
        per12 = per12 + w_consistency * ConsistencyFn.apply((f12 + p1f).reshape(n * b, -1, 3), a, p2f, r, k_cons).view(n, b).mean(1)
        per21 = per21 + w_consistency * ConsistencyFn.apply((f21 + p2f).reshape(n * b, -1, 3), r, p1f, a, k_cons).view(n, b).mean(1)
    return (per12 + per21) / 2


def self_supervised_loss(est_flow, batch, k=9, w_chamfer=1.0, w_smooth=1.0, w_laplacian=0.0, k_lap=10, k_int=5, w_consistency=0.0,
                         k_cons=3):
    """Self-supervised analogue of compute_loss for one flow [B,N,3] (what RSF_refine returns): mean over the batch of
    w_chamfer * Chamfer(P1 + flow, P2) + w_smooth * smoothness of the flow over P1's k-nearest-neighbour graph
    + w_laplacian * Laplacian regularity (LaplacianFn: P1's and P2's k_lap-nearest-neighbour graphs, P2's Laplacian
    interpolated from k_int points).  w_laplacian = 0 builds and launches nothing for the third term.
    est_flow may also be the pair (flow_12 [B,N1,3], flow_21 [B,N2,3]) of a bidirectional forward: then every term is taken
    per direction (P1 and P2 swapped for the reverse one), each direction adds w_consistency * its forward-backward
    consistency (ConsistencyFn, the reverse flow interpolated from k_cons points; nothing is launched for it at 0), and the
    two directions are averaged.  A single flow with w_consistency != 0 raises ValueError."""
    _check_k_cons(k_cons)

    def run(flows, bt):
        return _self_supervised(flows, bt, k, w_chamfer, w_smooth, w_laplacian, k_lap, k_int)

    if _is_pair(est_flow, sequence=False):
        return _pair_loss((est_flow[0].float().unsqueeze(0), est_flow[1].float().unsqueeze(0)), batch, k_cons, w_consistency, run)[0]
    if w_consistency != 0:
        raise ValueError('w_consistency needs the (forward, backward) pair of a bidirectional forward, got a single flow')
    return run(est_flow.float().unsqueeze(0), batch)[0]


def sequence_self_supervised_loss(est_flow, batch, gamma=0.8, k=9, w_chamfer=1.0, w_smooth=1.0, w_laplacian=0.0, k_lap=10, k_int=5,
                                  w_consistency=0.0, k_cons=3):
    """Self-supervised analogue of sequence_loss: sum_i gamma^(n-i-1) * self_supervised_loss(est_flow[i], batch), with all n
    predictions in one forward and one backward launch per term.  est_flow may also be the pair (flows_12, flows_21) of lists
    that a bidirectional RSF forward returns: see self_supervised_loss for the pair and w_consistency / k_cons."""
    _check_k_cons(k_cons)

    def run(flows, bt):
        return _self_supervised(flows, bt, k, w_chamfer, w_smooth, w_laplacian, k_lap, k_int)

    if _is_pair(est_flow, sequence=True):
        f12 = torch.stack([f.float() for f in est_flow[0]])
        f21 = torch.stack([f.float() for f in est_flow[1]])
        if f12.shape[0] != f21.shape[0]:
            raise ValueError(f'the two directions have {f12.shape[0]} and {f21.shape[0]} predictions')
        per = _pair_loss((f12, f21), batch, k_cons, w_consistency, run)
    else:
        if w_consistency != 0:
            raise ValueError('w_consistency needs the (forward, backward) pair of a bidirectional forward, got a single flow sequence')
        per = run(torch.stack([f.float() for f in est_flow]), batch)
    n = per.shape[0]
    weights = torch.pow(float(gamma), torch.arange(n - 1, -1, -1, dtype=torch.float32, device=per.device))
    return (weights * per).sum()


class Consistency(NamedTuple):
    res_12: torch.Tensor          # [B,N1,3] flow_12 + flow_21 interpolated at xyz1 + flow_12: the round trip's residual
    res_21: torch.Tensor          # [B,N2,3] the same from the second cloud
    consistent_12: torch.Tensor   # bool [B,N1]: the two flows agree at this point of xyz1
    consistent_21: torch.Tensor   # bool [B,N2]


def flow_consistency(xyz1, flow_12, xyz2, flow_21, k=3, alpha=0.01, beta=0.0025):
    """The forward-backward check of a pair of flows (what model(p, n, bidirectional=True) estimates): at every point of each
    cloud, the flow found there is followed by the other direction's flow interpolated where it lands (inverse squared
    distance over its k nearest points of the other cloud), and the point is consistent when the round trip returns:
    ||res||^2 < alpha (||f||^2 + ||bhat||^2) + beta.  The points of xyz1 that fail are the usual estimate of the ones with no
    counterpart in xyz2 (occluded, or out of view).  Runs under no_grad, one launch per direction.
    alpha = 0.01 is UnFlow's value for optical flow; beta = 0.05^2 m^2 is the 5 cm "strict" threshold of compute_epe.  Neither
    has been checked against annotated occlusions of a scene-flow dataset."""
    for name, t in (('xyz1', xyz1), ('flow_12', flow_12), ('xyz2', xyz2), ('flow_21', flow_21)):
        if not torch.is_tensor(t) or t.dim() != 3 or t.shape[-1] != 3:
            raise ValueError(f'flow_consistency: expected {name} [B,n,3], got {tuple(t.shape) if torch.is_tensor(t) else type(t)}')
    if flow_12.shape != xyz1.shape or flow_21.shape != xyz2.shape or xyz1.shape[0] != xyz2.shape[0]:
        raise ValueError(f'flow_consistency: flows {tuple(flow_12.shape)}, {tuple(flow_21.shape)} must match the clouds '
                         f'{tuple(xyz1.shape)}, {tuple(xyz2.shape)} of one batch')
    with torch.no_grad():
        p1, p2 = xyz1.float().contiguous(), xyz2.float().contiguous()
        f12, f21 = flow_12.float().contiguous(), flow_21.float().contiguous()
        _, _, r12, ok12 = ops.flow_consistency((p1 + f12).contiguous(), f12, p2, f21, k, alpha, beta)
        _, _, r21, ok21 = ops.flow_consistency((p2 + f21).contiguous(), f21, p1, f12, k, alpha, beta)
    return Consistency(r12, r21, ok12.bool(), ok21.bool())


def compute_epe_train(est_flow, batch):
    """tools/metric.py:6-31 -> 0-dim tensor on the device (the caller decides when to synchronise)."""
    mask, flow = _gt(batch)
    acc = _metrics(est_flow.detach().contiguous().float(), flow, mask)
    return (acc[2] / acc[1]).float()


def compute_epe(est_flow, batch):
    """tools/metric.py:34-79 -> (EPE3D, acc3d_strict, acc3d_relax, outlier) as python floats (one read-back of 6 doubles;
    the reference moves both flow tensors to the host and calls `np.float`, removed in numpy >= 1.24)."""
    mask, flow = _gt(batch)
    acc = _metrics(est_flow.detach().contiguous().float(), flow, mask).cpu()
    n = float(acc[1])
    return float(acc[2]) / n, float(acc[3]) / n, float(acc[4]) / n, float(acc[5]) / n
