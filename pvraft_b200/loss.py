"""Device-side loss and metrics -- mirrors of tools/loss.py:4-40 and tools/metric.py:6-79 with the same signatures
(`batch["ground_truth"] = [mask [B,N,1], flow [B,N,3]]`), one kernel pass per prediction and no host synchronisation
inside a training step (the reference indexes `error[mask > 0]`, a host-synchronising boolean gather, per prediction).
`tools/loss.py` and `tools/metric.py` of this repository re-export them under the reference's import paths."""
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


def self_supervised_loss(est_flow, batch, k=9, w_chamfer=1.0, w_smooth=1.0, w_laplacian=0.0, k_lap=10, k_int=5):
    """Self-supervised analogue of compute_loss for one flow [B,N,3] (what RSF_refine returns): mean over the batch of
    w_chamfer * Chamfer(P1 + flow, P2) + w_smooth * smoothness of the flow over P1's k-nearest-neighbour graph
    + w_laplacian * Laplacian regularity (LaplacianFn: P1's and P2's k_lap-nearest-neighbour graphs, P2's Laplacian
    interpolated from k_int points).  w_laplacian = 0 builds and launches nothing for the third term."""
    return _self_supervised(est_flow.float().unsqueeze(0), batch, k, w_chamfer, w_smooth, w_laplacian, k_lap, k_int)[0]


def sequence_self_supervised_loss(est_flow, batch, gamma=0.8, k=9, w_chamfer=1.0, w_smooth=1.0, w_laplacian=0.0, k_lap=10, k_int=5):
    """Self-supervised analogue of sequence_loss: sum_i gamma^(n-i-1) * self_supervised_loss(est_flow[i], batch), with all n
    predictions in one forward and one backward launch per term."""
    flows = torch.stack([f.float() for f in est_flow])
    n = flows.shape[0]
    per = _self_supervised(flows, batch, k, w_chamfer, w_smooth, w_laplacian, k_lap, k_int)
    weights = torch.pow(float(gamma), torch.arange(n - 1, -1, -1, dtype=torch.float32, device=per.device))
    return (weights * per).sum()


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
