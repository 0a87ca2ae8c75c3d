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
