"""Float64 restatements of the self-supervised loss terms (pvraft_b200/loss.py), shared by the loss-kernel tests and the
whole-model decision replay (grad_replay.py).  The reference has no self-supervised loss and the oracle module restates the
reference only, so these live with the tests.  Every function works on the tensors' own device; a neighbour set that is
given is held fixed (the function the kernels differentiate), one that is not is searched in float64.

    C_s = (1/N) sum_i ||W_i - P2_{ab(i)}||^2 + (1/M) sum_j ||W_{ba(j)} - P2_j||^2     W = P1 + f, sample s against P2[s % B]
    S_s = (1/(N k)) sum_i sum_{j in N_k(i)} ||f_j - f_i||
    R_s = (1/N) sum_i ||Lhat_i - L(W)_i||^2     (test_gpu_laplacian.py)
    F_s = (1/N) sum_i ||f12_i + bhat_i||^2       (test_gpu_flow_consistency.py)
"""
import torch


def chamfer64(w, p2, nn_ab=None, nn_ba=None):
    """[S] in float64.  With indices: the loss with the pairs held fixed (the function the kernels differentiate)."""
    out = []
    for s in range(w.shape[0]):
        b = p2[s % p2.shape[0]]
        if nn_ab is None:
            d = ((w[s][:, None, :] - b[None, :, :]) ** 2).sum(-1)
            out.append(d.min(1).values.mean() + d.min(0).values.mean())
        else:
            out.append(((w[s] - b[nn_ab[s]]) ** 2).sum(-1).mean() + ((w[s][nn_ba[s]] - b) ** 2).sum(-1).mean())
    return torch.stack(out)


def smooth64(f, nbr):
    """[S] in float64; the gradient of the length at 0 is 0."""
    out = []
    for s in range(f.shape[0]):
        d = f[s][nbr[s % nbr.shape[0]]] - f[s][:, None, :]
        n2 = (d * d).sum(-1)
        pos = n2 > 0
        out.append((torch.where(pos, n2, torch.ones_like(n2)).sqrt() * pos).mean())
    return torch.stack(out)


def nn64_indices(w, p2):
    """Float64 argmin of both directions for every sample: the pairs of the float64 loss."""
    ab, ba = [], []
    for s in range(w.shape[0]):
        d = ((w[s][:, None, :] - p2[s % p2.shape[0]][None, :, :]) ** 2).sum(-1)
        ab.append(d.argmin(1))
        ba.append(d.argmin(0))
    return torch.stack(ab), torch.stack(ba)


def lap64(x, nbr):
    """L(x) [N,3] over the graph nbr [N,k]."""
    return (x[nbr] - x[:, None, :]).sum(1) / (nbr.shape[1] - 1)


def term64(w, p2, l2, g1, nn_idx):
    """[S] R_s in float64 with the interpolation neighbours nn_idx [S,N,k_int] held fixed; l2 [B,M,3] given."""
    out = []
    for s in range(w.shape[0]):
        b = s % p2.shape[0]
        idx = nn_idx[s]
        d = ((w[s][:, None, :] - p2[b][idx]) ** 2).sum(-1)
        wt = 1.0 / (d + 1e-8)
        lhat = (wt[..., None] * l2[b][idx]).sum(1) / wt.sum(1, keepdim=True)
        out.append(((lhat - lap64(w[s], g1[b])) ** 2).sum(-1).mean())
    return torch.stack(out)


def laplacian64(w, p2, g1, g2, nn_idx):
    l2 = torch.stack([lap64(p2[b], g2[b]) for b in range(p2.shape[0])])
    return term64(w, p2, l2, g1, nn_idx)


def nn64_knearest(w, p2, k):
    """Float64 k nearest of every W_i in P2[s % B] -> [S,N,k]."""
    out = []
    for s in range(w.shape[0]):
        d = ((w[s][:, None, :] - p2[s % p2.shape[0]][None, :, :]) ** 2).sum(-1)
        out.append(d.topk(k, 1, largest=False).indices)
    return torch.stack(out)


def consistency64(w, f12, p2, f21, nn_idx):
    """[S] F_s, r [S,N,3] and bhat [S,N,3] in float64 with the neighbours nn_idx [S,N,k] held fixed."""
    out, res, bh = [], [], []
    for s in range(w.shape[0]):
        b, idx = s % p2.shape[0], nn_idx[s].long()
        d = ((w[s][:, None, :] - p2[b][idx]) ** 2).sum(-1)
        wt = 1.0 / (d + 1e-8)
        bhat = (wt[..., None] * f21[s][idx]).sum(1) / wt.sum(1, keepdim=True)
        r = f12[s] + bhat
        out.append((r ** 2).sum(-1).mean())
        res.append(r)
        bh.append(bhat)
    return torch.stack(out), torch.stack(res), torch.stack(bh)


def graphs(p1, p2, k_lap):
    """The library's k_lap-nearest-neighbour graphs of both clouds (ops.knn, mode 0), int32 on the clouds' device."""
    from pvraft_b200 import ops
    p1, p2 = p1.detach().contiguous(), p2.detach().contiguous()
    return ops.knn(p1, p1, k_lap, mode=0), ops.knn(p2, p2, k_lap, mode=0)


def loss64(flows, p1, p2, nbr, g1=None, g2=None, gamma=0.8, wc=1.0, ws=1.0, wl=0.3, k_int=5, lap_idx=None,
           chamfer_idx=None):
    """sequence_self_supervised_loss in float64 for a list of [B,N,3] flows: Chamfer and smoothness over nbr, plus wl times the
    Laplacian term over P1's graph g1 and P2's g2 when they are given.  Every search runs in float64 unless chamfer_idx (one
    (nn_ab, nn_ba) per flow) or lap_idx (one [B,N,k_int] per flow) gives its neighbours."""
    n, total = len(flows), 0
    p1, p2 = p1.double(), p2.double()
    for i, f in enumerate(flows):
        f = f.double()
        w = p1 + f
        nn_ab, nn_ba = nn64_indices(w.detach(), p2.detach()) if chamfer_idx is None else chamfer_idx[i]
        per = wc * chamfer64(w, p2, nn_ab, nn_ba) + ws * smooth64(f, nbr)
        if g1 is not None:
            idx = nn64_knearest(w.detach(), p2.detach(), k_int) if lap_idx is None else lap_idx[i]
            per = per + wl * laplacian64(w, p2, g1, g2, idx)
        total = total + gamma ** (n - i - 1) * per.mean()
    return total


def pair_loss64(f12s, f21s, p1, p2, dev=None, gamma=0.8, wc=1.0, ws=1.0, wl=0.3, wcons=0.3, k=9, k_lap=10, k_int=5, k_cons=3,
                lap_idx=None, cons_idx=None, chamfer_idx=None, nbrs=None):
    """sequence_self_supervised_loss of the pair (f12s [B,N1,3] list, f21s [B,N2,3] list) in float64: the loss of each direction
    (the reverse one with P1 and P2 swapped; the Laplacian term when wl != 0) plus wcons times its consistency term, the two
    averaged.  Per direction (forward, backward): nbrs gives (smoothness graph, g1, g2), else ops.knn builds them on `dev`;
    chamfer_idx, lap_idx and cons_idx give one entry per prediction (as loss64 takes them), else the searches run in float64."""
    n, total = len(f12s), 0
    dirs = ((f12s, f21s, p1, p2), (f21s, f12s, p2, p1))
    for d, (fs, fo, pa, pb) in enumerate(dirs):
        if nbrs is None:
            pad, pbd = pa.detach().float().to(dev).contiguous(), pb.detach().float().to(dev).contiguous()
            from pvraft_b200 import ops
            nbr = ops.knn(pad, pad, k, mode=0).long().to(pa.device)
            g1, g2 = (t.long().to(pa.device) for t in graphs(pad, pbd, k_lap))
        else:
            nbr, g1, g2 = nbrs[d]
        total = total + loss64(fs, pa, pb, nbr, g1 if wl != 0 else None, g2, gamma=gamma, wc=wc, ws=ws, wl=wl, k_int=k_int,
                               lap_idx=None if lap_idx is None else lap_idx[d],
                               chamfer_idx=None if chamfer_idx is None else chamfer_idx[d]) / 2
        if wcons == 0:
            continue
        for i in range(n):
            f, r = fs[i].double(), fo[i].double()
            w = pa.double() + f
            idx = nn64_knearest(w.detach(), pb.double().detach(), k_cons) if cons_idx is None else cons_idx[d][i]
            total = total + gamma ** (n - i - 1) * wcons * consistency64(w, f, pb.double(), r, idx)[0].mean() / 2
    return total
