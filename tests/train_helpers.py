"""Helpers shared by the whole-model training tests: the sequence loss, the kNN graph taken from the oracle, trained-looking
weights and the gradient comparison against autograd through the oracle."""
import contextlib

import torch

from oracle import pvraft_oracle as O


def sequence_loss(flows, gt, gamma=0.8):
    """tools/loss.py:4-13 with an all-ones mask: sum_i gamma^(n-i-1) * mean |flow_i - gt| (compute_loss, loss.py:16-40)."""
    n = len(flows)
    return sum(gamma ** (n - i - 1) * (flows[i] - gt).abs().sum(-1).mean() for i in range(n))


@contextlib.contextmanager
def oracle_adjacency():
    """kNN ties at the 32nd distance are either-valid (SURVEY H1): the model runs on the oracle's adjacency, handed in as
    `nbr`; the edge features stay differentiable w.r.t. the cloud through graph.edge_feats when the cloud requires grad."""
    from pvraft_b200 import Graph, graph as G

    def from_oracle(pcloud, k):
        b, n, _ = pcloud.shape
        og = O.construct_graph(pcloud.detach().float().cpu(), k)
        nbr = (og.edges.reshape(b, n, k) - (torch.arange(b) * n).view(b, 1, 1)).to(torch.int32).to(pcloud.device)
        rel = og.edge_feats.reshape(b, n, k, 3).to(pcloud.device).contiguous()
        if torch.is_grad_enabled() and pcloud.requires_grad:
            rel = G.edge_feats(pcloud.float(), nbr, rel)
        return Graph(nbr, rel, k, [b * n, b * n])

    orig = G.Graph.__dict__['construct_graph']
    G.Graph.construct_graph = staticmethod(from_oracle)
    try:
        yield
    finally:
        G.Graph.construct_graph = orig


def randomise_affine(model, seed, slopes):
    """GroupNorm affines drawn at random (some negative scales), as tests/golden/make_golden.py does, and the two PReLU slopes
    of the correlation block (out_conv.2, knn_conv.2) set to `slopes`."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if '.gn' in name or 'out_conv.1.' in name or 'knn_conv.1.' in name:
                if name.endswith('weight'):
                    p.copy_(torch.randn(p.shape, generator=g) * 0.5 + 0.8)
                else:
                    p.copy_(torch.randn(p.shape, generator=g) * 0.2)
        model.corr_block.out_conv[2].weight.fill_(slopes[0])
        model.corr_block.knn_conv[2].weight.fill_(slopes[1])


def compare_grads(got, want, tol_l2, tol_max):
    """Per tensor: relative L2 error < tol_l2 and max-abs / max-abs < tol_max; cosine of the whole gradient > 0.99999.
    Returns (worst relative L2, worst max-abs ratio, cosine)."""
    worst_l2, worst_max, dot, na, nb = ('', 0.0), ('', 0.0), 0.0, 0.0, 0.0
    for k, w in want.items():
        a, w = got[k].double().cpu(), w.double()
        assert a.shape == w.shape, k
        e2 = float((a - w).norm() / w.norm().clamp_min(1e-30))
        em = float((a - w).abs().max() / w.abs().max().clamp_min(1e-30))
        worst_l2 = (k, e2) if e2 > worst_l2[1] else worst_l2
        worst_max = (k, em) if em > worst_max[1] else worst_max
        dot += float((a * w).sum()); na += float((a * a).sum()); nb += float((w * w).sum())
    cos = dot / (na * nb) ** 0.5
    print(f'gradient parity over {len(want)} tensors: worst relative L2 {worst_l2[0]} {worst_l2[1]:.2e}, worst max-abs/max-abs '
          f'{worst_max[0]} {worst_max[1]:.2e}, cosine of the full gradient {cos:.8f}')
    assert worst_l2[1] < tol_l2, worst_l2
    assert worst_max[1] < tol_max, worst_max
    assert cos > 0.99999, cos
    return worst_l2[1], worst_max[1], cos
