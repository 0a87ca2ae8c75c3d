"""kNN graph of a point cloud -- mirror of the reference `Graph` (model/flot/graph.py:4-89).

`Graph.construct_graph(pcloud, nb_neighbors)` keeps the reference's signature and attributes
(`edges` = flat GLOBAL neighbour ids b*N + j as int64, `edge_feats` = neighbour - centre,
`k_neighbors`, `size`) but is built by the brute-force kNN kernel (pvraft_knn_fwd) instead of a
full N x N argsort; the kernels consume the compact int32 LOCAL adjacency `nbr` [B,N,k].
"""
import torch

from . import ops


class EdgeFeatsFn(torch.autograd.Function):
    """(xyz [B,N,3], nbr [B,N,k] int32, rel [B,N,k,3]) -> rel = xyz[nbr] - xyz, differentiable w.r.t. xyz
    (model/flot/graph.py:72; the adjacency carries no gradient).  The forward returns `rel` as given -- the kNN kernel writes
    it with the adjacency -- and the backward is pvraft_edge_bwd with C = 3: d xyz[nbr] += d rel, d xyz -= sum_j d rel."""

    @staticmethod
    def forward(ctx, xyz, nbr, rel):
        ctx.save_for_backward(nbr)
        ctx.shape = xyz.shape
        return rel

    @staticmethod
    def backward(ctx, d_rel):
        nbr, = ctx.saved_tensors
        b, n, k = nbr.shape
        dp = torch.zeros(ctx.shape, dtype=torch.float32, device=d_rel.device)
        ops.edge_bwd(d_rel.reshape(b, n * k, 3).contiguous(), nbr, dp)
        return dp, None, None


def edge_feats(xyz, nbr, rel):
    """Edge features of the adjacency nbr that gradients reach xyz through; rel: their values, xyz[nbr] - xyz."""
    return EdgeFeatsFn.apply(xyz, nbr, rel)


class Graph:
    def __init__(self, nbr, edge_feats, k_neighbors, size, order=None, plan=None):
        self.nbr = nbr                    # int32 [B,N,k] local ids
        self._rel = edge_feats            # f32 [B,N,k,3]
        self.order = order                # int32 [B,N] or None: processing order of the SetConv edge kernel (a Morton rank table)
        self.k_neighbors = k_neighbors
        self.size = tuple(size)
        self._edges = None
        self._plan = plan

    @property
    def plan(self):
        """The SetConv edge kernel's gather plan of (nbr, order) (ops.edge_plan), built on first use: every SetConv on this
        graph, whatever its channel count, runs from it."""
        if self._plan is None:
            self._plan = ops.edge_plan(self.nbr, self.order)
        return self._plan

    @property
    def edges(self):
        """Flat int64 global row ids, as model/flot/graph.py:77-79 builds them."""
        if self._edges is None:
            b, n, k = self.nbr.shape
            offs = (torch.arange(b, device=self.nbr.device, dtype=torch.int64) * n).view(b, 1, 1)
            self._edges = (self.nbr.long() + offs).reshape(-1)
        return self._edges

    @property
    def edge_feats(self):
        """[B*N*k, 3] neighbour - centre (model/flot/graph.py:69-74)."""
        return self._rel.reshape(-1, 3)

    @staticmethod
    def construct_graph(pcloud, nb_neighbors):
        b, n, _ = pcloud.shape
        if nb_neighbors != ops.KNN:
            raise NotImplementedError('the SetConv kernels are built for 32 neighbours (the only value the '
                                      'reference uses, model/extractor.py:9)')
        if n < nb_neighbors:
            raise ValueError(f'need at least {nb_neighbors} points per cloud, got {n}')
        pc = pcloud.detach().contiguous().float()
        nbr, rel = ops.knn(pc, pc, nb_neighbors, mode=0, want_rel=True)
        if torch.is_grad_enabled() and pcloud.requires_grad:
            rel = edge_feats(pcloud.float(), nbr, rel)
        # spatially coherent processing order for the edge kernel (changes no result: the 8 warps of a CTA then gather
        # overlapping neighbourhoods, which L1 serves)
        order = ops.point_order(pc) if n >= 64 else None
        return Graph(nbr, rel, nb_neighbors, [b * n, b * n], order)
