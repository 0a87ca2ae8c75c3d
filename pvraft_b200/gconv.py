"""SetConv -- mirror of the reference module (model/flot/gconv.py:4-85), same parameters and
state_dict keys (fc1/gn1/fc2/gn2/fc3/gn3), forward on the H100 kernels."""
import torch

from . import ops
from .ops import ACT_LRELU, IN_GN, IN_GN_MINMAX


class Deferred:
    """A SetConv output whose last GroupNorm+LeakyReLU has not been applied yet: the next consumer
    folds it into its own input staging (pvraft_linear_fwd IN_GN mode)."""

    def __init__(self, z, stats, gamma, beta, count):
        self.z, self.stats, self.gamma, self.beta, self.count = z, stats, gamma, beta, count

    def materialize(self, transpose_out=False):
        return ops.gn_act(self.z, self.stats, self.gamma, self.beta, self.count, ACT_LRELU, 0.1, transpose_out)


def _w(p):
    return p.detach()


class SetConv(torch.nn.Module):
    def __init__(self, nb_feat_in, nb_feat_out):
        super().__init__()
        # model/flot/gconv.py:21-24
        mid = nb_feat_out // 2 if nb_feat_in % 2 != 0 else (nb_feat_out + nb_feat_in) // 2
        self.nb_feat_in, self.nb_feat_out, self.mid = nb_feat_in, nb_feat_out, mid
        self.fc1 = torch.nn.Conv2d(nb_feat_in + 3, mid, 1, bias=False)
        self.gn1 = torch.nn.GroupNorm(8, mid, affine=True)
        self.fc2 = torch.nn.Conv1d(mid, nb_feat_out, 1, bias=False)
        self.gn2 = torch.nn.GroupNorm(8, nb_feat_out, affine=True)
        self.fc3 = torch.nn.Conv1d(nb_feat_out, nb_feat_out, 1, bias=False)
        self.gn3 = torch.nn.GroupNorm(8, nb_feat_out, affine=True)

    def forward_deferred(self, signal, graph, p=None):
        """signal: [B,N,cin] tensor or a Deferred from the previous SetConv -> Deferred.
        Layers whose shapes fit the tensor-core kernel (N % 128 == 0, K % 32 == 0) run on wgmma (3xTF32),
        the others on the CUDA-core kernel; both are fp32-accurate.  p: the fc1 pre-transform of a plain signal when the
        caller has already computed it (the fused update chain of the RAFT loop)."""
        cin, mid, cout = self.nb_feat_in, self.mid, self.nb_feat_out
        deferred = isinstance(signal, Deferred)
        x = signal.z if deferred else signal.detach().contiguous().float()
        b, n, _ = x.shape
        if graph.size[0] // b != n:
            raise ValueError('graph and signal disagree on the number of points')
        stats = ops.new_stats(b, x.device, 3)
        pro = dict(in_stats=signal.stats, in_gamma=signal.gamma, in_beta=signal.beta, in_count=signal.count,
                   in_act=ACT_LRELU, in_slope=0.1) if deferred else {}
        # fc1 pre-transform P = fc1.weight[:, :cin] . x   (gconv.py:65-73: fc1 is linear and bias-free)
        if p is not None:
            if deferred or p.shape != (b, n, mid):
                raise ValueError('a precomputed fc1 pre-transform needs a plain signal and shape [B,N,mid]')
        elif ops.tc_supported(n, cin) and mid <= 128:
            p = ops.tc_linear([x], ops.tc_weights(self.fc1.weight, col0=0, cols=cin), **pro)
        else:
            p = ops.linear(x, _w(self.fc1.weight), cin=cin, w_ld=cin + 3, cout=mid, in_mode=IN_GN if deferred else ops.IN_PLAIN, **pro)
        ymax, ymin = ops.setconv_edge(p, graph.nbr, graph._rel, _w(self.fc1.weight), cin, stats[0], order=graph.order,
                                      plan=graph.plan)
        gsz1, gsz = mid // 8, cout // 8
        pro1 = dict(in_min=ymin, in_stats=stats[0], in_gamma=_w(self.gn1.weight), in_beta=_w(self.gn1.bias),
                    in_count=float(n) * 32 * gsz1, in_act=ACT_LRELU, in_slope=0.1)
        if ops.tc_supported(n, mid) and cout <= 128:
            z2 = ops.tc_linear([ymax], ops.tc_weights(self.fc2.weight), out_stats=stats[1], **pro1)
        else:
            z2 = ops.linear(ymax, _w(self.fc2.weight), in_mode=IN_GN_MINMAX, out_stats=stats[1], **pro1)
        pro2 = dict(in_stats=stats[1], in_gamma=_w(self.gn2.weight), in_beta=_w(self.gn2.bias), in_count=float(n) * gsz,
                    in_act=ACT_LRELU, in_slope=0.1)
        if ops.tc_supported(n, cout) and cout <= 128:
            z3 = ops.tc_linear([z2], ops.tc_weights(self.fc3.weight), out_stats=stats[2], **pro2)
        else:
            z3 = ops.linear(z2, _w(self.fc3.weight), in_mode=IN_GN, out_stats=stats[2], **pro2)
        return Deferred(z3, stats[2], _w(self.gn3.weight), _w(self.gn3.bias), float(n) * gsz)

    def forward(self, signal, graph):
        """signal [B,N,cin], graph -> [B,N,cout]   (model/flot/gconv.py:38-85)."""
        return self.forward_deferred(signal, graph).materialize()
