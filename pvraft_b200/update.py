"""UpdateBlock = MotionEncoder + ConvGRU + FlowHead -- mirrors of model/update.py:8-87 with the same
parameters / state_dict keys; forward passes run on the H100 kernels.

Layouts: the module-level `forward` methods take and return the reference's channel-major [B,C,N]
tensors (drop-in seam); the `*_pm` methods work on point-major [B,N,C] buffers and are what the
RAFT loop uses (no transposes inside the loop).
"""
import torch
import torch.nn as nn

from . import ops
from .gconv import SetConv


def _w(p):
    return p.detach()


def fold_flow_head(w_o0, w_c1, b_c1, b_o0):
    """out_conv.0([s, conv1(x)]) = [W_a | W_b W_c1] [s, x] + (W_b b_c1 + b_o0) with out_conv.0.weight = [W_a | W_b]
    (model/update.py:68-71): the folded [64,128] weight and [64] bias, products in float64 rounded once to fp32."""
    wo = w_o0.detach().reshape(64, 128).double()
    wc, bc = w_c1.detach().reshape(64, 64).double(), b_c1.detach().double()
    w = torch.cat([wo[:, :64], wo[:, 64:] @ wc], 1).float().contiguous()
    return w, (wo[:, 64:] @ bc + b_o0.detach().double()).float().contiguous()


class MotionEncoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv_corr = nn.Conv1d(64, 64, 1)
        self.conv_flow = nn.Conv1d(3, 64, 1)
        self.conv = nn.Conv1d(64 + 64, 64 - 3, 1)

    def fill(self, a, flow, motion=None):
        """Attach the motion stage to a CorrFeatArgs (pvraft_corr_feature_fwd), with its output `motion` when given."""
        ops.pack.CorrFeatArgs(a, flow=flow, w_cc=_w(self.conv_corr.weight), b_cc=_w(self.conv_corr.bias),
                              w_cf=_w(self.conv_flow.weight), b_cf=_w(self.conv_flow.bias), w_cm=_w(self.conv.weight),
                              b_cm=_w(self.conv.bias), motion=motion)

    def forward_pm(self, flow, corr_pm):
        b, n, _ = flow.shape
        motion = torch.empty(b, n, 64, dtype=torch.float32, device=flow.device)
        a = ops.pack.CorrFeatArgs(corr_in=corr_pm, B=b, N=n)
        self.fill(a, flow, motion)
        ops.corr_feature(a)
        return motion

    def forward(self, flow, corr):
        """model/update.py:15-21: flow [B,N,3], corr [B,64,N] -> [B,64,N]."""
        return ops.transpose(self.forward_pm(flow.detach().contiguous().float(), ops.transpose(corr.detach().contiguous().float())))


class ConvGRU(nn.Module):
    def __init__(self, input_dim=128, hidden_dim=64):
        super().__init__()
        if input_dim != 128 or hidden_dim != 64:
            raise NotImplementedError('the GRU kernel is built for the reference sizes (input 128, hidden 64)')
        self.convz = nn.Conv1d(input_dim + hidden_dim, hidden_dim, 1)
        self.convr = nn.Conv1d(input_dim + hidden_dim, hidden_dim, 1)
        self.convq = nn.Conv1d(input_dim + hidden_dim, hidden_dim, 1)

    def forward_pm(self, net, inp, motion, out=None):
        b, n, _ = net.shape
        if out is None:
            out = torch.empty_like(net)
        if ops.tc_supported(n):
            # wgmma: [z|r] = sigmoid(W_zr [h,x]); q = tanh(W_q [r*h, x]); h' = (1-z) h + z q   (update.py:32-39)
            z, rh = torch.empty_like(net), torch.empty_like(net)
            ops.tc_linear([net, inp, motion], ops.tc_weights((self.convz.weight, self.convr.weight)), _w(self.convz.bias),
                          bias2=_w(self.convr.bias), epilogue=ops.TC_GRU_ZR, out=z, out2=rh, h=net, cout=64)
            ops.tc_linear([rh, inp, motion], ops.tc_weights(self.convq.weight), _w(self.convq.bias), epilogue=ops.TC_GRU_Q,
                          out=out, h=net, z=z, cout=64)
            return out
        ops.gru(ops.pack.GruArgs(net=net, inp=inp, motion=motion, w_z=_w(self.convz.weight), b_z=_w(self.convz.bias),
                                 w_r=_w(self.convr.weight), b_r=_w(self.convr.bias), w_q=_w(self.convq.weight),
                                 b_q=_w(self.convq.bias), net_out=out, B=b, N=n))
        return out

    def forward(self, h, x):
        """model/update.py:31-40: h [B,64,N], x [B,128,N] -> [B,64,N]."""
        xt = ops.transpose(x.detach().contiguous().float())
        inp, motion = xt[..., :64].contiguous(), xt[..., 64:].contiguous()
        return ops.transpose(self.forward_pm(ops.transpose(h.detach().contiguous().float()), inp, motion))


class ConvRNN(nn.Module):
    """Defined but never instantiated by the reference (model/update.py:43-54); kept so that
    `from model.update import ConvRNN` keeps working.  Plain PyTorch, not on the hot path."""

    def __init__(self, input_dim=128, hidden_dim=64):
        super().__init__()
        self.convx = nn.Conv1d(input_dim, hidden_dim, 1)
        self.convh = nn.Conv1d(hidden_dim, hidden_dim, 1)

    def forward(self, h, x):
        return torch.tanh(self.convx(x) + self.convh(h))


class FlowHead(nn.Module):
    def __init__(self, input_dim=128):
        super().__init__()
        if input_dim != 64:
            raise NotImplementedError('the flow-head kernels are built for hidden_dim = 64 (model/update.py:80)')
        self.conv1 = nn.Conv1d(input_dim, 64, 1)
        self.setconv = SetConv(64, 64)
        self.out_conv = nn.Sequential(
            nn.Conv1d(128, 64, 1),
            nn.ReLU(),
            nn.Conv1d(64, 3, 1),
        )

    def forward_pm(self, net, graph, coords1=None, coords2=None, coords2_out=None, flow_out=None, p=None):
        """net [B,N,64] -> delta_flow [B,N,3]; optionally also the RAFT coordinate update.  p: the SetConv's fc1
        pre-transform of net when it was computed with net (UpdateBlock.forward_chain_pm)."""
        b, n, _ = net.shape
        d = self.setconv.forward_deferred(net, graph, p=p)
        delta = torch.empty(b, n, 3, dtype=torch.float32, device=net.device)
        oc = self.out_conv
        if ops.tc_supported(n):
            # wgmma, one launch: out_conv.0 on [setconv(x), conv1(x)] (update.py:68-71) is linear in x through conv1, so
            # conv1 is folded into the second half of its weight: W [a3 | W_b W_c1] with bias W_b b_c1 + b_o0 (products in
            # float64, rounded once).  Prologue: a3 = lrelu(GN3(z3)); epilogue: ReLU, out_conv.2 and the RAFT update
            # (update.py:72, RAFTSceneFlow.py:45-46).
            w_eff, b_eff = ops.derived((oc[0].weight, self.conv1.weight, self.conv1.bias, oc[0].bias), 'flowhead', fold_flow_head)
            ops.tc_linear([d.z, net], ops.tc_weights(w_eff), b_eff, in_stats=d.stats, in_gamma=d.gamma, in_beta=d.beta,
                          in_count=d.count, in_act=ops.ACT_LRELU, in_slope=0.1, epilogue=ops.TC_FLOW, out=delta, cout=64,
                          w3=_w(oc[2].weight), b3=_w(oc[2].bias), coords1=coords1, coords2=coords2, coords2_out=coords2_out,
                          flow_out=flow_out)
            return delta
        ops.flow_out(ops.pack.FlowOutArgs(z3=d.z, z3_stats=d.stats, gn3_gamma=d.gamma, gn3_beta=d.beta, net=net,
                                          w_c1=_w(self.conv1.weight), b_c1=_w(self.conv1.bias), w_o0=_w(oc[0].weight),
                                          b_o0=_w(oc[0].bias), w_o2=_w(oc[2].weight), b_o2=_w(oc[2].bias), coords1=coords1,
                                          coords2=coords2, delta=delta, coords2_out=coords2_out, flow_out=flow_out, B=b, N=n))
        return delta

    def forward(self, x, graph):
        """model/update.py:68-72: x [B,64,N] -> [B,3,N]."""
        return ops.transpose(self.forward_pm(ops.transpose(x.detach().contiguous().float()), graph))


class UpdateBlock(nn.Module):
    def __init__(self, input_dim=128, hidden_dim=64):
        super().__init__()
        self.motion_encoder = MotionEncoder()
        self.gru = ConvGRU(input_dim=input_dim, hidden_dim=hidden_dim)
        self.flow_head = FlowHead(input_dim=hidden_dim)

    def forward_pm(self, net, inp, motion, graph, **coords):
        net = self.gru.forward_pm(net, inp, motion)
        delta = self.flow_head.forward_pm(net, graph, **coords)
        return net, delta

    def forward_chain_pm(self, net, inp, y1, kfeat, cflow, flow, gn, corr_motion, graph, **coords):
        """One RAFT update from the correlation block's pre-activations (CorrBlock.motion_inputs_tc) with the motion
        encoder, the ConvGRU and the flow head's fc1 pre-transform in one launch (ops.update_chain); the same values as
        CorrBlock.feature_motion_tc followed by forward_pm.  corr_motion: CorrBlock.corr_motion_weights().  Needs
        ops.tc_supported(N)."""
        me, gru, sc = self.motion_encoder, self.gru, self.flow_head.setconv
        w_eff, b_eff = corr_motion
        weights = (ops.tc_weights(w_eff), ops.tc_weights(me.conv.weight), ops.tc_weights((gru.convz.weight, gru.convr.weight)),
                   ops.tc_weights(gru.convq.weight), ops.tc_weights(sc.fc1.weight, col0=0, cols=sc.nb_feat_in))
        biases = (b_eff, _w(me.conv.bias), _w(gru.convz.bias), _w(gru.convr.bias), _w(gru.convq.bias))
        net, p = ops.update_chain(y1, gn, kfeat, cflow, flow, net, inp, weights, biases)
        delta = self.flow_head.forward_pm(net, graph, p=p, **coords)
        return net, delta

    def forward(self, net, inp, corr, flow, graph):
        """model/update.py:82-87: net, inp, corr [B,64,N], flow [B,N,3] -> (net [B,64,N], delta_flow [B,N,3])."""
        flow = flow.detach().contiguous().float()
        motion = self.motion_encoder.forward_pm(flow, ops.transpose(corr.detach().contiguous().float()))
        net_pm, delta = self.forward_pm(ops.transpose(net.detach().contiguous().float()),
                                        ops.transpose(inp.detach().contiguous().float()), motion, graph)
        return ops.transpose(net_pm), delta
