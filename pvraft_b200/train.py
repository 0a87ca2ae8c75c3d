"""Training path: the gradient contract of SURVEY.md section 8b.

`RSF.forward` / `RSF_refine.forward` take this path whenever autograd is recording and a parameter requires grad
(tools/engine.py:131-147 calls `loss.backward()` on the returned flows; tools/engine_refine.py trains `refine_block` only).
The forward runs layer by layer -- the fused inference kernels keep no activations -- and every layer is a
`torch.autograd.Function` whose forward AND backward are kernels of libpvraft_b200.so:

    LinearFn        1x1 convolution           pvraft_linear_fwd (y, and dx = dy.W through the transposed weight) + pvraft_linear_wgrad
                                              ('bf16-mixed' loop layers: pvraft_tc_linear_fwd on bf16 + pvraft_tc_wgrad_bf16)
    GnActFn         GroupNorm(8) + act        pvraft_gn_act_fwd / pvraft_gn_act_bwd
    GnActMaxFn      ... + max over 32 rows    pvraft_gn_act_maxk_fwd / pvraft_gn_act_bwd (arg form: no dense max gradient)
    EdgeFn          SetConv edge stage        pvraft_edge_fwd / pvraft_edge_bwd          (model/flot/gconv.py:65-73)
    MaxKFn          max over 32 neighbours    pvraft_maxk_fwd / pvraft_maxk_bwd          (gconv.py:80, model/corr.py:92)
    CorrInitFn      truncated correlation     wgmma GEMM + top-k + reorder / pvraft_corr_init_bwd (sparse)   (corr.py:31-42,95-100)
    CorrLookupFn    voxel means + kNN gather  pvraft_corr_lookup_fwd / pvraft_corr_lookup_bwd (+ pvraft_corr_lookup_xyz_bwd)  (corr.py:47-66,75-91)
    EdgeFeatsFn     graph edge features       the kNN kernel's output / pvraft_edge_bwd with C = 3            (graph.py:72; in graph.py)

PyTorch is the tape (which Function follows which) and the allocator; the glue between Functions that the reference also
writes as single ATen calls (cat / split / relu / sigmoid / tanh / add / mul on [B,N,64..192] tensors: model/update.py:18-20,
32-39, model/corr.py:45) stays ATen.  The input clouds stay attached, so gradients reach them as in the reference: through
the flows (coords2 - xyz1), the encoders' first SetConv (the cloud is its signal), the graphs' edge features and, for xyz2,
the kNN 4-vectors of every lookup.  `coords2` carries none: the reference detaches it every iteration
(model/RAFTSceneFlow.py:41) and derives every index under no_grad (model/corr.py:52-62).
All tensors are point-major [B,rows,C] (rows = N per-point, N*32 per-edge).
"""
import os

import torch

from . import ops
from .graph import Graph
from .ops import ACT_LRELU


def _zeros64(*shape, device):
    return torch.zeros(*shape, dtype=torch.float64, device=device)


# Per-point layers of the training path on the wgmma kernel: 'auto' = while the step is being captured into a CUDA graph
# (26.9 vs 30.0 ms per step); with eager launches the host cost of the tensor-core launch path (tensor-map encodes, the weight
# splits after every optimizer step) outweighs the faster kernels (40.5 vs 33.0 ms), so there the CUDA-core kernels stay.
_TC_TRAIN = os.environ.get('PVRAFT_TC_TRAIN', 'auto')


def _tc_train():
    return _TC_TRAIN == '1' or (_TC_TRAIN == 'auto' and torch.cuda.is_current_stream_capturing())


def bf16_layer_plan(n_points, cin, cout, want_stats=False):
    """Kernels of a per-point layer [B, n_points, cin] -> cout: (forward, dx, dW), each True where its shape suits the
    tensor-core kernel -- bf16 wgmma inside the RAFT loop of a 'bf16-mixed' training step, 3xTF32 for forward and dx in a
    captured fp32 step (no dW kernel there) -- and False where it keeps its fp32 CUDA-core kernel.  The forward follows
    the shape rule of the tensor-core path (N % 128 == 0, cin % 32 == 0, cout <= 128; GroupNorm sums need cout % 32 == 0);
    dx also needs cout % 32 == 0 (the transposed weight's K), dW cout % 32 == 0 and cin <= 192 (pvraft_tc_wgrad_bf16)."""
    fwd = ops.tc_supported(n_points, cin) and cout <= 128 and (not want_stats or cout % 32 == 0)
    return fwd, fwd and cout % 32 == 0, fwd and cout % 32 == 0 and cin <= 192


class LinearFn(torch.autograd.Function):
    """y[B,R,cout] = x[B,R,cin] . W^T (+ b); optionally also the GroupNorm sums [B,8,2] of y (not differentiable: the
    consumer GnActFn differentiates through the statistics itself)."""

    @staticmethod
    def forward(ctx, x, w, b, want_stats):
        w2 = w.reshape(w.shape[0], -1).contiguous()
        x = x.contiguous()
        stats = _zeros64(x.shape[0], 8, 2, device=x.device) if want_stats else None
        cout, cin = w2.shape
        # per-point layers whose shapes fit go to the wgmma kernel (3xTF32: fp32-accurate), forward and dx; the weight is
        # split once per parameter version, i.e. once per optimizer step however many iterations use the layer.
        # Inside the RAFT loop of 'bf16-mixed' (an ops.bf16_compute scope) they go there in eager steps too, on bf16
        # operands, and so does their weight gradient.  The backward runs on autograd's device thread, which does not see
        # the scope: the format is recorded here.
        fwd_tc, ctx.dx_tc, ctx.dw_tc = bf16_layer_plan(x.shape[1], cin, cout, want_stats) if x.dim() == 3 else (False,) * 3
        ctx.bf16 = fwd_tc and ops.bf16_compute_active()
        ctx.tc = ctx.bf16 or (_tc_train() and fwd_tc)
        ctx.w_ref = w
        if ctx.tc:
            y = ops.tc_linear([x], ops.tc_weights(w, bf16=ctx.bf16), None if b is None else b.detach(), out_stats=stats)
        else:
            y = ops.linear(x, w2, b, out_stats=stats)
        ctx.save_for_backward(x, w2)
        ctx.has_bias, ctx.w_shape = b is not None, w.shape
        if want_stats:
            ctx.mark_non_differentiable(stats)
            return y, stats
        return y

    @staticmethod
    def backward(ctx, dy, *unused):
        x, w2 = ctx.saved_tensors
        dy = dy.contiguous()
        dx = None
        if w2.shape[1] <= 4 and w2.shape[0] in (16, 32, 48, 64, 96, 128):
            # the edge-level layers (rows = B*N*32, three or four input columns): one pass over dy for all three gradients
            dw = torch.zeros_like(w2)
            db = torch.zeros(w2.shape[0], dtype=torch.float32, device=w2.device) if ctx.has_bias else None
            dx = ops.linear_bwd_small(x, dy, w2, dw, db, want_dx=ctx.needs_input_grad[0])
            return dx, dw.reshape(ctx.w_shape), db, None
        if ctx.needs_input_grad[0]:
            # dx = dy . W: the same kernel with the transposed weight, 128 output columns (the kernel's limit) at a time
            cout, cin = w2.shape
            if ctx.tc and ctx.dx_tc:
                parts = [ops.tc_linear([dy], ops.tc_weights(ctx.w_ref, transposed=(c0, min(c0 + 128, cin)), bf16=ctx.bf16))
                         for c0 in range(0, cin, 128)]
            else:
                parts = [ops.linear(dy, w2[:, c0:min(c0 + 128, cin)].t().contiguous()) for c0 in range(0, cin, 128)]
            dx = parts[0] if len(parts) == 1 else torch.cat(parts, -1)
        dw = db = None
        if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
            dw = torch.zeros_like(w2)
            db = torch.zeros(w2.shape[0], dtype=torch.float32, device=w2.device) if ctx.has_bias else None
            if ctx.bf16 and ctx.dw_tc:
                ops.tc_wgrad_bf16(x, dy, dw, db)
            else:
                ops.linear_wgrad(x, dy, dw, db)
            dw = dw.reshape(ctx.w_shape)
        return dx, dw, db, None


def linear(x, w, b=None, stats=False):
    return LinearFn.apply(x, w, b, stats)


class GnActFn(torch.autograd.Function):
    """act(GroupNorm8(x)) over [B,rows,C] with the producer's raw sums `stats` [B,8,2]; `slope_param` is the PReLU weight
    (one element, learnable) or None for the fixed LeakyReLU(0.1) / no activation."""

    @staticmethod
    def forward(ctx, x, stats, gamma, beta, slope_param, act, slope):
        b, rows, c = x.shape
        count = float(rows) * (c // 8)
        x = x.contiguous()
        sdev = None if slope_param is None else slope_param.detach().reshape(-1).contiguous()   # read on the device: no host sync
        y = ops.gn_act(x, stats, gamma.detach(), beta.detach(), count, act, slope, slope_dev=sdev)
        ctx.save_for_backward(x, stats, gamma.detach(), beta.detach(), *(() if sdev is None else (sdev,)))
        ctx.cfg = (count, act, float(slope), slope_param is not None, None if slope_param is None else slope_param.shape)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, stats, gamma, beta = ctx.saved_tensors[:4]
        count, act, slope, has_slope, slope_shape = ctx.cfg
        sdev = ctx.saved_tensors[4] if has_slope else None
        dx, dgamma, dbeta, dslope = ops.gn_act_bwd(x, dy.contiguous(), stats, gamma, beta, count, act, slope, has_slope, slope_dev=sdev)
        return dx, None, dgamma, dbeta, (dslope.reshape(slope_shape) if has_slope else None), None, None


def gn_act(x, stats, gn, act=ACT_LRELU, slope=0.1, prelu=None):
    """prelu: an nn.PReLU whose one-element weight is the slope -- handed to the kernels as a device pointer (the optimizer
    changes it every step; a host read-back would synchronise the stream twice per RAFT iteration)."""
    return GnActFn.apply(x, stats, gn.weight, gn.bias, None if prelu is None else prelu.weight, act, slope)


class GnActMaxFn(torch.autograd.Function):
    """max over each point's 32 consecutive rows of act(GroupNorm8(x)): [B,N*32,C] -> [B,N,C] (gconv.py:76-80, corr.py:87-92).
    One forward pass over x; in the backward the dense gradient of the max (31/32 zeros) is never materialised: the GroupNorm
    backward reads d(max) [B,N,C] and the arg-max directly."""

    @staticmethod
    def forward(ctx, x, stats, gamma, beta, slope_param, act, slope):
        b, rows, c = x.shape
        count = float(rows) * (c // 8)
        x = x.contiguous()
        sdev = None if slope_param is None else slope_param.detach().reshape(-1).contiguous()
        y, arg = ops.gn_act_maxk(x, stats, gamma.detach(), beta.detach(), count, act, slope, slope_dev=sdev)
        ctx.save_for_backward(x, stats, gamma.detach(), beta.detach(), arg, *(() if sdev is None else (sdev,)))
        ctx.cfg = (count, act, float(slope), slope_param is not None, None if slope_param is None else slope_param.shape)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, stats, gamma, beta, arg = ctx.saved_tensors[:5]
        count, act, slope, has_slope, slope_shape = ctx.cfg
        sdev = ctx.saved_tensors[5] if has_slope else None
        dx, dgamma, dbeta, dslope = ops.gn_act_bwd(x, dy.contiguous(), stats, gamma, beta, count, act, slope, has_slope, slope_dev=sdev,
                                                   arg=arg)
        return dx, None, dgamma, dbeta, (dslope.reshape(slope_shape) if has_slope else None), None, None


def gn_act_max(x, stats, gn, act=ACT_LRELU, slope=0.1, prelu=None):
    return GnActMaxFn.apply(x, stats, gn.weight, gn.bias, None if prelu is None else prelu.weight, act, slope)


class EdgeFn(torch.autograd.Function):
    """T[b,n,j,:] = P[b,nbr[b,n,j],:] - P[b,n,:] + E[b,n,j,:], written over E; also the GroupNorm sums of T."""

    @staticmethod
    def forward(ctx, p, e, nbr):
        stats = _zeros64(p.shape[0], 8, 2, device=p.device)
        ops.edge_fwd(p.contiguous(), nbr, e, stats)
        ctx.mark_dirty(e)
        ctx.mark_non_differentiable(stats)
        ctx.save_for_backward(nbr)
        ctx.p_shape = p.shape
        return e, stats

    @staticmethod
    def backward(ctx, dt, _):
        nbr, = ctx.saved_tensors
        dt = dt.contiguous()
        dp = torch.zeros(ctx.p_shape, dtype=torch.float32, device=dt.device)
        ops.edge_bwd(dt, nbr, dp)
        return dp, dt, None


class MaxKFn(torch.autograd.Function):
    """[B,N*32,C] -> [B,N,C]: max over each point's 32 consecutive edge rows."""

    @staticmethod
    def forward(ctx, x):
        b, rows, c = x.shape
        y, arg = ops.maxk_fwd(x.contiguous(), b * (rows // 32), c)
        ctx.save_for_backward(arg)
        ctx.shape = (b, rows, c)
        return y.view(b, rows // 32, c)

    @staticmethod
    def backward(ctx, dy):
        arg, = ctx.saved_tensors
        b, rows, c = ctx.shape
        return ops.maxk_bwd(dy.contiguous(), arg, b * (rows // 32), c).view(b, rows, c)


class CorrInitFn(torch.autograd.Function):
    """(fmap1 [B,N1,C], fmap2 [B,N2,C]) -> the K largest correlations of every row of fmap1, in the lookup kernel's stored
    order, with their column ids (rows of fmap2; not differentiable).  Backward is sparse: only the kept entries carry
    gradient (model/corr.py:37-40)."""

    @staticmethod
    def forward(ctx, fmap1, fmap2, k, corr_block):
        fmap1, fmap2 = fmap1.contiguous(), fmap2.contiguous()
        val, idx = ops.corr_build(fmap1, fmap2, k)
        val, idx = ops.corr_reorder(val, idx)
        ctx.save_for_backward(fmap1, fmap2, idx)
        ctx.mark_non_differentiable(idx)
        return val, idx

    @staticmethod
    def backward(ctx, g, _):
        fmap1, fmap2, idx = ctx.saved_tensors
        d1, d2 = ops.corr_init_bwd(g.contiguous(), idx, fmap1, fmap2)
        return d1, d2, None, None


class CorrLookupFn(torch.autograd.Function):
    """corr_val [B,N1,K] (+ ids, gather table [B,N2,4], query coordinates [B,N1,3]) -> voxel means [B,N1,levels*27],
    kNN 4-vectors [B,N1*32,4].  xyz2 [B,N2,3], the cloud the gather table was padded from (ops.xyz_pad), receives the
    gradient of the kNN 4-vectors' coordinate channels when it requires grad (model/corr.py:88-89)."""

    @staticmethod
    def forward(ctx, corr_val, corr_idx, xyz2p, coords, levels, base_scale, xyz2=None):
        coords = coords.contiguous()
        out = ops.corr_lookup(corr_val, corr_idx, xyz2p, coords, levels, base_scale, want_slots=True, vox_ld=levels * 27)
        ctx.save_for_backward(corr_idx, xyz2p, coords, out['knn_slot'])
        ctx.cfg = (levels, base_scale)
        b, n, _ = coords.shape
        return out['vox'], out['knn_sel'].view(b, n * 32, 4)

    @staticmethod
    def backward(ctx, g_vox, g_sel):
        corr_idx, xyz2p, coords, slots = ctx.saved_tensors
        levels, base_scale = ctx.cfg
        g_sel = g_sel.contiguous()
        d_corr = ops.corr_lookup_bwd(corr_idx, xyz2p, coords, slots, g_vox.contiguous(), g_sel, levels, base_scale)
        d_xyz2 = None
        if len(ctx.needs_input_grad) > 6 and ctx.needs_input_grad[6]:      # xyz2 given, and it requires grad
            b, m, _ = xyz2p.shape
            d_xyz2 = ops.corr_lookup_xyz_bwd(corr_idx, slots, g_sel, torch.zeros(b, m, 3, dtype=torch.float32, device=g_sel.device))
        return d_corr, None, None, None, None, None, d_xyz2


# ----------------------------------------------------------------------------------------------------------------------
# modules, layer by layer
# ----------------------------------------------------------------------------------------------------------------------
def set_conv(m, x, graph):
    """SetConv.forward (model/flot/gconv.py:58-85) on x [B,N,cin] -> [B,N,cout]; fc1 is linear and bias-free, so
    fc1([x_j - x_i, e]) = P_j - P_i + W_e e with P = W_x x (changes rounding only, SURVEY 8a row a8)."""
    b, n, cin = x.shape
    w = m.fc1.weight.reshape(m.mid, cin + 3)
    p = linear(x, w[:, :cin])
    e = linear(graph._rel.reshape(b, n * 32, 3), w[:, cin:])
    t, st = EdgeFn.apply(p, e, graph.nbr)
    z2, st2 = linear(gn_act_max(t, st, m.gn1), m.fc2.weight, None, True)
    z3, st3 = linear(gn_act(z2, st2, m.gn2), m.fc3.weight, None, True)
    return gn_act(z3, st3, m.gn3)


def flot_encoder(m, pc, graph):
    """FlotEncoder.forward (model/extractor.py:17-24) -> [B,N,128] point-major."""
    x = set_conv(m.feat_conv1, pc, graph)
    x = set_conv(m.feat_conv2, x, graph)
    return set_conv(m.feat_conv3, x, graph)


def corr_features(cb, vox, sel):
    """out_conv on the voxel means + knn_conv / max / knn_out on the kNN 4-vectors, summed (model/corr.py:71-73,86-93,45)."""
    oc, kc = cb.out_conv, cb.knn_conv
    y1, st1 = linear(vox, oc[0].weight, oc[0].bias, True)
    vfeat = linear(gn_act(y1, st1, oc[1], prelu=oc[2]), oc[3].weight, oc[3].bias)
    k1, stk = linear(sel, kc[0].weight, kc[0].bias, True)
    kfeat = linear(gn_act_max(k1, stk, kc[1], prelu=kc[2]), cb.knn_out.weight, cb.knn_out.bias)
    return vfeat + kfeat


def update_block(ub, net, inp, corr, flow, graph):
    """UpdateBlock.forward (model/update.py:82-87), point-major: -> (net [B,N,64], delta_flow [B,N,3])."""
    me, gru, fh = ub.motion_encoder, ub.gru, ub.flow_head
    cor = torch.relu(linear(corr, me.conv_corr.weight, me.conv_corr.bias))                         # update.py:16
    flo = torch.relu(linear(flow, me.conv_flow.weight, me.conv_flow.bias))                         # :17
    out = torch.relu(linear(torch.cat([cor, flo], -1), me.conv.weight, me.conv.bias))              # :18-19
    motion = torch.cat([out, flow], -1)                                                            # :20
    hx = torch.cat([net, inp, motion], -1)                                                         # :32, :84
    w_zr = torch.cat([gru.convz.weight, gru.convr.weight], 0)
    b_zr = torch.cat([gru.convz.bias, gru.convr.bias], 0)
    zr = torch.sigmoid(linear(hx, w_zr, b_zr))                                                     # :34-35
    z, r = zr[..., :64], zr[..., 64:]
    q = torch.tanh(linear(torch.cat([r * net, inp, motion], -1), gru.convq.weight, gru.convq.bias))   # :36
    net = (1 - z) * net + z * q                                                                    # :38
    a = linear(net, fh.conv1.weight, fh.conv1.bias)                                                # :69
    s = set_conv(fh.setconv, net, graph)                                                           # :70
    y = torch.relu(linear(torch.cat([s, a], -1), fh.out_conv[0].weight, fh.out_conv[0].bias))      # :71-72
    return net, linear(y, fh.out_conv[2].weight, fh.out_conv[2].bias)


def flot_refine(m, flow, graph):
    """FlotRefine.forward (model/refine.py:16-22)."""
    x = set_conv(m.ref_conv1, flow, graph)
    x = set_conv(m.ref_conv2, x, graph)
    x = set_conv(m.ref_conv3, x, graph)
    return flow + linear(x, m.fc.weight, m.fc.bias)


def rsf_forward(model, p, num_iters, flow_init=None, bidirectional=False):
    """RSF.forward with gradients (model/RAFTSceneFlow.py:22-50) -> list of num_iters flows [B,N1,3].  flow_init [B,N1,3]
    (detached, fp32): the loop starts at xyz1 + flow_init (RAFT's warm start; no gradient reaches it).
    bidirectional: (forward, backward), the lists of model(p) and model([xyz2, xyz1]).  Clouds of equal sizes run as one 2B
    stack on the encoder's 2B pass, its graph kept whole: CorrInitFn on (cat[f1, f2], cat[f2, f1]), whose backward reaches
    both feature maps through the stacking, and one context pass and loop.  Different sizes: one pass per direction."""
    cb = model.corr_block
    ops.check_pair(p[0], p[1], cb.truncate_k)
    if bidirectional:
        ops.check_pair(p[1], p[0], cb.truncate_k)
    xyz1 = p[0].contiguous().float()                                           # attached: gradients reach the inputs
    xyz2 = p[1].contiguous().float()
    b, n, _ = xyz1.shape
    if cb.state_dtype != torch.float32:
        raise NotImplementedError("training differentiates through the fp32 state: call model.set_precision('fp32')")
    if xyz1.shape == xyz2.shape:
        both = torch.cat([xyz1, xyz2], 0)
        g_both = Graph.construct_graph(both, 32)                               # :25-26 (one batch of 2B clouds)
        fmap = flot_encoder(model.feature_extractor, both, g_both)
        if bidirectional:
            preds = _rsf_loop(model, both, torch.cat([xyz2, xyz1], 0), fmap, g_both, torch.cat([fmap[b:], fmap[:b]], 0), num_iters)
            return [f[:b] for f in preds], [f[b:] for f in preds]
        graph1 = Graph(g_both.nbr[:b].contiguous(), g_both._rel[:b].contiguous(), 32, [b * n] * 2)   # (the training path does not use .order)
        fmap1, fmap2 = fmap[:b], fmap[b:]
    else:                                                                      # clouds of different sizes: one pass per cloud
        graph1 = Graph.construct_graph(xyz1, 32)
        fmap1 = flot_encoder(model.feature_extractor, xyz1, graph1)
        graph2 = Graph.construct_graph(xyz2, 32)
        fmap2 = flot_encoder(model.feature_extractor, xyz2, graph2)
        if bidirectional:
            return (_rsf_loop(model, xyz1, xyz2, fmap1, graph1, fmap2, num_iters),
                    _rsf_loop(model, xyz2, xyz1, fmap2, graph2, fmap1, num_iters))
    return _rsf_loop(model, xyz1, xyz2, fmap1, graph1, fmap2, num_iters, flow_init)


def _rsf_loop(model, xyz1, xyz2, fmap1, graph1, fmap2, num_iters, flow_init=None):
    """The part of rsf_forward after the feature encoder: correlation, context and the loop -> the list of flows."""
    cb = model.corr_block
    corr_val, corr_idx = CorrInitFn.apply(fmap1, fmap2, cb.truncate_k, cb)     # :29
    xyz2p = ops.xyz_pad(xyz2)
    fct1 = flot_encoder(model.context_extractor, xyz1, graph1)                 # :31 (same cloud, same graph)
    net = torch.tanh(fct1[..., :model.hidden_dim])                             # :33-35
    inp = torch.relu(fct1[..., model.hidden_dim:])
    coords2 = xyz1.clone() if flow_init is None else xyz1 + flow_init          # (detached at the top of every iteration)
    preds = []
    # 'bf16-mixed': the loop's per-point layers on bf16 wgmma (LinearFn, bf16_layer_plan); the lookup stays fp32
    with ops.bf16_compute(model.bf16_compute):
        for _ in range(num_iters):
            coords2 = coords2.detach()                                         # :41
            vox, sel = CorrLookupFn.apply(corr_val, corr_idx, xyz2p, coords2, cb.num_levels, cb.base_scale, xyz2)
            corr = corr_features(cb, vox, sel)                                 # :42
            flow = coords2 - xyz1                                              # :43
            net, delta = update_block(model.update_block, net, inp, corr, flow, graph1)   # :44
            coords2 = coords2 + delta                                          # :45
            preds.append(coords2 - xyz1)                                       # :46
    return preds
