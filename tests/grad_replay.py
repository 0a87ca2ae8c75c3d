"""Decision-replay float64 oracle for whole-model gradients.

A training step takes discrete decisions: the kNN adjacency of every graph, the top-K candidates of the correlation, per
RAFT iteration the lookup's 32 nearest candidates and the voxel cell of every (point, candidate, level), the arg-max of
every max over 32 neighbours, and the branch of every ReLU, LeakyReLU and PReLU.  Two evaluations in different
precisions may take different decisions at near-ties, and then their gradients differ by far more than rounding: one
ReLU input within the fp32 error of 0 that takes the other branch moves a whole-model gradient by up to 1e-2.  Here the decisions are recorded from one run and the oracle
(oracle/pvraft_oracle.py) is re-run in float64 with every decision taken from the record instead of recomputed, so what
is left between the two gradients is the arithmetic.

* `record_library(model, xyz1, xyz2)` records the decisions of one forward of the library's training path
  (pvraft_b200/train.py): Graph.construct_graph's adjacency, CorrInitFn's top-K ids in the stored order, CorrLookupFn's
  slots and the lookup kernel's own cells (its `want_cube` output), the arg of every GnActMaxFn, the branch that
  gn_act_bwd takes for every element of a GroupNorm activation (restated bit for bit: t = fma(fl(fl(x - mean) * rstd),
  gamma, beta) >= 0, mean and rstd rounded to fp32 from the double statistics), and the branch of every torch.relu of
  the training path (its output > 0, what autograd's backward tests).
* `oracle_decisions(d, xyz1, xyz2, base_scale, 'record' | 'replay')` patches the oracle functions that decide
  (construct_graph, corr_init, voxel_cube_index, knn_select, neighbour_max, leaky_relu, prelu, relu): 'record' keeps
  what the oracle decides, 'replay' takes the decisions from `d`.

Records are keyed by what they decide and where, never by call order: ('graph', cloud), ('topk', dir), ('slots', it, dir),
('cells', it, level, dir), (GroupNorm name, *phase) for an arg-max, ('act', GroupNorm name, *phase) and
('relu', layer, it, dir), with phase = (cloud,) for an encoder, (it, dir) in the loop (it = -1 before it) and
('refine', dir) in the refiner.  dir is the direction a loop or refiner runs in: '12' for xyz1 -> xyz2, '21' for a
bidirectional forward's reverse pass.  The library runs an equal-size bidirectional forward as one 2B stack; each of its
records is split into the first B samples ('12') and the last B ('21').  Clouds of different sizes run one loop per
direction.  The oracle runs O.rsf_forward(P, x1, x2) and O.rsf_forward(P, x2, x1), each under its direction.
Masks and args are kept in the oracle's layout.  The library encodes both clouds in one 2B pass and reuses pc1's graph for
the context encoder, while the oracle calls these separately; `Decisions.get` asserts that every oracle call finds its one
record, and `Decisions.unused` lists records no call asked for.

The self-supervised loss (pvraft_b200/loss.py) decides too, and record_library keeps those decisions from the `ops` calls
the loss makes: ('knn', cloud, k), the smoothness and Laplacian graphs of ops.knn(p, p, k, mode=0), recorded once however
many directions build them; ('nn_ab', dir) / ('nn_ba', dir), Chamfer's nearest points; ('lap', dir), the Laplacian's
interpolation neighbours; ('cons', dir), the consistency term's.  Each of the last three is the [n*B, ...] tensor of its one
launch.  `self_supervised64` restates the loss in float64 on those records (tests/losses64.py).  A rigid fit's inlier set
is recorded by the caller as ('inliers',).
"""
import contextlib
import functools
import importlib.util
import math
import os

import numpy as np
import torch

import losses64 as L
from oracle import pvraft_oracle as O
from ties_restated import fma32


class Decisions:
    def __init__(self):
        self.rec, self.hits = {}, {}

    def put(self, key, value):
        assert key not in self.rec, f'two records for {key}'
        self.rec[key] = value

    def put_same(self, key, value):
        """A decision that several calls take (a graph two directions share): recorded once, and equal every time."""
        if key in self.rec:
            assert torch.equal(self.rec[key], value), f'two different records for {key}'
        else:
            self.rec[key] = value

    def get(self, key):
        assert key in self.rec, f'no record for {key}'
        self.hits[key] = self.hits.get(key, 0) + 1
        return self.rec[key]

    def unused(self):
        return sorted(set(self.rec) - set(self.hits), key=str)

    def to(self, device):
        d = Decisions()
        d.rec = {k: v.to(device) for k, v in self.rec.items()}
        return d


class _Patches:
    def __init__(self):
        self.undo = []

    def set(self, obj, name, value, static=False):
        self.undo.append((obj, name, obj.__dict__[name] if isinstance(obj, type) else getattr(obj, name)))
        setattr(obj, name, staticmethod(value) if static else value)

    def restore(self):
        for obj, name, old in reversed(self.undo):
            setattr(obj, name, old)


# ----------------------------------------------------------------------------------------------------------------------
# the library's decisions
# ----------------------------------------------------------------------------------------------------------------------
def gn_branch(x, stats, gamma, beta):
    """x [B,rows,C] fp32 with its raw GroupNorm sums stats [B,8,2] -> bool [B,rows,C]: t >= 0 as gn_act_bwd forms t
    (csrc/train.cu gn_mean_rstd, then fmaf((x - mean) * rstd, gamma, beta))."""
    b, rows, c = x.shape
    count = float(rows) * (c // 8)
    m = stats[..., 0] / count
    var = (stats[..., 1] / count - m * m).clamp_min(0.0)
    mean = m.float().repeat_interleave(c // 8, 1).unsqueeze(1)
    rstd = torch.rsqrt(var + 1e-5).float().repeat_interleave(c // 8, 1).unsqueeze(1)
    out = torch.empty(x.shape, dtype=torch.bool, device=x.device)
    for r0 in range(0, rows, 1 << 16):                        # (fma32 works in double: bound its temporaries)
        xh = (x[:, r0:r0 + (1 << 16)] - mean) * rstd
        out[:, r0:r0 + (1 << 16)] = fma32(xh, gamma.float().expand_as(xh), beta.float().expand_as(xh)) >= 0
    return out


def _edge_layout(mask, axis):
    """[B, N*32, C] -> the oracle's [B,C,32,N] (axis 2, SetConv) or [B,C,N,32] (axis 3, the kNN branch)."""
    b, rows, c = mask.shape
    m = mask.view(b, rows // 32, 32, c)
    return m.permute(0, 3, 2, 1) if axis == 2 else m.permute(0, 3, 1, 2)


@contextlib.contextmanager
def record_library(model, xyz1, xyz2):
    """Records the decisions of the library's training-path forward(s), and of the self-supervised loss, run inside the
    scope -> Decisions.  Also keeps each refiner's input flow under ('refine_input', dir) (not a decision: the replay of a
    refine step starts from it)."""
    from pvraft_b200 import graph as G, ops, train as T
    d = Decisions()
    names = {id(m): n for n, m in model.named_modules()}
    x1, x2 = xyz1.detach().float(), xyz2.detach().float()
    b = x1.shape[0]
    # dirs: [(direction, batch slice)] of the loop running now, None outside one
    st = dict(phase=None, it=-1, arg=None, lin=None, ctx=None, dirs=None)
    pnames = {id(prm): n for n, prm in model.named_parameters()}

    def clouds_of(pc):
        pc = pc.detach()
        if x1.shape == x2.shape and pc.shape[0] == 2 * b and torch.equal(pc, torch.cat([x1, x2], 0)):
            return [('pc1', slice(0, b)), ('pc2', slice(b, 2 * b))]
        for name, x in (('pc1', x1), ('pc2', x2)):
            if pc.shape == x.shape and torch.equal(pc, x):
                return [(name, slice(None))]
        raise AssertionError('a cloud that is neither input')

    def directions(pc):
        """The loop or refiner that starts on pc -> [(direction, slice)]: the 2B stack is both directions."""
        return [('12' if cloud == 'pc1' else '21', sl) for cloud, sl in clouds_of(pc)]

    def direction_of(target):
        """The direction of a loss launch, from the cloud it searches (pc2 for '12')."""
        (cloud, _), = clouds_of(target)
        return '12' if cloud == 'pc2' else '21'

    p = _Patches()
    construct = G.Graph.__dict__['construct_graph'].__func__

    def construct_graph(pcloud, k):
        g = construct(pcloud, k)
        for cloud, sl in clouds_of(pcloud):
            d.put(('graph', cloud), g.nbr[sl].long())
        return g

    def flot_encoder(m, pc, graph, _orig=T.flot_encoder):
        st['phase'] = [((cloud,), sl) for cloud, sl in clouds_of(pc)]
        try:
            out = _orig(m, pc, graph)
        finally:
            st['phase'] = None
        if m is model.context_extractor:
            st['ctx'] = out
        return out

    def phases():
        return st['phase'] if st['phase'] is not None else [((st['it'], dr), sl) for dr, sl in st['dirs']]

    def put_branch(name, x, stats, gn, act, edge_axis=None):
        if act != ops.ACT_LRELU:
            return
        mask = gn_branch(x.detach(), stats, gn.weight.detach(), gn.bias.detach())
        for ph, sl in phases():
            d.put(('act', name, *ph), _edge_layout(mask[sl], edge_axis) if edge_axis else mask[sl].transpose(1, 2))

    def gn_act(x, stats, gn, act=ops.ACT_LRELU, *a, _orig=T.gn_act, **k):
        put_branch(names[id(gn)], x, stats, gn, act)
        return _orig(x, stats, gn, act, *a, **k)

    def linear(x, w, b=None, stats=False, _orig=T.linear):
        y = _orig(x, w, b, stats)
        st['lin'] = ((y[0] if stats else y), pnames.get(id(w), '')[:-len('.weight')])
        return y

    def relu(x, _orig=torch.relu):
        y = _orig(x)
        if st['lin'] is not None and x is st['lin'][0]:
            layer = st['lin'][1]
        elif st['ctx'] is not None and x._base is st['ctx']:
            layer = 'context_extractor'
        else:
            return y
        for dr, sl in st['dirs']:
            d.put(('relu', layer, st['it'], dr), (y[sl] > 0).transpose(1, 2))
        return y

    def flot_refine(m, flow, graph, _orig=T.flot_refine):
        if flow.shape[0] == 2 * b and x1.shape == x2.shape:         # the 2B stack of a bidirectional forward
            dirs = [('12', slice(0, b)), ('21', slice(b, 2 * b))]
        else:
            dirs = [('12' if flow.shape[1] == x1.shape[1] else '21', slice(None))]
        for dr, sl in dirs:
            d.put(('refine_input', dr), flow[sl].detach().clone())
        st['phase'] = [(('refine', dr), sl) for dr, sl in dirs]
        try:
            return _orig(m, flow, graph)
        finally:
            st['phase'] = None

    def gn_act_maxk(*a, _orig=ops.gn_act_maxk, **k):
        y, st['arg'] = _orig(*a, **k)
        return y, st['arg']

    def gn_act_max(x, stats, gn, act=ops.ACT_LRELU, *a, _orig=T.gn_act_max, **k):
        name = names[id(gn)]
        put_branch(name, x, stats, gn, act, 3 if name.endswith('knn_conv.1') else 2)
        st['arg'] = None
        y = _orig(x, stats, gn, act, *a, **k)
        for ph, sl in phases():
            d.put((name, *ph), st['arg'][sl].long())
        return y

    def rsf_loop(model_, xyz1_, *a, _orig=T._rsf_loop, **k):
        st['dirs'], st['it'] = directions(xyz1_), -1                  # the iteration count restarts per direction
        try:
            return _orig(model_, xyz1_, *a, **k)
        finally:
            st['dirs'] = None

    def corr_reorder(val, idx, _orig=ops.corr_reorder):
        val, idx = _orig(val, idx)
        if st['dirs'] is not None:                                      # (not the inference path's correlation)
            for dr, sl in st['dirs']:
                d.put(('topk', dr), idx[sl].long())
        return val, idx

    def corr_lookup(*a, _orig=ops.corr_lookup, **k):
        if not k.get('want_slots'):
            return _orig(*a, **k)
        st['it'] += 1
        k['want_cube'] = True
        out = _orig(*a, **k)
        for dr, sl in st['dirs']:
            d.put(('slots', st['it'], dr), out['knn_slot'][sl].long())
            for lvl in range(out['cube'].shape[-1]):
                d.put(('cells', st['it'], lvl, dr), out['cube'][sl][..., lvl].long())
        return out

    # the self-supervised loss's own searches
    def knn(xyz, query, k, *a, _orig=ops.knn, **kw):
        out = _orig(xyz, query, k, *a, **kw)
        if not a and kw.get('mode', 0) == 0 and not kw.get('want_rel', False) and torch.equal(xyz, query):
            (cloud, _), = clouds_of(xyz)
            d.put_same(('knn', cloud, k), out.long())
        return out

    def chamfer(w, target, *a, _orig=ops.chamfer, **kw):
        out = _orig(w, target, *a, **kw)
        dr = direction_of(target)
        d.put(('nn_ab', dr), out[1].long())
        d.put(('nn_ba', dr), out[2].long())
        return out

    def laplacian(w, target, *a, _orig=ops.laplacian, **kw):
        out = _orig(w, target, *a, **kw)
        d.put(('lap', direction_of(target)), out[1].long())
        return out

    def flow_consistency(w, f12, target, *a, _orig=ops.flow_consistency, **kw):
        out = _orig(w, f12, target, *a, **kw)
        d.put(('cons', direction_of(target)), out[1].long())
        return out

    p.set(G.Graph, 'construct_graph', construct_graph, static=True)
    p.set(T, 'flot_encoder', flot_encoder)
    p.set(T, 'flot_refine', flot_refine)
    p.set(T, 'gn_act_max', gn_act_max)
    p.set(T, 'gn_act', gn_act)
    p.set(T, 'linear', linear)
    p.set(torch, 'relu', relu)
    p.set(ops, 'gn_act_maxk', gn_act_maxk)
    p.set(ops, 'corr_reorder', corr_reorder)
    p.set(ops, 'corr_lookup', corr_lookup)
    p.set(T, '_rsf_loop', rsf_loop)
    p.set(ops, 'knn', knn)
    p.set(ops, 'chamfer', chamfer)
    p.set(ops, 'laplacian', laplacian)
    p.set(ops, 'flow_consistency', flow_consistency)
    try:
        yield d
    finally:
        p.restore()


# ----------------------------------------------------------------------------------------------------------------------
# the oracle, recording or replaying
# ----------------------------------------------------------------------------------------------------------------------
def graph_from(pc, nbr):
    """An oracle Graph on the adjacency nbr [B,N,k] (local ids): edge features pc[nbr] - pc, differentiable w.r.t. pc."""
    b, n, k = nbr.shape
    bi = torch.arange(b, device=pc.device).view(b, 1, 1)
    feats = (pc[bi, nbr] - pc.unsqueeze(2)).reshape(b * n * k, 3)
    edges = (nbr + bi * n).reshape(-1)
    return O.Graph(edges, feats, k, (b * n, b * n))


def _corr_state(fmap1, fmap2, xyz2, idx):
    """CorrState of the candidates idx [B,N1,K]: their correlations (model/corr.py:95-100) and xyz2 rows, in idx's order.
    (Gathering K rows of fmap2 per point would take B*N1*K*C values; the all-pairs matrix takes B*N1*N2.)"""
    bi = torch.arange(idx.shape[0], device=idx.device).view(-1, 1, 1)
    return O.CorrState(torch.gather(O.calculate_corr(fmap1, fmap2), 2, idx), idx, xyz2[bi, idx])


# the PReLU slopes: their gradients sum dy * t over t < 0, which cancels; `slope_terms` collects sum |dy * t| instead
PRELU_SLOPE = {'corr_block.out_conv.1': 'corr_block.out_conv.2.weight', 'corr_block.knn_conv.1': 'corr_block.knn_conv.2.weight'}


@contextlib.contextmanager
def oracle_decisions(d, xyz1, xyz2, base_scale, mode, slope_terms=None, direction='12'):
    """Inside the scope the oracle's deciding functions record into (mode 'record') or replay from (mode 'replay') the
    Decisions d.  xyz1 / xyz2 are the very tensors the oracle is given (an encoder's cloud is recognised by identity);
    direction: '12' for a forward on (xyz1, xyz2), '21' for one on (xyz2, xyz1).  slope_terms: a dict that every later
    backward through a PReLU adds sum |dy * t| over its t < 0 to, under the slope's parameter name.  In 'record' mode a
    decision that is taken again (an encoder that both directions run) must equal its record."""
    assert mode in ('record', 'replay') and direction in ('12', '21')
    rec = mode == 'record'
    st = dict(phase=None, it=-1)
    put = d.put_same
    orig = {n: getattr(O, n) for n in ('construct_graph', 'flot_encoder', 'flot_refine', 'corr_init', 'corr_lookup',
                                       'voxel_cube_index', 'knn_select', 'neighbour_max', 'leaky_relu', 'prelu', 'relu')}

    def cloud_of(pc):
        if pc is xyz1:
            return 'pc1'
        assert pc is xyz2, 'a cloud that is neither input'
        return 'pc2'

    def construct_graph(pc, k=O.KNN):
        key = ('graph', cloud_of(pc))
        if rec:
            g = orig['construct_graph'](pc, k)
            b, n, _ = pc.shape
            put(key, g.edges.reshape(b, n, k) - (torch.arange(b, device=pc.device) * n).view(b, 1, 1))   # (again for the context encoder)
            # the replay's arithmetic on the decision: a float64 record and its replay give the same bits
            return graph_from(pc, d.rec[key])
        return graph_from(pc, d.get(key))

    def flot_encoder(P, prefix, pc, graph=None):
        st['phase'] = (cloud_of(pc),)
        try:
            return orig['flot_encoder'](P, prefix, pc, graph)
        finally:
            st['phase'] = None

    def flot_refine(P, prefix, flow, graph):
        st['phase'] = ('refine', direction)
        try:
            return orig['flot_refine'](P, prefix, flow, graph)
        finally:
            st['phase'] = None

    def corr_init(fmap1, fmap2, xyz2_, truncate_k):
        if rec:
            s = orig['corr_init'](fmap1, fmap2, xyz2_, truncate_k)
            put(('topk', direction), s.indices)
            return _corr_state(fmap1, fmap2, xyz2_, s.indices)
        return _corr_state(fmap1, fmap2, xyz2_, d.get(('topk', direction)))

    def corr_lookup(*a, **k):
        st['it'] += 1
        return orig['corr_lookup'](*a, **k)

    def voxel_cube_index(state, coords, r):
        key = ('cells', st['it'], int(round(math.log2(r / base_scale))), direction)
        if rec:
            cube, valid = orig['voxel_cube_index'](state, coords, r)
            put(key, torch.where(valid, cube, -1))
            return cube, valid
        cell = d.get(key)
        return cell.clamp_min(0), cell >= 0

    def knn_select(state, coords, knn=O.KNN):
        if rec:
            s = orig['knn_select'](state, coords, knn)
            put(('slots', st['it'], direction), s)
            return s
        return d.get(('slots', st['it'], direction))

    def neighbour_max(x, dim, layer):
        # x [B,C,32,N] (dim 2) or [B,C,N,32] (dim 3); the arg is kept as the library keeps it, [B,N,C]
        key = (layer, *phase())
        if rec:
            v, i = x.max(dim=dim)
            put(key, i.transpose(1, 2))
            return v
        idx = d.get(key).transpose(1, 2).unsqueeze(dim)
        return x.gather(dim, idx).squeeze(dim)

    def phase():
        return st['phase'] if st['phase'] is not None else (st['it'], direction)

    def branch(key, x):
        if rec:
            put(key, x >= 0)
            return x >= 0
        return d.get(key)

    def leaky_relu(x, slope=0.1, layer=None):
        return torch.where(branch(('act', layer, *phase()), x), x, slope * x)

    def prelu(x, a, layer=None):
        mask = branch(('act', layer, *phase()), x)
        y = torch.where(mask, x, a.view(-1)[0] * x)
        if slope_terms is not None and y.requires_grad:
            def terms(g, x=x.detach(), neg=~mask, name=PRELU_SLOPE[layer]):
                slope_terms[name] = slope_terms.get(name, 0.0) + float((g * x).abs()[neg].sum())
            y.register_hook(terms)
        return y

    def relu(x, layer=None):
        key = ('relu', layer, st['it'], direction)
        if rec:
            put(key, x > 0)
            return torch.relu(x)
        return torch.where(d.get(key), x, torch.zeros_like(x))

    new = dict(construct_graph=construct_graph, flot_encoder=flot_encoder, flot_refine=flot_refine, corr_init=corr_init,
               corr_lookup=corr_lookup, voxel_cube_index=voxel_cube_index, knn_select=knn_select, neighbour_max=neighbour_max,
               leaky_relu=leaky_relu, prelu=prelu, relu=relu)
    assert set(new) == set(orig)
    for n, f in new.items():
        setattr(O, n, f)
    try:
        yield d
    finally:
        for n, f in orig.items():
            setattr(O, n, f)


# ----------------------------------------------------------------------------------------------------------------------
# losses and the comparison
# ----------------------------------------------------------------------------------------------------------------------
def linear_loss(flows, gs):
    """sum_i <flows_i, G_i>: no kink, so no decision in the loss."""
    return sum((f * g.to(f.dtype)).sum() for f, g in zip(flows, gs))


def sequence_loss(flows, gt, signs=None, gamma=0.8):
    """tests/train_helpers.sequence_loss; with `signs` (one tensor per flow) |x| is taken as signs * x, the L1 kinks
    decided by another run."""
    n = len(flows)
    gt = gt.to(flows[0].dtype)
    if signs is None:
        return sum(gamma ** (n - i - 1) * (flows[i] - gt).abs().sum(-1).mean() for i in range(n))
    return sum(gamma ** (n - i - 1) * (signs[i].to(gt.dtype) * (flows[i] - gt)).sum(-1).mean() for i in range(n))


def self_supervised64(d, flows, x1, x2, gamma=0.8, k=9, wc=1.0, ws=1.0, wl=0.0, k_lap=10, k_int=5, wcons=0.0):
    """sequence_self_supervised_loss in float64 with every neighbour set taken from d's loss records.  flows: a list of
    [B,N1,3] (one direction), or the pair (list [B,N1,3], list [B,N2,3]) of a bidirectional forward.  A refiner's loss,
    self_supervised_loss of one flow or of a pair, is the same with one-element lists."""
    pair = isinstance(flows, tuple)
    n = len(flows[0]) if pair else len(flows)
    recs = []
    for dr, a, b in (('12', 'pc1', 'pc2'), ('21', 'pc2', 'pc1'))[:2 if pair else 1]:
        def split(key):                                # the [n*B, ...] tensor of one launch -> n tensors [B, ...]
            t = d.get((key, dr))
            return list(t.unflatten(0, (n, t.shape[0] // n)))
        graphs = (d.get(('knn', a, k)),) + ((d.get(('knn', a, k_lap)), d.get(('knn', b, k_lap))) if wl != 0 else (None, None))
        recs.append(dict(nbrs=graphs, chamfer=list(zip(split('nn_ab'), split('nn_ba'))),
                         lap=split('lap') if wl != 0 else None, cons=split('cons') if pair and wcons != 0 else None))
    if not pair:
        r = recs[0]
        nbr, g1, g2 = r['nbrs']
        return L.loss64(flows, x1, x2, nbr, g1, g2, gamma=gamma, wc=wc, ws=ws, wl=wl, k_int=k_int, lap_idx=r['lap'],
                        chamfer_idx=r['chamfer'])
    return L.pair_loss64(flows[0], flows[1], x1, x2, gamma=gamma, wc=wc, ws=ws, wl=wl, wcons=wcons, k_int=k_int,
                         nbrs=[r['nbrs'] for r in recs], chamfer_idx=[r['chamfer'] for r in recs],
                         lap_idx=[r['lap'] for r in recs], cons_idx=[r['cons'] for r in recs] if wcons != 0 else None)


def rsf_flows(P, x1, x2, iters, levels, base_scale, truncate_k, flow_init=None):
    """O.rsf_forward, with the loop started at xyz1 + flow_init when it is given (a constant: no gradient reaches it;
    RSF.forward's warm start)."""
    li = O.prepare(P, x1, x2, truncate_k)
    if flow_init is None:
        return O.raft_loop(P, li, x1, iters, levels, base_scale)
    coords2, net, flows = x1 + flow_init.detach(), li.net, []
    for _ in range(iters):
        coords2 = coords2.detach()
        corr = O.corr_lookup(P, li.state, coords2, levels, base_scale)
        net, delta = O.update_block(P, net, li.inp, corr, coords2 - x1, li.graph)
        coords2 = coords2 + delta
        flows.append(coords2 - x1)
    return flows


def detached(out):
    return tuple(detached(o) for o in out) if isinstance(out, tuple) else [f.detach() for f in out] if isinstance(out, list) else out.detach()


def replay_rsf(W, pc1, pc2, d, iters, levels, base_scale, truncate_k, losses, device, flow_init=None, bidirectional=False):
    """The oracle's RSF forward in float64 on `device` with d's decisions; -> (flows, [grads of each loss], [the PReLU
    slopes' sum |dy * t| of each loss]) where a grads dict holds every parameter and 'xyz1' / 'xyz2'.  losses: functions
    (flows, xyz1, xyz2) -> scalar, the clouds being the replay's float64 leaves.  flow_init: the warm start.
    bidirectional: flows is the pair (O.rsf_forward(P, x1, x2) under '12', O.rsf_forward(P, x2, x1) under '21')."""
    P = {k: v.detach().to(device, torch.float64).requires_grad_(True) for k, v in W.items()}
    x1 = pc1.detach().to(device, torch.float64).requires_grad_(True)
    x2 = pc2.detach().to(device, torch.float64).requires_grad_(True)
    init = None if flow_init is None else flow_init.detach().to(device, torch.float64)
    terms = {}
    with oracle_decisions(d, x1, x2, base_scale, 'replay', terms):
        flows = rsf_flows(P, x1, x2, iters, levels, base_scale, truncate_k, init)
    if bidirectional:
        with oracle_decisions(d, x1, x2, base_scale, 'replay', terms, direction='21'):
            flows = (flows, rsf_flows(P, x2, x1, iters, levels, base_scale, truncate_k))
    grads, scales = [], []
    for i, fn in enumerate(losses):
        terms.clear()
        grads += _grads([fn], flows, P, x1, x2, retain=i + 1 < len(losses))
        scales.append(dict(terms))
    return detached(flows), grads, scales


def replay_refine(W, pc1, pc2, d, losses, device, bidirectional=False):
    """The refine step (RSF_refine's refiner on the loop's last flow, RAFTSceneFlowRefine.py:46) in float64 with d's
    arg-max decisions, starting from the recorded ('refine_input', dir) (the other run's loop output, no gradient) on the
    recorded graph of the cloud it starts on.  bidirectional: both directions, the refined flows as a pair.  losses:
    functions (refined, xyz1, xyz2) -> scalar.  -> (refined, [grads of each loss]): the refine_block parameters and 'xyz1'
    (= - d flow), and 'xyz2' for a pair."""
    P = {k: v.detach().to(device, torch.float64).requires_grad_(k.startswith('refine_block.')) for k, v in W.items()}
    x1 = pc1.detach().to(device, torch.float64).requires_grad_(True)
    x2 = pc2.detach().to(device, torch.float64).requires_grad_(bidirectional)
    out = []
    for dr, x, cloud in (('12', x1, 'pc1'), ('21', x2, 'pc2'))[:2 if bidirectional else 1]:
        f = d.get(('refine_input', dr)).to(device, torch.float64) + (x.detach() - x)
        graph = graph_from(x.detach(), d.get(('graph', cloud)).to(device))
        with oracle_decisions(d, x1, x2, 1.0, 'replay', direction=dr):
            out.append(O.flot_refine(P, 'refine_block', f, graph))
    refined = tuple(out) if bidirectional else out[0]
    P = {k: v for k, v in P.items() if v.requires_grad}
    return detached(refined), _grads(losses, refined, P, x1, x2 if bidirectional else None)


def _grads(losses, out, P, x1, x2, retain=False):
    leaves = dict(P, xyz1=x1, **({} if x2 is None else {'xyz2': x2}))
    res = []
    for i, fn in enumerate(losses):
        g = torch.autograd.grad(fn(out, x1, x2), list(leaves.values()), retain_graph=retain or i + 1 < len(losses), allow_unused=True)
        res.append({k: (torch.zeros_like(v) if gv is None else gv) for (k, v), gv in zip(leaves.items(), g)})
    return res


def rel_l2(got, want):
    """{name: ||got - want|| / ||want||} in float64."""
    out = {}
    for k, w in want.items():
        a, w = got[k].detach().double().to(w.device), w.detach().double()
        assert a.shape == w.shape, (k, a.shape, w.shape)
        out[k] = float((a - w).norm() / w.norm().clamp_min(1e-300))
    return out


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


@functools.lru_cache(None)
def _make_golden():
    spec = importlib.util.spec_from_file_location('make_golden', os.path.join(GOLDEN, 'make_golden.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_gradients(name):
    """tests/golden/<name> (a gradient fixture of make_golden.py) -> (the float64 sketch of every gradient by tensor name,
    the other arrays)."""
    z = np.load(os.path.join(GOLDEN, name), allow_pickle=False)
    return ({k[2:]: z[k] for k in z.files if k.startswith('s/')},
            {k: torch.from_numpy(z[k].copy()) for k in z.files if not k.startswith('s/')})


def sketched_rel_l2(got, want):
    """{name: relative L2 error of got[name] against a fixture's sketch want[name]}: exact for tensors the fixture keeps
    whole, a Johnson-Lindenstrauss estimate (within a factor 1 +- 0.2) for the others (make_golden.grad_sketch)."""
    sketch = _make_golden().grad_sketch
    out = {}
    for k, w in want.items():
        a = sketch(k, got[k].detach().double().cpu())
        assert a.shape == w.shape, (k, a.shape, w.shape)
        out[k] = float(np.linalg.norm(a - w) / max(float(np.linalg.norm(w)), 1e-300))
    return out


def worst(errs, n=6):
    return sorted(errs.items(), key=lambda kv: -kv[1])[:n]
