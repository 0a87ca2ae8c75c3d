"""Whole-model gradients of the self-supervised, bidirectional, warm-started and rigid-fit training steps against float64 at
the library's own decisions.

test_gpu_grad_replay.py replays the supervised stage-1 and refine steps.  Here the step's loss has discrete decisions of
its own -- the smoothness and Laplacian graphs, Chamfer's nearest points, the Laplacian and consistency interpolation
neighbours, a rigid fit's inlier set -- and a bidirectional forward runs the loop once per direction, or once on the 2B
stack of an equal-size pair.  tests/grad_replay.py records all of them per direction, and the oracle replays both
directions and the float64 restatement of the loss (tests/losses64.py, the Horn fit of test_gpu_rigid_motion.py) with
them.  What is left between the gradients is the library's arithmetic: how S = n B predictions share one loss launch,
the gamma weights, the reverse direction's swapped clouds, the stacked forward's d fmap reaching each feature map through
both halves, and d xyz2 as the sum of the lookup table's, the encoder's and the loss's gradients.

Every case runs in the default form and under torch.use_deterministic_algorithms(True); every parameter gradient, both
input gradients and the flows are compared, the PReLU slopes as |error| / sum |dy t| (test_gpu_grad_replay.py).  Run
with -s to print the measured values.
"""
import pytest
import torch

import grad_replay as R
import test_gpu_grad_replay as G
from test_gpu_rigid_motion import horn_torch, random_rotation

pytestmark = pytest.mark.gpu

SS = dict(w_laplacian=0.3)                  # the three-term loss
PAIR = dict(w_laplacian=0.3, w_consistency=0.3)
CASES = {
    # name: (model, B, N1, N2, iterations, trained-looking weights, forward, loss)
    'two_term':           ('RSF', 2, 1024, 1024, 3, False, 'one', {}),
    'laplacian_unequal':  ('RSF', 2, 1024, 1536, 3, False, 'one', SS),
    'laplacian_straddle': ('RSF', 3, 1004, 1004, 3, True, 'one', SS),
    'pair_stacked':       ('RSF', 2, 1024, 1024, 3, True, 'pair', PAIR),
    'pair_unequal':       ('RSF', 2, 1024, 1280, 3, False, 'pair', PAIR),
    'refine_pair':        ('RSF_refine', 2, 1024, 1024, 3, True, 'pair', PAIR),
    'warm':               ('RSF', 2, 1024, 1024, 3, False, 'warm', None),
    'rigid':              ('RSF', 2, 1024, 1024, 3, False, 'rigid', None),
}
K = 128

# Per case: the worst relative L2 over every gradient but the PReLU slopes, both forms and every loss; the flows' (the
# refined flows'); the slopes' |error| / sum |dy t|.  Measured on an H100 80GB HBM3 (700 W), worst of two runs:
#   two_term 1.26e-5, laplacian_unequal 1.27e-5, laplacian_straddle 1.13e-5, pair_stacked 6.2e-6, pair_unequal 9.5e-6,
#   refine_pair 1.24e-6, warm 4.8e-6, rigid 3.8e-6;
#   flows 3.2e-6, 3.3e-6, 2.4e-6, 2.4e-6, 3.4e-6, 4.9e-7 (refined), 2.7e-6, 1.0e-6;  PReLU slopes 5.0e-8 (pair_unequal).
# Each bound is at most 3x its measured value.
BOUND = {'two_term': 3.7e-5, 'laplacian_unequal': 3.8e-5, 'laplacian_straddle': 3.3e-5, 'pair_stacked': 1.8e-5,
         'pair_unequal': 2.8e-5, 'refine_pair': 3.7e-6, 'warm': 1.4e-5, 'rigid': 1.1e-5}
BOUND_FLOWS = {'two_term': 9.6e-6, 'laplacian_unequal': 9.9e-6, 'laplacian_straddle': 7.2e-6, 'pair_stacked': 7.2e-6,
               'pair_unequal': 1.0e-5, 'refine_pair': 1.4e-6, 'warm': 8.1e-6, 'rigid': 3.0e-6}
BOUND_SLOPE = 1.5e-7


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def leaf(t):
    return t.detach().clone().requires_grad_(True)


def boxes_pair(b, n, seed):
    """A ground slab 4 m x 4 m x 0.3 m under two boxes of n/8 points each; pc2 = the ego motion (R_gt, t_gt) of pc1, the
    boxes moved a further 0.27 m and 0.32 m.  -> pc1, pc2, R_gt [B,3,3], t_gt [B,3] (float64), the box points' mask."""
    g = torch.Generator().manual_seed(seed)
    nb = n // 8
    boxes = (((1.0, 1.0), (0.25, 0.1)), ((3.0, 2.5), (-0.1, 0.3)))
    pc1, pc2, rs, ts = [], [], [], []
    for _ in range(b):
        x = torch.rand(n, 3, generator=g) * torch.tensor([4.0, 4.0, 0.3])
        rot, t = random_rotation(g, 2.0), torch.tensor([0.05, -0.03, 0.0], dtype=torch.float64)
        for j, ((cx, cy), _) in enumerate(boxes):
            x[j * nb:(j + 1) * nb] = torch.rand(nb, 3, generator=g) * torch.tensor([0.8, 0.5, 0.6]) + torch.tensor([cx, cy, 0.3])
        y = (x.double() @ rot.T + t).float()
        for j, (_, (mx, my)) in enumerate(boxes):
            y[j * nb:(j + 1) * nb] += torch.tensor([mx, my, 0.0])
        pc1.append(x), pc2.append(y), rs.append(rot), ts.append(t)
    moving = torch.zeros(b, n, dtype=torch.bool)
    moving[:, :2 * nb] = True
    return torch.stack(pc1), torch.stack(pc2), torch.stack(rs), torch.stack(ts), moving


def rigid64(d, flow, x1, r_gt, t_gt):
    """sum_s ||R_s - R_gt||^2 + ||t_s - t_gt||^2 of the float64 Horn fit on the recorded inliers."""
    inl = d.get(('inliers',))
    total = 0
    for s in range(flow.shape[0]):
        rot, t = horn_torch(x1[s][inl[s]], (x1[s] + flow[s])[inl[s]])
        total = total + ((rot - r_gt[s]) ** 2).sum() + ((t - t_gt[s]) ** 2).sum()
    return total


def setup(case, dev):
    """-> model, W, pc1, pc2, forward kwargs, [library losses (out, x1, x2, d)], [replay losses (out, x1, x2)] (built once
    the library's out and decisions exist, by the returned `replay_losses(out, d)`)."""
    from pvraft_b200 import RSF, RSF_refine
    import pvraft_b200
    from pvraft_b200.loss import self_supervised_loss, sequence_self_supervised_loss
    name, b, n1, n2, iters, trained, fwd, kw = CASES[case]
    m = G.model_for(RSF_refine if name == 'RSF_refine' else RSF, K, trained, seed=4 if name == 'RSF_refine' else 2)
    fk = dict(bidirectional=fwd == 'pair')
    if fwd == 'rigid':
        pc1, pc2, r_gt, t_gt, moving = boxes_pair(b, n1, seed=3)
        with torch.no_grad():           # a flow head whose steps are small: the warm start at the motion decides the inliers
            for p in m.update_block.flow_head.out_conv[2].parameters():
                p.mul_(0.05)
        fk['flow_init'] = (pc2 - pc1).to(dev)
    else:
        pc1, pc2 = G.clouds(b, n1, n2, seed=n1 + n2 + b)
    if fwd == 'warm':
        fk['flow_init'] = (0.6 * (pc2[:, :n1] - pc1) + 0.01 * torch.randn(b, n1, 3, generator=torch.Generator().manual_seed(3))).to(dev)
    m = m.to(dev).train()
    if name == 'RSF_refine':
        for k, p in m.named_parameters():
            p.requires_grad_(k.startswith('refine_block.'))
    W = {k: v.detach().clone() for k, v in m.state_dict().items()}
    pc1, pc2 = pc1.to(dev), pc2.to(dev)
    if fwd in ('one', 'pair'):
        fn = self_supervised_loss if name == 'RSF_refine' else sequence_self_supervised_loss
        lib = [lambda out, x1, x2, d: fn(out, {'sequence': [x1, x2]}, **kw)]
        rep_kw = dict(wl=kw.get('w_laplacian', 0.0), wcons=kw.get('w_consistency', 0.0))
        if name == 'RSF_refine':
            def replay_losses(out, d):
                return [lambda r, x1, x2: R.self_supervised64(d, ([r[0]], [r[1]]), x1, x2, **rep_kw)]
        else:
            def replay_losses(out, d):
                return [lambda f, x1, x2: R.self_supervised64(d, f, x1, x2, **rep_kw)]
    elif fwd == 'warm':
        gt = pc2 - pc1
        gs = [torch.randn(b, n1, 3, generator=torch.Generator().manual_seed(5 + i), dtype=torch.float64).to(dev) for i in range(iters)]
        lib = [lambda out, *_: R.linear_loss(out, gs), lambda out, *_: R.sequence_loss(out, gt)]

        def replay_losses(out, d):
            signs = [torch.sign(f - gt) for f in out]
            return [lambda f, *_: R.linear_loss(f, gs), lambda f, *_: R.sequence_loss(f, gt, signs)]
    else:
        r_gt, t_gt, moving = r_gt.to(dev), t_gt.to(dev), moving.to(dev)

        def fit(out, x1, x2, d):
            o = pvraft_b200.rigid_motion(x1, out[-1], threshold=0.05)
            d.put(('inliers',), o.inliers.clone())
            assert not bool(o.degenerate.any())
            # a proper subset: the static scene, every box point out
            assert bool((o.inliers.sum(1) < n1).all()) and bool((o.inliers.sum(1) > n1 // 2).all()), o.inliers.sum(1)
            assert not bool((o.inliers & moving).any())
            return ((o.rotation.double() - r_gt) ** 2).sum() + ((o.translation.double() - t_gt) ** 2).sum()
        lib = [fit]

        def replay_losses(out, d):
            return [lambda f, x1, x2: rigid64(d, f[-1], x1, r_gt, t_gt)]
    return m, W, pc1, pc2, iters, fk, lib, replay_losses


def flows_error(got, want):
    flat = (lambda o: [t for part in o for t in flat(part)] if isinstance(o, (tuple, list)) else [o])
    return max(float((a.double() - r).norm() / r.norm()) for a, r in zip(flat(got), flat(want)))


@pytest.mark.parametrize('det', [False, True], ids=['default', 'DET'])
@pytest.mark.parametrize('case', list(CASES))
def test_gradients_match_float64_replay(dev, case, det):
    m, W, pc1, pc2, iters, fk, lib, replay_losses = setup(case, dev)
    refine = CASES[case][0] == 'RSF_refine'
    x1, x2 = leaf(pc1), leaf(pc2)
    with G.det_mode(det), R.record_library(m, x1, x2) as d:
        out = m([x1, x2], iters, **fk)
        values = [fn(out, x1, x2, d) for fn in lib]
    named = [(k, p) for k, p in m.named_parameters() if p.requires_grad] + [('xyz1', x1), ('xyz2', x2)]
    assert len(named) == (29 if refine else 95) + 2
    got = []
    for i, v in enumerate(values):
        with G.det_mode(det):
            g = torch.autograd.grad(v, [t for _, t in named], retain_graph=i + 1 < len(values), allow_unused=True)
        got.append({k: (torch.zeros_like(t) if gv is None else gv) for (k, t), gv in zip(named, g)})
    out = R.detached(out)
    del m, values
    torch.cuda.empty_cache()
    losses = replay_losses(out, d)
    if refine:
        ref, want = R.replay_refine(W, pc1, pc2, d, losses, dev, bidirectional=True)
        scales = [{}] * len(want)
    else:
        ref, want, scales = R.replay_rsf(W, pc1, pc2, d, iters, 3, 0.25, K, losses, dev, flow_init=fk.get('flow_init'),
                                         bidirectional=fk['bidirectional'])
    assert not d.unused(), d.unused()
    e_f = flows_error(out, ref)
    worst = worst_slope = 0.0
    for i, (gg, ww, sc) in enumerate(zip(got, want, scales)):
        errs = R.rel_l2(gg, ww)
        slope = {k: float((gg[k].double() - ww[k]).abs().sum()) / sc[k] for k in R.PRELU_SLOPE.values() if k in sc}
        tag = f'{case} {"DET" if det else "default"} loss {i} (flows {e_f:.1e})'
        worst = max(worst, G.report(tag, {k: v for k, v in errs.items() if k not in R.PRELU_SLOPE.values()}))
        if slope:
            print(f'{tag}: PReLU slopes, error / sum |dy t|: ' + ', '.join(f'{k} {v:.2e} (relative L2 {errs[k]:.2e})' for k, v in slope.items()))
            worst_slope = max(worst_slope, *slope.values())
    assert e_f < BOUND_FLOWS[case], e_f
    assert worst < BOUND[case], worst
    assert worst_slope < BOUND_SLOPE, worst_slope
