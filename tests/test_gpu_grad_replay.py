"""Whole-model gradients against float64 at the library's own decisions.

The whole-model tests of test_gpu_train.py / test_gpu_train_coverage.py compare with autograd through the fp32 CPU oracle,
which takes its own discrete decisions (kNN sets, top-K membership, voxel cells, arg-maxes, activation branches); where the
two runs decide a near-tie differently a gradient contribution moves, so those tests need 2e-2 per tensor.  (One ReLU input
within the fp32 error of 0 taking the other branch moved GroupNorm-bias gradients by up to 8.5e-3; DESIGN.md section 5.)  Here every decision of the
library's step is recorded and the oracle replays them in float64 on the device (tests/grad_replay.py), so the
difference is the library's arithmetic alone and the bound is 1e-4 relative L2 per tensor or tighter.

Every case runs in the default form and under torch.use_deterministic_algorithms(True), with two losses on one forward:
  linear  sum_i <flows_i, G_i>, G fixed random: no kink
  l1      the sequence loss (tools/loss.py), its signs taken from the library's flows in the replay
Cases: stage-1 RSF at B = 2, N = 1024, K = 128 with default and trained-looking weights (random GroupNorm affines, PReLU
slopes -0.3 / 1.7); B = 3, N = 1004 (the CUDA-core layers; 8-point CTAs straddle samples); N1 = 1024, N2 = 1536; the
bench training shape B = 2, N = 8192, K = 512, 8 iterations; an RSF_refine refine step.  The stage-1 step is also checked
against the reference's own float64 gradients (tests/golden/ref_grads_rsf.npz).

Bounds are per case, at most 3x the worst value measured on an H100 80GB HBM3 (700 W); run with -s to print the
measured values.
"""
import types

import pytest
import torch

import grad_replay as R
from conftest import default_weights, load_golden
from oracle import pvraft_oracle as O
from train_helpers import randomise_affine

pytestmark = pytest.mark.gpu

CASES = {
    'default':  dict(b=2, n1=1024, n2=1024, k=128, iters=3, trained=False),
    'trained':  dict(b=2, n1=1024, n2=1024, k=128, iters=3, trained=True),
    'straddle': dict(b=3, n1=1004, n2=1004, k=128, iters=3, trained=True),
    'unequal':  dict(b=2, n1=1024, n2=1536, k=128, iters=3, trained=True),
    'bench':    dict(b=2, n1=8192, n2=8192, k=512, iters=8, trained=False),
}
# Per case: the worst relative L2 over every parameter gradient except the PReLU slopes and both input gradients, both
# losses and both forms; the worst relative L2 of the flows (the refined flow).  Measured on an H100 80GB HBM3 (700 W),
# worst of two runs: default 4.5e-6, trained 4.6e-6, straddle 4.3e-6, unequal 4.4e-6, bench 9.8e-6, refine 2.1e-6;
# flows 3.2e-6 (N <= 1536), 6.5e-6 (bench); refined 5.0e-7.
BOUND = {'default': 1.3e-5, 'trained': 1.3e-5, 'straddle': 1.2e-5, 'unequal': 1.3e-5, 'bench': 2.9e-5, 'refine': 6e-6}
BOUND_FLOWS = {'default': 9e-6, 'trained': 9e-6, 'straddle': 9e-6, 'unequal': 9e-6, 'bench': 1.9e-5, 'refine': 1.5e-6}
# The PReLU slopes (corr_block.out_conv.2, knn_conv.2): each gradient is sum dy * t over t < 0, which cancels -- knn_conv.2's
# relative L2 reaches 1.1e-4 (N1 = 1024, N2 = 1536) while every other tensor stays below 1e-5.  They are bounded by
# |error| / (the float64 sum |dy * t| of their terms): measured 2.5e-8.
BOUND_SLOPE = 7e-8
# The library against the reference's float64 gradients (N = 256), through the fixture's sketches: every tensor but
# knn_conv.2 within 1.3e-6 (measured); knn_conv.2, the cancelling sum above and kept whole, 7.5e-5.
BOUND_FIXTURE, BOUND_FIXTURE_SLOPE = 3.8e-6, 2e-4


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


class det_mode:
    def __init__(self, flag):
        self.flag = flag

    def __enter__(self):
        self.was, self.warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
        torch.use_deterministic_algorithms(self.flag)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.was, warn_only=self.warn)
        return False


def clouds(b, n1, n2, seed):
    """pc1 in a 4 m box (dense enough for non-empty cells at every level); pc2 = pc1 moved by 0.1 N(0,1) plus n2 - n1 more
    points in the same box."""
    g = torch.Generator().manual_seed(seed)
    pc1 = 4.0 * torch.rand(b, n1, 3, generator=g)
    pc2 = pc1 + 0.1 * torch.randn(b, n1, 3, generator=g)
    if n2 > n1:
        pc2 = torch.cat([pc2, 4.0 * torch.rand(b, n2 - n1, 3, generator=g)], 1)
    return pc1, pc2


def model_for(cls, k, trained, seed=2):
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    m = cls(args)
    m.load_state_dict(default_weights(refine=cls.__name__ == 'RSF_refine', args=args, seed=seed))
    if trained:
        randomise_affine(m, 7, (-0.3, 1.7))
    return m


def library_grads(m, inputs, losses, det, run):
    """run(m, *inputs) under the recorder, then the gradient of each loss w.r.t. the parameters and the inputs that
    require grad -> (output, Decisions, [grads])."""
    with det_mode(det), R.record_library(m, inputs[0], inputs[1]) as d:
        out = run(m, *inputs)
    named = [(k, p) for k, p in m.named_parameters() if p.requires_grad]
    named += [(n, x) for n, x in zip(('xyz1', 'xyz2'), inputs) if x.requires_grad]
    res = []
    for i, fn in enumerate(losses):
        with det_mode(det):
            g = torch.autograd.grad(fn(out), [t for _, t in named], retain_graph=i + 1 < len(losses), allow_unused=True)
        res.append({k: (torch.zeros_like(t) if gv is None else gv) for (k, t), gv in zip(named, g)})
    out = [f.detach() for f in out] if isinstance(out, list) else out.detach()
    return out, d, res


def report(tag, errs):
    top = R.worst(errs, 4)
    print(f'{tag}: worst relative L2 ' + ', '.join(f'{k} {v:.2e}' for k, v in top))
    return top[0][1]


@pytest.mark.parametrize('det', [False, True], ids=['default', 'DET'])
@pytest.mark.parametrize('case', list(CASES))
def test_stage1_gradients_match_float64_replay(dev, case, det):
    from pvraft_b200 import RSF
    c = CASES[case]
    m = model_for(RSF, c['k'], c['trained']).to(dev).train()
    W = {k: v.detach().clone() for k, v in m.state_dict().items()}
    pc1, pc2 = clouds(c['b'], c['n1'], c['n2'], seed=c['n1'] + c['n2'] + c['b'])
    pc1, pc2 = pc1.to(dev), pc2.to(dev)
    gt = pc2[:, :c['n1']] - pc1
    g = torch.Generator().manual_seed(5)
    G = [torch.randn(c['b'], c['n1'], 3, generator=g, dtype=torch.float64).to(dev) for _ in range(c['iters'])]
    flows, d, got = library_grads(m, (pc1.clone().requires_grad_(True), pc2.clone().requires_grad_(True)),
                                  [lambda f: R.linear_loss(f, G), lambda f: R.sequence_loss(f, gt)], det,
                                  lambda m, x1, x2: m([x1, x2], num_iters=c['iters']))
    assert len(got[0]) == 95 + 2
    signs = [torch.sign(f - gt) for f in flows]
    del m
    torch.cuda.empty_cache()
    ref_flows, want, scales = R.replay_rsf(W, pc1, pc2, d, c['iters'], 3, 0.25, c['k'],
                                           [lambda f, *_: R.linear_loss(f, G), lambda f, *_: R.sequence_loss(f, gt, signs)], dev)
    assert not d.unused(), d.unused()
    e_f = max(float((f.double() - r).norm() / r.norm()) for f, r in zip(flows, ref_flows))
    worst = worst_slope = 0.0
    for loss, gg, ww, sc in zip(('linear', 'l1'), got, want, scales):
        errs = R.rel_l2(gg, ww)
        slope = {k: float((gg[k].double() - ww[k]).abs().sum()) / sc[k] for k in R.PRELU_SLOPE.values()}
        tag = f'{case} {"DET" if det else "default"} {loss} (flows {e_f:.1e})'
        worst = max(worst, report(tag, {k: v for k, v in errs.items() if k not in slope}))
        print(f'{tag}: PReLU slopes, error / sum |dy t|: ' + ', '.join(f'{k} {v:.2e} (relative L2 {errs[k]:.2e})' for k, v in slope.items()))
        worst_slope = max(worst_slope, *slope.values())
    assert e_f < BOUND_FLOWS[case], e_f
    assert worst < BOUND[case], worst
    assert worst_slope < BOUND_SLOPE, worst_slope


@pytest.mark.parametrize('det', [False, True], ids=['default', 'DET'])
def test_refine_gradients_match_float64_replay(dev, det):
    """Stage 2: the loop under no_grad on the fused kernels, the refiner with gradients; its 29 parameters and d xyz1."""
    from pvraft_b200 import RSF_refine
    b, n, k, iters = 2, 1024, 128, 3
    m = model_for(RSF_refine, k, True, seed=4).to(dev).train()
    W = {kk: v.detach().clone() for kk, v in m.state_dict().items()}
    for kk, p in m.named_parameters():
        p.requires_grad_(kk.startswith('refine_block.'))
    pc1, pc2 = (t.to(dev) for t in clouds(b, n, n, seed=21))
    gt = pc2 - pc1
    G = torch.randn(b, n, 3, generator=torch.Generator().manual_seed(6), dtype=torch.float64).to(dev)
    refined, d, got = library_grads(m, (pc1.clone().requires_grad_(True), pc2.clone()),
                                    [lambda r: (r * G).sum(), lambda r: (r - gt).abs().sum(-1).mean()], det,
                                    lambda m, x1, x2: m([x1, x2], iters))
    assert len(got[0]) == 29 + 1
    signs = torch.sign(refined - gt)
    ref, want = R.replay_refine(W, pc1, pc2, d, [lambda r, *_: (r * G).sum(), lambda r, *_: (signs * (r - gt)).sum(-1).mean()], dev)
    e_f = float((refined.double() - ref).norm() / ref.norm())
    worst = 0.0
    for loss, gg, ww in zip(('linear', 'l1'), got, want):
        worst = max(worst, report(f'refine {"DET" if det else "default"} {loss} (refined {e_f:.1e})', R.rel_l2(gg, ww)))
    assert e_f < BOUND_FLOWS['refine'], e_f
    assert worst < BOUND['refine'], worst


def test_stage1_gradients_match_the_reference(dev):
    """The library against the reference's own float64 gradients (fixture 1's weights and clouds, the sequence loss), and
    its decisions against the reference's: the same kNN sets and top-K ids."""
    from pvraft_b200 import RSF
    arrays, weights = load_golden('small_rsf_refine.npz')
    want, z = R.reference_gradients('ref_grads_rsf.npz')
    m = RSF(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=64))
    m.load_state_dict({k: v for k, v in weights.items() if not k.startswith('refine_block.')})
    m = m.to(dev).train()
    pc1, pc2 = arrays['pc1'].to(dev), arrays['pc2'].to(dev)
    _, d, (got,) = library_grads(m, (pc1.clone().requires_grad_(True), pc2.clone().requires_grad_(True)),
                                 [lambda f: R.sequence_loss(f, pc2 - pc1)], False,
                                 lambda m, x1, x2: m([x1, x2], num_iters=3))
    for cloud, key in (('pc1', 'nbr1'), ('pc2', 'nbr2')):
        assert torch.equal(d.rec[('graph', cloud)].sort(-1).values.cpu(), z[key].long().sort(-1).values)
    assert torch.equal(d.rec[('topk', '12')].sort(-1).values.cpu(), z['topk'].long().sort(-1).values)
    errs = R.sketched_rel_l2(got, want)          # (estimates within 1 +- 0.2 for tensors of more than 128 elements)
    slope = 'corr_block.knn_conv.2.weight'
    worst = report('library vs reference float64', {k: v for k, v in errs.items() if k != slope})
    print(f'library vs reference float64: {slope} {errs[slope]:.2e}')
    assert worst < BOUND_FIXTURE, worst
    assert errs[slope] < BOUND_FIXTURE_SLOPE, errs[slope]
