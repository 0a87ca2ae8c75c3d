"""The gradient oracle pinned to the reference's own autograd (CPU).

tests/golden/ref_grads_rsf.npz and ref_grads_refine.npz hold float64 gradients of the unmodified reference with fixture
1's weights and clouds (B = 2, N = 256, K = 64, 3 iterations; tests/golden/make_golden.py): all 95 parameter gradients
of an RSF step under the sequence loss with d xyz1 and d xyz2, and the 29 refine_block gradients of an RSF_refine step
under the refined flow's L1 error with d xyz1.  Tensors of more than 128 elements are kept as a fixed 128-row random
sketch, so their relative L2 errors are estimates within a factor 1 +- 0.2 (grad_replay.sketched_rel_l2); smaller ones
(the PReLU slopes, most GroupNorm affines) whole.  Three things are checked against them:
  * the fixture's discrete decisions (both clouds' kNN adjacency, the top-K ids) equal the fp32 oracle's;
  * autograd through the fp32 oracle is within a few fp32 rounding errors per tensor (measured worst values beside the
    bounds; corr_block.knn_conv.2.weight, a PReLU slope whose gradient is a cancelling sum, is the largest);
  * the float64 oracle replaying the fp32 oracle's decisions (tests/grad_replay.py) matches to 1e-10: the replay's
    arithmetic is the reference's, so what the GPU replay tests measure is the library's error alone.
"""
import pytest
import torch

import grad_replay as R
from conftest import load_golden
from oracle import pvraft_oracle as O

K, ITERS, BASE = 64, 3, 0.25


@pytest.fixture(scope='module')
def fixture1():
    arrays, weights = load_golden('small_rsf_refine.npz')
    return arrays['pc1'], arrays['pc2'], weights


def leaf(t, dtype, grad=True):
    return t.detach().to(dtype).clone().requires_grad_(grad)


def oracle_rsf_step(W, pc1, pc2, dtype, mode, d):
    P = {k: leaf(v, dtype) for k, v in W.items() if not k.startswith('refine_block.')}
    x1, x2 = leaf(pc1, dtype), leaf(pc2, dtype)
    with R.oracle_decisions(d, x1, x2, BASE, mode):
        flows = O.rsf_forward(P, x1, x2, ITERS, 3, BASE, K)
    R.sequence_loss(flows, x2.detach() - x1.detach()).backward()
    return dict({k: v.grad for k, v in P.items()}, xyz1=x1.grad, xyz2=x2.grad)


def oracle_refine_step(W, pc1, pc2, dtype, mode, d):
    P = {k: leaf(v, dtype, k.startswith('refine_block.')) for k, v in W.items()}
    x1, x2 = leaf(pc1, dtype), leaf(pc2, dtype, False)
    with R.oracle_decisions(d, x1, x2, BASE, mode):
        with torch.no_grad():                                   # RAFTSceneFlowRefine.py:23
            li = O.prepare(P, x1, x2, K)
            flow = O.raft_loop(P, li, x1, ITERS, 3, BASE)[-1]
        refined = O.flot_refine(P, 'refine_block', flow + (x1.detach() - x1), li.feat_graph)
    (refined - (x2 - x1.detach())).abs().sum(-1).mean().backward()
    return dict({k: v.grad for k, v in P.items() if v.requires_grad}, xyz1=x1.grad)


def errors(got, name):
    want, _ = R.reference_gradients(name)
    assert set(got) == set(want), set(got) ^ set(want)
    return R.sketched_rel_l2(got, want)


def test_reference_decisions_equal_the_fp32_oracle(fixture1):
    pc1, pc2, W = fixture1
    _, g = R.reference_gradients('ref_grads_rsf.npz')
    d = R.Decisions()
    oracle_rsf_step(W, pc1, pc2, torch.float32, 'record', d)
    for cloud, key in (('pc1', 'nbr1'), ('pc2', 'nbr2')):
        assert torch.equal(d.rec[('graph', cloud)].sort(-1).values, g[key].long().sort(-1).values), cloud
    assert torch.equal(d.rec[('topk', '12')].sort(-1).values, g['topk'].long().sort(-1).values)


def test_fp32_oracle_gradients_match_the_reference(fixture1):
    pc1, pc2, W = fixture1
    e = errors(oracle_rsf_step(W, pc1, pc2, torch.float32, 'record', R.Decisions()), 'ref_grads_rsf.npz')
    slopes = ('corr_block.knn_conv.2.weight', 'corr_block.out_conv.2.weight')
    print('fp32 oracle vs reference, RSF step:', R.worst(e))
    # measured over runs (CPU threads change the summation order): the PReLU slopes, cancelling sums, 1.2e-6 .. 7.0e-6;
    # every other parameter <= 1.2e-6; d xyz1 1.8e-7, d xyz2 5.0e-7
    assert max(e[k] for k in slopes) < 2e-5, [(k, e[k]) for k in slopes]
    assert max(v for k, v in e.items() if k not in slopes + ('xyz1', 'xyz2')) < 3e-6, R.worst(e)
    assert max(e['xyz1'], e['xyz2']) < 1.5e-6, (e['xyz1'], e['xyz2'])
    e = errors(oracle_refine_step(W, pc1, pc2, torch.float32, 'record', R.Decisions()), 'ref_grads_refine.npz')
    print('fp32 oracle vs reference, refine step:', R.worst(e))
    assert max(e.values()) < 4e-6, R.worst(e)                          # measured 1.5e-6 (d xyz1 8.1e-7)


@pytest.mark.parametrize('step', ['rsf', 'refine'])
def test_float64_replay_matches_the_reference(fixture1, step):
    """Decisions recorded from the fp32 oracle, replayed in float64: every gradient within 1e-10 of the reference's."""
    pc1, pc2, W = fixture1
    run = oracle_rsf_step if step == 'rsf' else oracle_refine_step
    d = R.Decisions()
    run(W, pc1, pc2, torch.float32, 'record', d)
    got = run(W, pc1, pc2, torch.float64, 'replay', d)
    assert not d.unused(), d.unused()
    assert all(n == 1 for k, n in d.hits.items() if k[0] != 'graph'), d.hits
    e = errors(got, f'ref_grads_{step}.npz')
    print(f'float64 replay vs reference, {step} step:', R.worst(e))
    assert max(e.values()) < 1e-10, R.worst(e)
