"""The decision replay of the self-supervised training steps, checked on the host before any GPU time is spent on it.

tests/test_gpu_grad_replay_losses.py replays the library's decisions in float64: the model's, per direction, and the
self-supervised loss's own neighbour searches.  Here the fp32 CPU oracle takes the place of the library (B = 2, N = 256,
K = 64, 2 iterations, fixture 1's weights and clouds): its decisions are recorded per direction, the loss's neighbours
come from float64 searches on its flows, and the float64 oracle replays them, for the one-direction three-term loss and
for the bidirectional four-term pair loss.  Every oracle call has to find its record and every record has to be read,
so this shows that grad_replay routes every call of both directions and of the loss.
"""
import pytest
import torch

import grad_replay as R
import losses64 as L
from conftest import load_golden
from oracle import pvraft_oracle as O

K, ITERS, BASE = 64, 2, 0.25
LOSS = {'three_term': dict(wl=0.3), 'pair': dict(wl=0.3, wcons=0.3)}
# The float64 replay against fp32 autograd through the same decisions: relative L2 of every tensor but the PReLU slopes,
# measured 7.0e-6 (three_term) and 3.6e-6 (pair), a few fp32 roundings of the 95-parameter step; the slopes, whose
# gradients are cancelling sums, as |error| / sum |dy t| (grad_replay.PRELU_SLOPE): 8.4e-8 and 3.8e-9.
BOUND, BOUND_SLOPE = 2e-5, 5e-7


@pytest.fixture(scope='module')
def fixture1():
    arrays, weights = load_golden('small_rsf_refine.npz')
    return arrays['pc1'], arrays['pc2'], {k: v for k, v in weights.items() if not k.startswith('refine_block.')}


def knn64(p, k):
    """The k nearest points of every point of p [B,N,3] (itself included), in float64."""
    d = ((p[:, :, None, :] - p[:, None, :, :]) ** 2).sum(-1)
    return d.topk(k, -1, largest=False).indices


def record_loss(d, flows, x1, x2, pair, k=9, k_lap=10, k_int=5, k_cons=3):
    """The loss's decisions from float64 searches on the flows, under the keys record_library gives the library's."""
    x1, x2 = x1.detach().double(), x2.detach().double()
    dirs = [('12', flows[0], x1, x2), ('21', flows[1], x2, x1)] if pair else [('12', flows, x1, x2)]
    for dr, fs, pa, pb in dirs:
        ca, cb = ('pc1', 'pc2') if dr == '12' else ('pc2', 'pc1')
        for cloud, p, kk in ((ca, pa, k), (ca, pa, k_lap), (cb, pb, k_lap)):
            d.put_same(('knn', cloud, kk), knn64(p, kk))
        w = torch.cat([pa + f.detach().double() for f in fs])            # [n*B,N,3]: sample i*B + b, as one launch
        ab, ba = L.nn64_indices(w, pb)
        d.put(('nn_ab', dr), ab)
        d.put(('nn_ba', dr), ba)
        d.put(('lap', dr), L.nn64_knearest(w, pb, k_int))
        if pair:
            d.put(('cons', dr), L.nn64_knearest(w, pb, k_cons))


def step(W, pc1, pc2, dtype, mode, d, case):
    """One RSF step under the case's loss (both directions for 'pair') -> every gradient and the PReLU slopes' sum |dy t|."""
    pair = case == 'pair'
    P = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in W.items()}
    x1, x2 = (t.detach().to(dtype).clone().requires_grad_(True) for t in (pc1, pc2))
    terms = {}
    with R.oracle_decisions(d, x1, x2, BASE, mode, terms):
        flows = O.rsf_forward(P, x1, x2, ITERS, 3, BASE, K)
    if pair:
        with R.oracle_decisions(d, x1, x2, BASE, mode, terms, direction='21'):
            flows = (flows, O.rsf_forward(P, x2, x1, ITERS, 3, BASE, K))
    if mode == 'record':
        record_loss(d, flows, x1, x2, pair)
    R.self_supervised64(d, flows, x1, x2, **LOSS[case]).backward()
    return dict({k: v.grad for k, v in P.items()}, xyz1=x1.grad, xyz2=x2.grad), terms


@pytest.mark.parametrize('case', list(LOSS))
def test_float64_replay_matches_fp32_autograd(fixture1, case):
    pc1, pc2, W = fixture1
    d = R.Decisions()
    got, _ = step(W, pc1, pc2, torch.float32, 'record', d, case)
    want, terms = step(W, pc1, pc2, torch.float64, 'replay', d, case)
    assert not d.unused(), d.unused()
    dirs = ('12', '21') if case == 'pair' else ('12',)
    assert {k[-1] for k in d.rec if k[0] in ('topk', 'nn_ab', 'nn_ba', 'lap', 'cons')} == set(dirs)
    errs = R.rel_l2(got, want)
    slope = {k: float((got[k].double() - want[k]).abs().sum()) / terms[k] for k in R.PRELU_SLOPE.values()}
    print(f'{case}: fp32 oracle vs float64 replay', R.worst({k: v for k, v in errs.items() if k not in slope}), slope)
    assert max(v for k, v in errs.items() if k not in slope) < BOUND, R.worst(errs)
    assert max(slope.values()) < BOUND_SLOPE, slope
    assert min(float(v.norm()) for v in want.values()) > 0


@pytest.mark.parametrize('case', list(LOSS))
def test_float64_record_then_replay_gives_the_same_bits(fixture1, case):
    pc1, pc2, W = fixture1
    d = R.Decisions()
    recorded, _ = step(W, pc1, pc2, torch.float64, 'record', d, case)
    replayed, _ = step(W, pc1, pc2, torch.float64, 'replay', d, case)
    assert not d.unused(), d.unused()
    for k, v in recorded.items():
        assert torch.equal(v, replayed[k]), (k, float((v - replayed[k]).abs().max()))
