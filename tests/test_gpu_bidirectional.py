"""The flow in both directions in one forward (model(p, n, bidirectional=True)): under deterministic mode each direction is
bitwise its one-direction call, eager and replayed, for RSF and RSF_refine and in every precision mode; within the parity
tolerance elsewhere; and training through it with the forward-backward consistency term."""
import types

import pytest
import torch

from conftest import default_weights, rel_err
import unequal_oracle as U
from losses64 import graphs, pair_loss64
from test_gpu_laplacian import leaf, same_bits
from train_helpers import compare_grads, oracle_adjacency

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture
def det():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def model(dev, refine=False, k=64, seed=0):
    from pvraft_b200 import RSF, RSF_refine
    torch.manual_seed(seed)
    return (RSF_refine if refine else RSF)(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)).to(dev).eval()


def pair(dev, b, n1, n2, seed=0):
    g = torch.Generator().manual_seed(seed)
    x1 = torch.rand(b, n1, 3, generator=g) * 4
    x2 = torch.rand(b, n2, 3, generator=g) * 4 + torch.tensor([0.1, 0.0, -0.05])
    return x1.to(dev), x2.to(dev)


def flat(out):
    return [out] if torch.is_tensor(out) else list(out)


def check_bitwise(m, x1, x2, iters, graph):
    m.use_cuda_graph = graph
    with torch.no_grad():
        fwd, bwd = m([x1, x2], iters, bidirectional=True)
        one, rev = m([x1, x2], iters), m([x2, x1], iters)
    for a, b in zip(flat(fwd) + flat(bwd), flat(one) + flat(rev)):
        assert a.shape == b.shape and same_bits(a, b)


@pytest.mark.parametrize('refine', [False, True])
@pytest.mark.parametrize('b', [1, 2])
@pytest.mark.parametrize('n1,n2', [(1024, 1024), (8192, 8192), (4096, 6144)])
@pytest.mark.parametrize('graph', [False, True])
def test_bitwise_contract(dev, det, refine, b, n1, n2, graph):
    x1, x2 = pair(dev, b, n1, n2, seed=n1 + b)
    check_bitwise(model(dev, refine), x1, x2, 3, graph)


@pytest.mark.parametrize('mode', ['bf16', 'bf16-compute', 'bf16-mixed'])
@pytest.mark.parametrize('refine', [False, True])
def test_bitwise_contract_in_every_precision_mode(dev, det, mode, refine):
    """The 2B stack (equal sizes, eager and replayed) and one pair of different sizes; the bf16 state takes K >= 128."""
    for (n1, n2), graph in (((1024, 1024), False), ((1024, 1024), True), ((2048, 3072), False)):
        x1, x2 = pair(dev, 2, n1, n2, seed=3)
        check_bitwise(model(dev, refine, k=128).set_precision(mode), x1, x2, 3, graph)


@pytest.mark.parametrize('refine', [False, True])
def test_parity_at_1000_points(dev, refine):
    x1, x2 = pair(dev, 2, 1000, 1000, seed=9)
    m = model(dev, refine)
    with torch.no_grad():
        fwd, bwd = m([x1, x2], 4, bidirectional=True)
        one, rev = m([x1, x2], 4), m([x2, x1], 4)
    for a, r in zip(flat(fwd) + flat(bwd), flat(one) + flat(rev)):
        assert float((a - r).abs().mean()) < 2e-3 * float(r.abs().mean())


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_data_parallel(dev):
    m = model(dev)
    x1, x2 = pair(dev, 2, 1024, 1024, seed=4)
    with torch.no_grad():
        want = m([x1, x2], 3, bidirectional=True)
        got = torch.nn.DataParallel(m, device_ids=[0, 1])([x1, x2], 3, bidirectional=True)
    for a, r in zip(got[0] + got[1], want[0] + want[1]):
        assert float((a - r).abs().mean()) < 2e-3 * float(r.abs().mean())


# ---- training --------------------------------------------------------------------------------------------------------------
def loss_of(m, x1, x2, iters, w_cons):
    from pvraft_b200.loss import sequence_self_supervised_loss
    out = m([x1, x2], iters, bidirectional=True)
    return sequence_self_supervised_loss(out, {'sequence': [x1, x2]}, w_laplacian=0.3, w_consistency=w_cons)


def test_training_step_reaches_every_parameter_and_both_clouds(dev):
    m = model(dev).train()
    x1, x2 = pair(dev, 2, 1024, 1024, seed=2)
    x1, x2 = x1.requires_grad_(True), x2.requires_grad_(True)
    loss_of(m, x1, x2, 3, 0.3).backward()
    grads = [q.grad for q in m.parameters() if q.requires_grad]
    assert len(grads) == 95 and all(g is not None and torch.isfinite(g).all() for g in grads)
    assert x1.grad.abs().sum() > 0 and x2.grad.abs().sum() > 0


def test_training_gradients_match_two_one_direction_forwards(dev):
    """The stacked training forward against two one-direction training forwards of the same model: all 95 parameter
    gradients and both input gradients.  (The loss itself is checked against float64 by the oracle tests below.)"""
    from pvraft_b200.loss import sequence_self_supervised_loss
    x1, x2 = pair(dev, 2, 1024, 1024, seed=6)
    grads = []
    for stacked in (True, False):
        m = model(dev, seed=1).train()
        a, b = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
        out = m([a, b], 3, bidirectional=True) if stacked else (m([a, b], 3), m([b, a], 3))
        sequence_self_supervised_loss(out, {'sequence': [a, b]}, w_laplacian=0.3, w_consistency=0.3).backward()
        grads.append([q.grad for q in m.parameters()] + [a.grad, b.grad])
    for g1, g2 in zip(*grads):
        assert float((g1 - g2).norm() / g2.norm().clamp_min(1e-30)) < 1e-3


def test_pair_loss_with_zero_consistency_is_the_mean_of_both_directions(dev):
    from pvraft_b200.loss import sequence_self_supervised_loss
    x1, x2 = pair(dev, 2, 1024, 1280, seed=8)
    m = model(dev)
    with torch.no_grad():
        fwd, bwd = m([x1, x2], 3, bidirectional=True)
        both = sequence_self_supervised_loss((fwd, bwd), {'sequence': [x1, x2]})
        a = sequence_self_supervised_loss(fwd, {'sequence': [x1, x2]})
        b = sequence_self_supervised_loss(bwd, {'sequence': [x2, x1]})
    assert torch.allclose(both, (a + b) / 2, rtol=1e-6)


def test_captured_step_equals_eager_bitwise(dev, det):
    from pvraft_b200 import train as T
    was = T._TC_TRAIN
    T._TC_TRAIN = '1'
    try:
        m = model(dev).train()
        x1, x2 = pair(dev, 1, 1024, 1024, seed=12)

        def step():
            m.zero_grad(set_to_none=False)
            loss = loss_of(m, x1, x2, 2, 0.3)
            loss.backward()
            return [loss.detach().clone()] + [q.grad.clone() for q in m.parameters()]

        for q in m.parameters():
            q.grad = torch.zeros_like(q)
        eager = step()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            step()
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            static = step()
        g.replay()
        torch.cuda.synchronize()
        assert all(same_bits(a, b) for a, b in zip(eager, static))
    finally:
        T._TC_TRAIN = was


def test_adam_lowers_the_four_term_loss(dev):
    m = model(dev).train()
    x1, _ = pair(dev, 1, 1024, 1024, seed=13)
    x2 = x1 @ torch.tensor([[0.995, -0.0998, 0.0], [0.0998, 0.995, 0.0], [0.0, 0.0, 1.0]], device=dev) + 0.2   # a rigid motion
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    losses = []
    for _ in range(12):
        opt.zero_grad()
        loss = loss_of(m, x1, x2, 2, 0.3)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < 0.8 * losses[0], losses


# ---- against the oracle and float64 ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('n1,n2', [(1024, 1024), (1024, 1280)])
def test_rsf_gradients_match_oracle(dev, n1, n2):
    """A 3-iteration stage-1 step with a bidirectional forward and the four-term pair loss (w_laplacian = w_consistency =
    0.3) against autograd through two oracle forwards ([pc1, pc2] and [pc2, pc1]) plus the float64 loss: all 95 parameter
    gradients, with the bounds of test_gpu_laplacian.py::test_rsf_gradients_match_oracle."""
    from pvraft_b200 import RSF
    from pvraft_b200.loss import sequence_self_supervised_loss
    b, k, iters = 2, 128, 3
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    W = default_weights(args=args, seed=2)
    g = torch.Generator().manual_seed(n1 + n2)
    pc1 = 4.0 * torch.rand(b, n1, 3, generator=g)
    pc2 = 4.0 * torch.rand(b, n2, 3, generator=g) + torch.tensor([0.1, 0.0, -0.05])
    Wr = {kk: leaf(v) for kk, v in W.items()}
    ref12 = U.rsf_forward(Wr, pc1, pc2, iters, 3, 0.25, k)
    ref21 = U.rsf_forward(Wr, pc2, pc1, iters, 3, 0.25, k)
    want_loss = pair_loss64(ref12, ref21, pc1, pc2, dev)
    want_loss.backward()
    want = {kk: v.grad for kk, v in Wr.items()}
    m = RSF(args)
    m.load_state_dict(W)
    m = m.to(dev).train()
    with oracle_adjacency():
        fwd, bwd = m([pc1.to(dev), pc2.to(dev)], num_iters=iters, bidirectional=True)
    for f, fr in zip(fwd + bwd, ref12 + ref21):
        assert f.shape == fr.shape
        assert float((f.detach().cpu() - fr.detach()).abs().mean()) < 1e-4 * float(fr.detach().abs().mean())
    loss = sequence_self_supervised_loss((fwd, bwd), {'sequence': [pc1.to(dev), pc2.to(dev)]}, w_laplacian=0.3, w_consistency=0.3)
    assert abs(float(loss.detach()) - float(want_loss.detach())) < 1e-4 * abs(float(want_loss.detach()))
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters()}
    assert len(got) == 95 and all(v is not None for v in got.values())
    compare_grads(got, want, 2e-2, 5e-2)


def test_pair_loss_input_gradients_against_float64(dev):
    """The pair loss alone, clouds of different sizes: its value and its gradients into both flow sequences and both clouds
    against float64 autograd, the interpolation neighbours taken from the kernels."""
    from pvraft_b200 import ops
    from pvraft_b200.loss import sequence_self_supervised_loss
    b, n1, n2, n_pred, k_int, k_cons = 2, 900, 1100, 3, 4, 2
    gen = torch.Generator().manual_seed(6)
    p1, p2 = torch.rand(b, n1, 3, generator=gen) * 4, torch.rand(b, n2, 3, generator=gen) * 4
    f12 = [torch.randn(b, n1, 3, generator=gen) * 0.2 for _ in range(n_pred)]
    f21 = [torch.randn(b, n2, 3, generator=gen) * 0.2 for _ in range(n_pred)]
    p1d, p2d = leaf(p1, dev), leaf(p2, dev)
    f12d, f21d = [leaf(f, dev) for f in f12], [leaf(f, dev) for f in f21]
    kw = dict(gamma=0.7, w_chamfer=2.0, w_smooth=0.5, w_laplacian=0.7, k_int=k_int, w_consistency=1.3, k_cons=k_cons)
    loss = sequence_self_supervised_loss((f12d, f21d), {'sequence': [p1d, p2d]}, **kw)
    loss.backward()

    lap_idx, cons_idx = [], []
    for fs, fo, pa, pb in ((f12d, f21d, p1d, p2d), (f21d, f12d, p2d, p1d)):
        pa, pb = pa.detach(), pb.detach()
        g1, g2 = graphs(pa, pb, 10)
        l2 = ops.cloud_laplacian(pb, g2)
        lap_idx.append([ops.laplacian((pa + f).detach().contiguous(), pb, l2, g1, k_int)[1].long().cpu() for f in fs])
        cons_idx.append([ops.flow_consistency((pa + f).detach().contiguous(), f.detach().contiguous(), pb, r.detach().contiguous(),
                                              k_cons, 0.0, 0.0)[1].long().cpu() for f, r in zip(fs, fo)])
    p164, p264 = leaf(p1.double()), leaf(p2.double())
    f1264, f2164 = [leaf(f.double()) for f in f12], [leaf(f.double()) for f in f21]
    want = pair_loss64(f1264, f2164, p164, p264, dev, gamma=0.7, wc=2.0, ws=0.5, wl=0.7, wcons=1.3, k_int=k_int, k_cons=k_cons,
                       lap_idx=lap_idx, cons_idx=cons_idx)
    want.backward()
    assert abs(float(loss.detach()) - float(want.detach())) <= 1e-6 * abs(float(want.detach()))
    assert rel_err(p1d.grad.cpu(), p164.grad) <= 1e-5 and rel_err(p2d.grad.cpu(), p264.grad) <= 1e-5
    for a, r in zip(f12d + f21d, f1264 + f2164):
        assert rel_err(a.grad.cpu(), r.grad) <= 1e-5


@pytest.mark.parametrize('n1,n2', [(1024, 1024), (1024, 1280)])
def test_rsf_refine_training_matches_two_one_direction_calls(dev, n1, n2):
    """RSF_refine's training path with bidirectional=True (the refiner on the 2B stack, or once per direction) against two
    one-direction training calls: the refined flows, the 29 refiner gradients and the gradients into both clouds."""
    from pvraft_b200.loss import self_supervised_loss
    x1, x2 = pair(dev, 2, n1, n2, seed=21)
    outs = []
    for stacked in (True, False):
        m = model(dev, refine=True, seed=3).train()
        a, b = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
        out = m([a, b], 3, bidirectional=True) if stacked else (m([a, b], 3), m([b, a], 3))
        self_supervised_loss(out, {'sequence': [a, b]}, w_laplacian=0.3, w_consistency=0.3).backward()
        grads = {kk: q.grad for kk, q in m.named_parameters() if q.grad is not None}
        assert len(grads) == 29 and all(kk.startswith('refine_block.') for kk in grads)
        outs.append([o.detach() for o in out] + [grads[kk] for kk in sorted(grads)] + [a.grad, b.grad])
    for g1, g2 in zip(*outs):
        assert float(g2.norm()) > 0
        assert float((g1 - g2).norm() / g2.norm()) < 1e-3
