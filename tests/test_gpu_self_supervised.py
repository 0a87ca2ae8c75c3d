"""Self-supervised losses on the device (pvraft_b200/loss.py, csrc/self_supervised.cu): the Chamfer search bit-exact against a
numpy float32 restatement of the difference form, values and gradients against float64 restatements of both losses (kept
here: the reference has no self-supervised loss, and the oracle module restates the reference only), deterministic mode, and
training the model with them.

    C_b = (1/N) sum_i min_j ||W_i - P2_j||^2 + (1/M) sum_j min_i ||W_i - P2_j||^2,   W = P1 + f
    S_b = (1/(N k)) sum_i sum_{j in N_k(i)} ||f_j - f_i||,   N_k(i) = ops.knn(P1, P1, k, mode=0)[i]
    L   = sum_i gamma^(n-i-1) mean_b (w_c C_b(f_i) + w_s S_b(f_i))
"""
import types

import numpy as np
import pytest
import torch

from conftest import default_weights, rel_err
from losses64 import chamfer64, loss64, smooth64
from oracle import pvraft_oracle as O
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


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int64 if t.element_size() == 8 else torch.int32) if t.is_floating_point() else t


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


# ---- host restatements ---------------------------------------------------------------------------------------------------
def nn_host(q, c, dtype):
    """Nearest point of c for every point of q, in `dtype`: (dx*dx + dy*dy) + dz*dz of the differences (numpy rounds each
    operation to nearest and never contracts), lowest index on ties -> (argmin [n], min [n])."""
    q, c = q.astype(dtype), c.astype(dtype)
    arg, best = np.empty(len(q), np.int64), np.empty(len(q), dtype)
    rows = max(1, (1 << 22) // len(c))
    for r0 in range(0, len(q), rows):
        d = q[r0:r0 + rows, None, :] - c[None, :, :]
        dd = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        arg[r0:r0 + rows] = dd.argmin(1)
        best[r0:r0 + rows] = dd.min(1)
    return arg, best


def dist64(q, c, idx):
    d = q.astype(np.float64) - c.astype(np.float64)[idx]
    return (d * d).sum(-1)


# ---- search ----------------------------------------------------------------------------------------------------------------
def clouds(s, b, n, m, seed, shift=0.0, scale=5.0):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(s, n, 3, generator=g) * scale + shift
    bb = torch.rand(b, m, 3, generator=g) * scale + shift
    return a, bb


def check_search(a, b, dev):
    from pvraft_b200 import ops
    acc, nn_ab, nn_ba = ops.chamfer(a.to(dev).contiguous(), b.to(dev).contiguous())
    nn_ab, nn_ba, acc = nn_ab.cpu().numpy(), nn_ba.cpu().numpy(), acc.cpu().numpy()
    for s in range(a.shape[0]):
        an, bn = a[s].numpy(), b[s % b.shape[0]].numpy()
        for q, c, got, col in ((an, bn, nn_ab[s], 0), (bn, an, nn_ba[s], 1)):
            want, best = nn_host(q, c, np.float32)
            assert np.array_equal(got, want), (s, col, int((got != want).sum()))
            # the fp32 minima summed in double
            assert abs(acc[s, col] - best.astype(np.float64).sum()) <= 1e-12 * max(1.0, abs(acc[s, col])) + 1e-9 * best.sum()
            # every pick is within 8 fp32 ulp of the float64 minimum
            _, min64 = nn_host(q, c, np.float64)
            picked = dist64(q, c, got)
            assert np.all(picked - min64 <= 8 * np.spacing(min64.astype(np.float32)).astype(np.float64)), (s, col)


@pytest.mark.parametrize('s,b,n,m', [(4, 2, 1000, 1537), (2, 1, 32, 33), (3, 3, 1537, 1000), (2, 2, 4096, 4096)])
def test_search_bit_exact(dev, s, b, n, m):
    check_search(*clouds(s, b, n, m, seed=n + m), dev)


def test_search_far_from_the_origin(dev):
    """Clouds shifted by 1e3, where the expanded form |q|^2 + |x|^2 - 2 q.x would cancel."""
    a, b = clouds(2, 2, 3000, 2500, seed=5, shift=1e3, scale=20.0)
    check_search(a, b, dev)


def test_search_20000(dev):
    check_search(*clouds(1, 1, 20000, 20000, seed=7, scale=50.0), dev)


def test_search_duplicates_and_exact_ties(dev):
    """Integer coordinates make many distances exactly equal; duplicated points have equal distances to everything."""
    g = torch.Generator().manual_seed(3)
    a = torch.randint(-6, 7, (2, 700, 3), generator=g).float()
    b = torch.randint(-6, 7, (1, 900, 3), generator=g).float()
    b[0, 450:600] = b[0, 0:150]                    # duplicated points of the searched cloud
    a[1, 400:] = a[1, :300].clone()                # duplicated queries
    a[0, :50] = b[0, 10:60]                        # distance 0
    check_search(a, b, dev)


# ---- values and gradients -----------------------------------------------------------------------------------------------------
def leaf(t, dev=None):
    t = t.detach().clone()
    return (t.to(dev) if dev is not None else t).requires_grad_(True)


@pytest.mark.parametrize('k', [1, 9, 32])
@pytest.mark.parametrize('n_pred,b,n,m', [(3, 2, 1000, 1537), (1, 1, 2048, 1024)])
def test_values_and_gradients_against_float64(dev, k, n_pred, b, n, m):
    from pvraft_b200 import ops
    from pvraft_b200.loss import ChamferFn, SmoothFn
    s = n_pred * b
    gen = torch.Generator().manual_seed(k + n)
    p1, p2 = torch.rand(b, n, 3, generator=gen) * 4, torch.rand(b, m, 3, generator=gen) * 4
    f = torch.randn(s, n, 3, generator=gen) * 0.1
    w = (f.view(n_pred, b, n, 3) + p1).reshape(s, n, 3)
    g_c, g_s = torch.rand(s, generator=gen) + 0.5, torch.rand(s, generator=gen) + 0.5
    nbr = ops.knn(p1.to(dev), p1.to(dev), k, mode=0)

    wd, p2d, fd = leaf(w, dev), leaf(p2, dev), leaf(f, dev)
    c = ChamferFn.apply(wd, p2d)
    sm = SmoothFn.apply(fd, nbr)
    ((c * g_c.to(dev)).sum() + (sm * g_s.to(dev)).sum()).backward()
    acc, nn_ab, nn_ba = ops.chamfer(wd.detach(), p2d.detach())

    assert rel_err(c.detach().cpu(), chamfer64(w.double(), p2.double())) <= 1e-6
    w64, p264, f64 = leaf(w.double()), leaf(p2.double()), leaf(f.double())
    nbr64 = nbr.long().cpu()
    assert rel_err(sm.detach().cpu(), smooth64(f64.detach(), nbr64)) <= 1e-6
    ((chamfer64(w64, p264, nn_ab.long().cpu(), nn_ba.long().cpu()) * g_c.double()).sum()
     + (smooth64(f64, nbr64) * g_s.double()).sum()).backward()
    assert rel_err(wd.grad.cpu(), w64.grad) <= 1e-5
    assert rel_err(p2d.grad.cpu(), p264.grad) <= 1e-5
    assert rel_err(fd.grad.cpu(), f64.grad) <= 1e-5


def test_self_edges_give_zero_gradient(dev):
    from pvraft_b200.loss import SmoothFn
    gen = torch.Generator().manual_seed(1)
    f = leaf(torch.randn(2, 300, 3, generator=gen), dev)
    own = torch.arange(300, dtype=torch.int32).view(1, 300, 1).expand(2, 300, 5).contiguous().to(dev)
    v = SmoothFn.apply(f, own)
    v.sum().backward()
    assert torch.equal(v.detach(), torch.zeros_like(v)) and torch.equal(f.grad, torch.zeros_like(f))
    # one self edge among real ones: the same gradient as without it, up to the mean's divisor
    other = torch.randint(0, 300, (2, 300, 4), generator=gen).to(torch.int32).to(dev)
    mixed = torch.cat([own[..., :1], other], -1).contiguous()
    f1, f2 = leaf(f.detach()), leaf(f.detach())
    (SmoothFn.apply(f1, mixed) * 5).sum().backward()
    (SmoothFn.apply(f2, other) * 4).sum().backward()
    assert rel_err(f1.grad.cpu(), f2.grad.cpu()) <= 1e-6


def test_one_launch_equals_separate_calls(dev, det):
    """S = n B samples in one launch give what n calls of B samples give (bitwise in deterministic mode)."""
    from pvraft_b200 import ops
    n_pred, b, n, m, k = 3, 2, 1500, 1200, 9
    gen = torch.Generator().manual_seed(9)
    p1, p2 = (torch.rand(b, n, 3, generator=gen) * 3).to(dev), (torch.rand(b, m, 3, generator=gen) * 3).to(dev)
    f = (torch.randn(n_pred * b, n, 3, generator=gen) * 0.2).to(dev)
    w = (f.view(n_pred, b, n, 3) + p1).reshape(-1, n, 3).contiguous()
    g = torch.rand(n_pred * b, generator=gen).to(dev)
    nbr = ops.knn(p1, p1, k, mode=0)
    acc, ab, ba = ops.chamfer(w, p2)
    sm = ops.flow_smooth(f, nbr)
    da, _ = ops.chamfer_bwd(w, p2, ab, ba, g, want_db=False)
    df = ops.flow_smooth_bwd(f, nbr, g)
    for i in range(n_pred):
        sl = slice(i * b, (i + 1) * b)
        acc_i, ab_i, ba_i = ops.chamfer(w[sl].contiguous(), p2)
        assert torch.equal(ab_i, ab[sl]) and torch.equal(ba_i, ba[sl]) and same_bits(acc_i, acc[sl])
        assert same_bits(ops.flow_smooth(f[sl].contiguous(), nbr), sm[sl])
        da_i, _ = ops.chamfer_bwd(w[sl].contiguous(), p2, ab_i, ba_i, g[sl].contiguous(), want_db=False)
        assert same_bits(da_i, da[sl])
        assert same_bits(ops.flow_smooth_bwd(f[sl].contiguous(), nbr, g[sl].contiguous()), df[sl])


# ---- deterministic mode --------------------------------------------------------------------------------------------------------
def _loss_step(dev, seed=2, n_pred=3, b=2, n=3000, m=2600):
    from pvraft_b200.loss import sequence_self_supervised_loss
    gen = torch.Generator().manual_seed(seed)
    p1 = leaf(torch.rand(b, n, 3, generator=gen) * 10 - 5, dev)
    p2 = leaf(torch.rand(b, m, 3, generator=gen) * 10 - 5, dev)
    flows = [leaf(torch.randn(b, n, 3, generator=gen) * 0.3, dev) for _ in range(n_pred)]

    def run():
        for t in [p1, p2] + flows:
            t.grad = None
        loss = sequence_self_supervised_loss(flows, {'sequence': [p1, p2]})
        loss.backward()
        return (loss.detach(), p1.grad, p2.grad) + tuple(f.grad for f in flows)
    return run


def test_deterministic_mode_is_bitwise_repeatable(dev, det):
    run = _loss_step(dev)
    outs = [tuple(t.clone() for t in run()) for _ in range(3)]
    for o in outs[1:]:
        assert all(same_bits(x, y) for x, y in zip(outs[0], o))
    torch.use_deterministic_algorithms(False)
    default = tuple(t.clone() for t in run())
    torch.use_deterministic_algorithms(True)
    assert rel_err(outs[0][0].cpu(), default[0].cpu()) <= 1e-6
    for x, y in zip(outs[0][1:], default[1:]):
        assert rel_err(x.cpu(), y.cpu()) <= 1e-5


def _model(dev, refine=False, k=64, seed=0):
    from pvraft_b200 import RSF, RSF_refine
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    torch.manual_seed(seed)
    return (RSF_refine if refine else RSF)(args).to(dev).train()


@pytest.fixture
def tc_train():
    """The model's per-point layers on the tensor-core kernels in eager steps too (by default only a captured step takes
    them), so that an eager and a captured step run the same kernels."""
    from pvraft_b200 import train as T
    was = T._TC_TRAIN
    T._TC_TRAIN = '1'
    try:
        yield
    finally:
        T._TC_TRAIN = was


def test_captured_step_equals_eager_bitwise(dev, det, tc_train):
    """Forward + sequence_self_supervised_loss + backward captured as one CUDA graph gives the eager step's bits."""
    from pvraft_b200.loss import sequence_self_supervised_loss
    m = _model(dev)
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(2, 1024, seed=41)]
    batch = {'sequence': [pc1, pc2]}
    out = {}

    def step():
        m.zero_grad(set_to_none=True)
        loss = sequence_self_supervised_loss(m([pc1, pc2], num_iters=2), batch)
        loss.backward()
        out['loss'] = loss.detach()   # no reference to the step's autograd graph outlives it

    step()
    eager = [out['loss'].detach().clone()] + [p.grad.detach().clone() for p in m.parameters()]
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream(dev).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    graph.replay()
    torch.cuda.synchronize()
    replayed = [out['loss'].detach()] + [p.grad.detach() for p in m.parameters()]
    assert len(replayed) == 96
    assert all(same_bits(x, y) for x, y in zip(eager, replayed))


# ---- model -----------------------------------------------------------------------------------------------------------------------
def test_rsf_gradients_match_oracle(dev):
    """One 3-iteration stage-1 step with sequence_self_supervised_loss against autograd through the oracle's rsf_forward plus
    the float64 loss: all 95 parameter gradients, with test_gpu_train.py's bounds."""
    from pvraft_b200 import RSF, ops
    from pvraft_b200.loss import sequence_self_supervised_loss
    b, n, k, iters = 2, 1024, 128, 3
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    W = default_weights(args=args, seed=2)
    pc1, pc2 = O.synthetic_clouds(b, n, seed=11)
    pc1, pc2 = pc1 * 0.4, pc2 * 0.4
    nbr = ops.knn(pc1.to(dev).contiguous(), pc1.to(dev).contiguous(), 9, mode=0).long().cpu()
    Wr = {kk: leaf(v) for kk, v in W.items()}
    flows_ref = O.rsf_forward(Wr, pc1, pc2, iters, 3, 0.25, k)
    want_loss = loss64(flows_ref, pc1, pc2, nbr)
    want_loss.backward()
    want = {kk: v.grad for kk, v in Wr.items()}
    m = RSF(args)
    m.load_state_dict(W)
    m = m.to(dev).train()
    with oracle_adjacency():
        flows = m([pc1.to(dev), pc2.to(dev)], num_iters=iters)
    loss = sequence_self_supervised_loss(flows, {'sequence': [pc1.to(dev), pc2.to(dev)]})
    assert abs(float(loss.detach()) - float(want_loss.detach())) < 1e-4 * abs(float(want_loss.detach()))
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters()}
    assert len(got) == 95 and all(v is not None for v in got.values())
    compare_grads(got, want, 2e-2, 5e-2)        # measured: 1.3e-3 relative L2, 2.4e-3 max-abs, cosine 0.99999998


def test_loss_input_gradients_against_float64(dev):
    """Gradients of the loss alone into the flows, P1 (through W = P1 + f) and P2 (through d_b)."""
    from pvraft_b200 import ops
    from pvraft_b200.loss import sequence_self_supervised_loss
    b, n, m = 2, 900, 1100
    gen = torch.Generator().manual_seed(6)
    p1, p2 = torch.rand(b, n, 3, generator=gen) * 4, torch.rand(b, m, 3, generator=gen) * 4
    fl = [torch.randn(b, n, 3, generator=gen) * 0.2 for _ in range(3)]
    p1d, p2d, fd = leaf(p1, dev), leaf(p2, dev), [leaf(f, dev) for f in fl]
    loss = sequence_self_supervised_loss(fd, {'sequence': [p1d, p2d]}, gamma=0.7, w_chamfer=2.0, w_smooth=0.5)
    loss.backward()
    nbr = ops.knn(p1d.detach(), p1d.detach(), 9, mode=0).long().cpu()
    p164, p264, f64 = leaf(p1.double()), leaf(p2.double()), [leaf(f.double()) for f in fl]
    want = loss64(f64, p164, p264, nbr, gamma=0.7, wc=2.0, ws=0.5)
    want.backward()
    assert abs(float(loss.detach()) - float(want.detach())) <= 1e-6 * abs(float(want.detach()))
    assert rel_err(p1d.grad.cpu(), p164.grad) <= 1e-5 and rel_err(p2d.grad.cpu(), p264.grad) <= 1e-5
    for a, r in zip(fd, f64):
        assert rel_err(a.grad.cpu(), r.grad) <= 1e-5


def test_model_input_gradients(dev):
    """Through the model's input-gradient path: P1 and P2 receive gradient from the flows and from the loss."""
    from pvraft_b200.loss import sequence_self_supervised_loss
    m = _model(dev)
    pc1, pc2 = [leaf(t * 0.4, dev) for t in O.synthetic_clouds(2, 1024, seed=13)]
    loss = sequence_self_supervised_loss(m([pc1, pc2], num_iters=2), {'sequence': [pc1, pc2]})
    loss.backward()
    for t in (pc1, pc2):
        assert t.grad is not None and bool(torch.isfinite(t.grad).all()) and float(t.grad.abs().max()) > 0
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in m.parameters())


def test_rsf_refine_with_self_supervised_loss(dev):
    from pvraft_b200.loss import self_supervised_loss
    m = _model(dev, refine=True)
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(2, 512, seed=17)]
    refined = m([pc1, pc2], 3)
    assert refined.shape == (2, 512, 3)
    loss = self_supervised_loss(refined, {'sequence': [pc1, pc2]})
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters() if p.grad is not None}
    assert len(got) == 29 and all(kk.startswith('refine_block.') for kk in got)
    assert bool(torch.isfinite(loss)) and all(bool(torch.isfinite(v).all()) for v in got.values())


def test_bf16_mixed_runs(dev):
    from pvraft_b200.loss import sequence_self_supervised_loss
    m = _model(dev).set_precision('bf16-mixed')
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(2, 1024, seed=19)]
    loss = sequence_self_supervised_loss(m([pc1, pc2], num_iters=2), {'sequence': [pc1, pc2]})
    loss.backward()
    assert bool(torch.isfinite(loss))
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in m.parameters())


def test_adam_lowers_the_loss_on_a_rigidly_moved_pair(dev):
    """30 Adam steps on one pair: P2 is P1 rotated by 5 degrees, moved by (0.1, -0.05, 0.08) and given 5 mm of noise."""
    from pvraft_b200.loss import sequence_self_supervised_loss
    m = _model(dev)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    gen = torch.Generator().manual_seed(23)
    pc1 = O.synthetic_clouds(1, 1024, seed=23)[0] * 0.4
    t = torch.tensor(5.0 * np.pi / 180)
    rot = torch.tensor([[torch.cos(t), -torch.sin(t), 0.0], [torch.sin(t), torch.cos(t), 0.0], [0.0, 0.0, 1.0]])
    pc2 = pc1 @ rot.T + torch.tensor([0.1, -0.05, 0.08]) + torch.randn(pc1.shape, generator=gen) * 0.005
    pc1, pc2 = pc1.to(dev), pc2.to(dev)
    batch = {'sequence': [pc1, pc2]}
    losses = []
    for _ in range(30):
        opt.zero_grad()
        loss = sequence_self_supervised_loss(m([pc1, pc2], num_iters=2), batch)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    ratio = losses[-1] / losses[0]
    print(f'self-supervised loss over 30 Adam steps: {losses[0]:.5f} -> {losses[-1]:.5f} (ratio {ratio:.3f})')
    # measured on an H100: 0.51091 -> 0.06188, a ratio of 0.121
    assert all(np.isfinite(losses)) and ratio < 0.4, losses


def test_drop_in_import_with_batch(dev):
    from pvraft_b200 import loss as L
    from pvraft_b200.data import Batch
    from tools.loss import self_supervised_loss, sequence_self_supervised_loss
    g = torch.Generator().manual_seed(2)
    items = [{'sequence': [torch.rand(1, 256, 3, generator=g), torch.rand(1, 300, 3, generator=g)],
              'ground_truth': [torch.ones(1, 256, 1), torch.zeros(1, 256, 3)]} for _ in range(2)]
    batch = Batch(items).to(dev)
    flows = [torch.randn(2, 256, 3, generator=g).to(dev) * 0.1 for _ in range(3)]
    seq = sequence_self_supervised_loss(flows, batch)
    one = self_supervised_loss(flows[-1], batch)
    assert seq.dim() == 0 and one.dim() == 0 and seq.is_cuda
    want = sum(0.8 ** (2 - i) * L.self_supervised_loss(f, batch) for i, f in enumerate(flows))
    assert abs(float(seq) - float(want)) <= 1e-6 * abs(float(want))
    assert sequence_self_supervised_loss is L.sequence_self_supervised_loss
