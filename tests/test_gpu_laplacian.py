"""The Laplacian regularity term of the self-supervised loss (pvraft_b200/loss.py LaplacianFn, csrc/laplacian.cu): the
interpolation search bit-exact against a numpy float32 restatement of the difference form and the tie rule, values and
gradients against the float64 restatement below (kept here: the reference has no self-supervised loss), batching,
deterministic mode, capture, and training the model with the three-term loss.

    L(X)_i = sum_{j in G(i)} (X_j - X_i) / (k_lap - 1)            G1 = knn(P1, P1, k_lap), G2 = knn(P2, P2, k_lap), mode 0
    Lhat_i = sum_r w_r L(P2)_{j_r} / sum_r w_r,  w_r = 1 / (d_r + 1e-8)   j_r: the k_int nearest of W_i in P2, d_r squared
    R_s    = (1/N) sum_i ||Lhat_i - L(W)_i||^2,  L(W) over G1,  W = P1 + f
    L      = sum_i gamma^(n-i-1) mean_b (w_c C_b + w_s S_b + w_l R_b)
"""
import types

import numpy as np
import pytest
import torch

from conftest import default_weights, rel_err
from oracle import pvraft_oracle as O
from test_gpu_self_supervised import chamfer64, nn64_indices, smooth64
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


def same_bits(a, b):
    a, b = a.detach().contiguous(), b.detach().contiguous()
    if a.is_floating_point():
        a, b = (t.view(torch.int64 if t.element_size() == 8 else torch.int32) for t in (a, b))
    return torch.equal(a, b)


def leaf(t, dev=None):
    t = t.detach().clone()
    return (t.to(dev) if dev is not None else t).requires_grad_(True)


# ---- host restatements ---------------------------------------------------------------------------------------------------
def knearest_host(q, c, k):
    """The k nearest points of c for every point of q in float32, (dx*dx + dy*dy) + dz*dz of the differences (numpy rounds
    every operation and never contracts), ranked on (distance, index) -> [n,k], nearest first."""
    q, c = q.astype(np.float32), c.astype(np.float32)
    out = np.empty((len(q), k), np.int64)
    ids = np.arange(len(c), dtype=np.int64)
    rows = max(1, (1 << 22) // len(c))
    for r0 in range(0, len(q), rows):
        d = q[r0:r0 + rows, None, :] - c[None, :, :]
        dd = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        # a non-negative float's bits order like the float: one int64 key per (distance, index)
        key = (dd.view(np.int32).astype(np.int64) << 32) | ids
        part = np.partition(key, k - 1, axis=1)[:, :k] if k < len(c) else key
        part.sort(axis=1)
        out[r0:r0 + rows] = part[:, :k] & 0xffffffff
    return out


def lap64(x, nbr):
    """L(x) [N,3] over the graph nbr [N,k]."""
    return (x[nbr] - x[:, None, :]).sum(1) / (nbr.shape[1] - 1)


def term64(w, p2, l2, g1, nn_idx):
    """[S] R_s in float64 with the interpolation neighbours nn_idx [S,N,k_int] held fixed; l2 [B,M,3] given."""
    out = []
    for s in range(w.shape[0]):
        b = s % p2.shape[0]
        idx = nn_idx[s]
        d = ((w[s][:, None, :] - p2[b][idx]) ** 2).sum(-1)
        wt = 1.0 / (d + 1e-8)
        lhat = (wt[..., None] * l2[b][idx]).sum(1) / wt.sum(1, keepdim=True)
        out.append(((lhat - lap64(w[s], g1[b])) ** 2).sum(-1).mean())
    return torch.stack(out)


def laplacian64(w, p2, g1, g2, nn_idx):
    l2 = torch.stack([lap64(p2[b], g2[b]) for b in range(p2.shape[0])])
    return term64(w, p2, l2, g1, nn_idx)


def nn64_knearest(w, p2, k):
    """Float64 k nearest of every W_i in P2[s % B] -> [S,N,k]."""
    out = []
    for s in range(w.shape[0]):
        d = ((w[s][:, None, :] - p2[s % p2.shape[0]][None, :, :]) ** 2).sum(-1)
        out.append(d.topk(k, 1, largest=False).indices)
    return torch.stack(out)


def graphs(p1, p2, k_lap):
    from pvraft_b200 import ops
    p1, p2 = p1.detach().contiguous(), p2.detach().contiguous()
    return ops.knn(p1, p1, k_lap, mode=0), ops.knn(p2, p2, k_lap, mode=0)


def loss64(flows, p1, p2, nbr, g1, g2, gamma=0.8, wc=1.0, ws=1.0, wl=0.3, k_int=5, lap_idx=None):
    """The three-term sequence loss in float64 for a list of [B,N,3] flows; every search in float64 unless lap_idx (one
    [S,N,k_int] per flow) gives the interpolation neighbours."""
    n, total = len(flows), 0
    for i, f in enumerate(flows):
        f = f.double()
        w = p1.double() + f
        nn_ab, nn_ba = nn64_indices(w.detach(), p2.double())
        idx = nn64_knearest(w.detach(), p2.double(), k_int) if lap_idx is None else lap_idx[i]
        per = (wc * chamfer64(w, p2.double(), nn_ab, nn_ba) + ws * smooth64(f, nbr)
               + wl * laplacian64(w, p2.double(), g1, g2, idx))
        total = total + gamma ** (n - i - 1) * per.mean()
    return total


# ---- search ----------------------------------------------------------------------------------------------------------------
def clouds(s, b, n, m, seed, shift=0.0, scale=5.0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(s, n, 3, generator=g) * scale + shift, torch.rand(b, m, 3, generator=g) * scale + shift


def check_search(w, p2, k_int, dev, k_lap=4):
    from pvraft_b200 import ops
    wd, p2d = w.to(dev).contiguous(), p2.to(dev).contiguous()
    b = p2.shape[0]
    g1 = ops.knn(wd[:b].contiguous(), wd[:b].contiguous(), k_lap, mode=0)
    l2 = ops.cloud_laplacian(p2d, ops.knn(p2d, p2d, k_lap, mode=0))
    _, nn_idx, _ = ops.laplacian(wd, p2d, l2, g1, k_int)
    nn_idx = nn_idx.cpu().numpy()
    for s in range(w.shape[0]):
        want = knearest_host(w[s].numpy(), p2[s % b].numpy(), k_int)
        assert np.array_equal(nn_idx[s], want), (s, int((nn_idx[s] != want).any(1).sum()))


@pytest.mark.parametrize('k_int', [1, 3, 5, 8])
@pytest.mark.parametrize('s,b,n,m', [(4, 2, 1000, 1537), (2, 1, 32, 33), (2, 2, 4096, 4096)])
def test_search_bit_exact(dev, s, b, n, m, k_int):
    check_search(*clouds(s, b, n, m, seed=n + m + k_int), k_int, dev)


def test_search_20000(dev):
    check_search(*clouds(1, 1, 20000, 20000, seed=7, scale=50.0), 5, dev)


@pytest.mark.parametrize('k_int', [1, 5, 8])
def test_search_far_from_the_origin(dev, k_int):
    """Clouds shifted by 1e3, where the expanded form |q|^2 + |x|^2 - 2 q.x would cancel."""
    check_search(*clouds(2, 2, 3000, 2500, seed=5, shift=1e3, scale=20.0), k_int, dev)


@pytest.mark.parametrize('k_int', [1, 3, 8])
def test_search_duplicates_and_exact_ties(dev, k_int):
    """Integer coordinates make many distances exactly equal; duplicated points have equal distances to everything."""
    g = torch.Generator().manual_seed(3)
    w = torch.randint(-6, 7, (2, 700, 3), generator=g).float()
    p2 = torch.randint(-6, 7, (1, 900, 3), generator=g).float()
    p2[0, 450:600] = p2[0, 0:150]                  # duplicated points of the searched cloud
    w[1, 400:] = w[1, :300].clone()                # duplicated queries
    w[0, :50] = p2[0, 10:60]                       # distance 0
    check_search(w, p2, k_int, dev)


# ---- values and gradients -----------------------------------------------------------------------------------------------------
def _case(dev, n_pred, b, n, m, k_lap, seed, dup=False):
    from pvraft_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    p1, p2 = torch.rand(b, n, 3, generator=gen) * 4, torch.rand(b, m, 3, generator=gen) * 4
    f = torch.randn(n_pred * b, n, 3, generator=gen) * 0.1
    if dup:
        p2[:, m // 2:m // 2 + 100] = p2[:, :100]                       # duplicated points of P2
        p1[:, :60] = p2[:, 200:260]
        f[:, :60] = 0.0                                                # W_i = P2_j exactly: d = 0, w = 1e8
    w = (f.view(n_pred, b, n, 3) + p1).reshape(-1, n, 3)
    g1, g2 = graphs(p1.to(dev), p2.to(dev), k_lap)
    return w, p2, g1, g2, ops


@pytest.mark.parametrize('dup', [False, True])
@pytest.mark.parametrize('k_lap', [2, 10, 32])
def test_values_and_gradients_against_float64(dev, k_lap, dup):
    from pvraft_b200.loss import LaplacianFn
    n_pred, b, n, m, k_int = 3, 2, 1000, 1537, 5
    w, p2, g1, g2, ops = _case(dev, n_pred, b, n, m, k_lap, seed=k_lap, dup=dup)
    gen = torch.Generator().manual_seed(100 + k_lap)
    g = torch.rand(n_pred * b, generator=gen) + 0.5

    wd, p2d = leaf(w, dev), leaf(p2, dev)
    r = LaplacianFn.apply(wd, p2d, g1, g2, k_int)
    (r * g.to(dev)).sum().backward()
    l2 = ops.cloud_laplacian(p2d.detach(), g2)
    _, nn_idx, res = ops.laplacian(wd.detach(), p2d.detach(), l2, g1, k_int)
    _, _, d_l2 = ops.laplacian_bwd(wd.detach(), p2d.detach(), l2, g1, nn_idx, res, g.to(dev))

    idx, g164, g264 = nn_idx.long().cpu(), g1.long().cpu(), g2.long().cpu()
    w64, p264 = leaf(w.double()), leaf(p2.double())
    want = laplacian64(w64, p264, g164, g264, idx)
    got = r.detach().cpu().double()
    assert torch.all((got - want.detach()).abs() <= 1e-6 * want.detach().abs()), (got, want)
    (want * g.double()).sum().backward()
    assert rel_err(wd.grad.cpu(), w64.grad) <= 1e-5
    assert rel_err(p2d.grad.cpu(), p264.grad) <= 1e-5
    # d_l2 alone: L2 as a leaf of its own
    l264 = leaf(torch.stack([lap64(p2.double()[i], g264[i]) for i in range(b)]))
    (term64(w.double(), p2.double(), l264, g164, idx) * g.double()).sum().backward()
    assert rel_err(d_l2.cpu(), l264.grad) <= 1e-5
    assert rel_err(l2.cpu(), l264.detach()) <= 1e-6


def test_cloud_laplacian_against_float64(dev):
    from pvraft_b200 import ops
    gen = torch.Generator().manual_seed(4)
    x = torch.rand(3, 777, 3, generator=gen) * 10 - 5
    for k in (2, 7, 32):
        nbr = ops.knn(x.to(dev), x.to(dev), k, mode=0)
        xd = leaf(x, dev)
        got = ops.cloud_laplacian(xd.detach(), nbr)
        x64 = leaf(x.double())
        want = torch.stack([lap64(x64[i], nbr[i].long().cpu()) for i in range(3)])
        assert rel_err(got.cpu(), want.detach()) <= 1e-6
        gl = torch.randn(3, 777, 3, generator=gen)
        (want * gl.double()).sum().backward()
        d = ops.cloud_laplacian_bwd(gl.to(dev), nbr, torch.zeros_like(xd))
        assert rel_err(d.cpu(), x64.grad) <= 1e-5


def test_one_launch_equals_separate_calls(dev, det):
    """S = n B samples in one launch give what n calls of B samples give (bitwise in deterministic mode)."""
    n_pred, b, n, m, k_lap, k_int = 3, 2, 1500, 1200, 10, 5
    w, p2, g1, g2, ops = _case(dev, n_pred, b, n, m, k_lap, seed=9)
    w, p2 = w.to(dev).contiguous(), p2.to(dev).contiguous()
    g = torch.rand(n_pred * b, generator=torch.Generator().manual_seed(9)).to(dev)
    l2 = ops.cloud_laplacian(p2, g2)
    acc, idx, res = ops.laplacian(w, p2, l2, g1, k_int)
    dw, _, _ = ops.laplacian_bwd(w, p2, l2, g1, idx, res, g, want_dp2=False)
    for i in range(n_pred):
        sl = slice(i * b, (i + 1) * b)
        acc_i, idx_i, res_i = ops.laplacian(w[sl].contiguous(), p2, l2, g1, k_int)
        assert torch.equal(idx_i, idx[sl]) and same_bits(acc_i, acc[sl]) and same_bits(res_i, res[sl])
        dw_i, _, _ = ops.laplacian_bwd(w[sl].contiguous(), p2, l2, g1, idx_i, res_i, g[sl].contiguous(), want_dp2=False)
        assert same_bits(dw_i, dw[sl])


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
        loss = sequence_self_supervised_loss(flows, {'sequence': [p1, p2]}, w_laplacian=0.3)
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
    """The per-point layers on the tensor-core kernels in eager steps too, so that an eager and a captured step run the same
    kernels."""
    from pvraft_b200 import train as T
    was = T._TC_TRAIN
    T._TC_TRAIN = '1'
    try:
        yield
    finally:
        T._TC_TRAIN = was


def test_captured_step_equals_eager_bitwise(dev, det, tc_train):
    """Forward + the three-term loss + backward captured as one CUDA graph gives the eager step's bits."""
    from pvraft_b200.loss import sequence_self_supervised_loss
    m = _model(dev)
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(2, 1024, seed=41)]
    batch = {'sequence': [pc1, pc2]}
    out = {}

    def step():
        m.zero_grad(set_to_none=True)
        loss = sequence_self_supervised_loss(m([pc1, pc2], num_iters=2), batch, w_laplacian=0.3)
        loss.backward()
        out['loss'] = loss.detach()

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
    """One 3-iteration stage-1 step with the three-term loss (w_laplacian = 0.3) against autograd through the oracle's
    rsf_forward plus the float64 loss: all 95 parameter gradients, with the bounds of test_gpu_self_supervised.py."""
    from pvraft_b200 import RSF, ops
    from pvraft_b200.loss import sequence_self_supervised_loss
    b, n, k, iters = 2, 1024, 128, 3
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    W = default_weights(args=args, seed=2)
    pc1, pc2 = O.synthetic_clouds(b, n, seed=11)
    pc1, pc2 = pc1 * 0.4, pc2 * 0.4
    nbr = ops.knn(pc1.to(dev).contiguous(), pc1.to(dev).contiguous(), 9, mode=0).long().cpu()
    g1, g2 = (t.long().cpu() for t in graphs(pc1.to(dev), pc2.to(dev), 10))
    Wr = {kk: leaf(v) for kk, v in W.items()}
    flows_ref = O.rsf_forward(Wr, pc1, pc2, iters, 3, 0.25, k)
    want_loss = loss64(flows_ref, pc1, pc2, nbr, g1, g2)
    want_loss.backward()
    want = {kk: v.grad for kk, v in Wr.items()}
    m = RSF(args)
    m.load_state_dict(W)
    m = m.to(dev).train()
    with oracle_adjacency():
        flows = m([pc1.to(dev), pc2.to(dev)], num_iters=iters)
    loss = sequence_self_supervised_loss(flows, {'sequence': [pc1.to(dev), pc2.to(dev)]}, w_laplacian=0.3)
    assert abs(float(loss.detach()) - float(want_loss.detach())) < 1e-4 * abs(float(want_loss.detach()))
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters()}
    assert len(got) == 95 and all(v is not None for v in got.values())
    compare_grads(got, want, 2e-2, 5e-2)


def test_loss_input_gradients_against_float64(dev):
    """Gradients of the three-term loss alone into the flows, P1 (through W = P1 + f) and P2 (through the distances and
    through L(P2))."""
    from pvraft_b200 import ops
    from pvraft_b200.loss import sequence_self_supervised_loss
    b, n, m, k_lap, k_int = 2, 900, 1100, 8, 4
    gen = torch.Generator().manual_seed(6)
    p1, p2 = torch.rand(b, n, 3, generator=gen) * 4, torch.rand(b, m, 3, generator=gen) * 4
    fl = [torch.randn(b, n, 3, generator=gen) * 0.2 for _ in range(3)]
    p1d, p2d, fd = leaf(p1, dev), leaf(p2, dev), [leaf(f, dev) for f in fl]
    loss = sequence_self_supervised_loss(fd, {'sequence': [p1d, p2d]}, gamma=0.7, w_chamfer=2.0, w_smooth=0.5, w_laplacian=0.7,
                                         k_lap=k_lap, k_int=k_int)
    loss.backward()
    nbr = ops.knn(p1d.detach(), p1d.detach(), 9, mode=0).long().cpu()
    g1, g2 = graphs(p1d, p2d, k_lap)
    l2 = ops.cloud_laplacian(p2d.detach(), g2)
    lap_idx = [ops.laplacian((p1d + f).detach().contiguous(), p2d.detach(), l2, g1, k_int)[1].long().cpu() for f in fd]
    p164, p264, f64 = leaf(p1.double()), leaf(p2.double()), [leaf(f.double()) for f in fl]
    want = loss64(f64, p164, p264, nbr, g1.long().cpu(), g2.long().cpu(), gamma=0.7, wc=2.0, ws=0.5, wl=0.7, k_int=k_int,
                  lap_idx=lap_idx)
    want.backward()
    assert abs(float(loss.detach()) - float(want.detach())) <= 1e-6 * abs(float(want.detach()))
    assert rel_err(p1d.grad.cpu(), p164.grad) <= 1e-5 and rel_err(p2d.grad.cpu(), p264.grad) <= 1e-5
    for a, r in zip(fd, f64):
        assert rel_err(a.grad.cpu(), r.grad) <= 1e-5


def test_model_input_gradients(dev):
    """Through the model's input-gradient path: P1 and P2 receive gradient from the flows and from the three-term loss."""
    from pvraft_b200.loss import sequence_self_supervised_loss
    m = _model(dev)
    pc1, pc2 = [leaf(t * 0.4, dev) for t in O.synthetic_clouds(2, 1024, seed=13)]
    loss = sequence_self_supervised_loss(m([pc1, pc2], num_iters=2), {'sequence': [pc1, pc2]}, w_laplacian=0.3)
    loss.backward()
    for t in (pc1, pc2):
        assert t.grad is not None and bool(torch.isfinite(t.grad).all()) and float(t.grad.abs().max()) > 0
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in m.parameters())


def test_rsf_refine_with_laplacian(dev):
    from pvraft_b200.loss import self_supervised_loss
    m = _model(dev, refine=True)
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(2, 512, seed=17)]
    loss = self_supervised_loss(m([pc1, pc2], 3), {'sequence': [pc1, pc2]}, w_laplacian=0.3)
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters() if p.grad is not None}
    assert len(got) == 29 and all(kk.startswith('refine_block.') for kk in got)
    assert bool(torch.isfinite(loss)) and all(bool(torch.isfinite(v).all()) for v in got.values())


def test_bf16_mixed_runs(dev):
    from pvraft_b200.loss import sequence_self_supervised_loss
    m = _model(dev).set_precision('bf16-mixed')
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(2, 1024, seed=19)]
    loss = sequence_self_supervised_loss(m([pc1, pc2], num_iters=2), {'sequence': [pc1, pc2]}, w_laplacian=0.3)
    loss.backward()
    assert bool(torch.isfinite(loss))
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in m.parameters())


def test_adam_lowers_the_three_term_loss_on_a_rigidly_moved_pair(dev):
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
        loss = sequence_self_supervised_loss(m([pc1, pc2], num_iters=2), batch, w_laplacian=0.3)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    ratio = losses[-1] / losses[0]
    print(f'three-term self-supervised loss over 30 Adam steps: {losses[0]:.5f} -> {losses[-1]:.5f} (ratio {ratio:.3f})')
    assert all(np.isfinite(losses)) and ratio < 0.5, losses


# ---- the default is unchanged ------------------------------------------------------------------------------------------------------
def test_zero_weight_is_the_two_term_loss(dev, det):
    """w_laplacian = 0: the loss and every gradient are the two-term loss's bits, from the same launches."""
    from pvraft_b200 import ops
    from pvraft_b200.loss import ChamferFn, SmoothFn, sequence_self_supervised_loss
    gen = torch.Generator().manual_seed(31)
    b, n, m = 2, 1200, 1000
    p1, p2 = leaf(torch.rand(b, n, 3, generator=gen) * 4, dev), leaf(torch.rand(b, m, 3, generator=gen) * 4, dev)
    fl = [leaf(torch.randn(b, n, 3, generator=gen) * 0.2, dev) for _ in range(3)]

    def grads(fn):
        for t in [p1, p2] + fl:
            t.grad = None
        n0 = ops.launch_count
        loss = fn()
        loss.backward()
        return [loss.detach().clone()] + [t.grad.clone() for t in [p1, p2] + fl], ops.launch_count - n0

    def two_term():
        flows = torch.stack(fl)
        nbr = ops.knn(p1.detach().contiguous(), p1.detach().contiguous(), 9, mode=0)
        w = (flows + p1).reshape(3 * b, n, 3)
        per = (1.0 * ChamferFn.apply(w, p2) + 1.0 * SmoothFn.apply(flows.reshape(3 * b, n, 3), nbr)).view(3, b).mean(1)
        weights = torch.pow(0.8, torch.arange(2, -1, -1, dtype=torch.float32, device=dev))
        return (weights * per).sum()

    want, launches = grads(two_term)
    for kw in ({}, dict(w_laplacian=0.0), dict(w_laplacian=0, k_lap=32, k_int=8)):
        got, got_launches = grads(lambda: sequence_self_supervised_loss(fl, {'sequence': [p1, p2]}, **kw))
        assert got_launches == launches, kw
        assert all(same_bits(x, y) for x, y in zip(got, want)), kw
