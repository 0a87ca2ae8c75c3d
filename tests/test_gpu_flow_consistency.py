"""The forward-backward consistency kernels (csrc/flow_consistency.cu, loss.ConsistencyFn, pvraft_b200.flow_consistency): the
search bit-exact against a numpy float32 restatement, the grid form bitwise the brute-force form, values and gradients
against the float64 restatement below, deterministic mode and batching.

    bhat_i = sum_r w_r f21[j_r] / sum_r w_r,  w_r = 1 / (d_r + 1e-8)   j_r: the k nearest of W_i = P1_i + f12_i in P2
    r_i    = f12_i + bhat_i,  ok_i = ||r_i||^2 < alpha (||f12_i||^2 + ||bhat_i||^2) + beta,  F_s = (1/N) sum_i ||r_i||^2
"""
import numpy as np
import pytest
import torch

from test_gpu_laplacian import knearest_host, same_bits

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


def consistency64(w, f12, p2, f21, nn_idx):
    """[S] F_s, r [S,N,3] and bhat [S,N,3] in float64 with the neighbours nn_idx [S,N,k] held fixed."""
    out, res, bh = [], [], []
    for s in range(w.shape[0]):
        b, idx = s % p2.shape[0], nn_idx[s].long()
        d = ((w[s][:, None, :] - p2[b][idx]) ** 2).sum(-1)
        wt = 1.0 / (d + 1e-8)
        bhat = (wt[..., None] * f21[s][idx]).sum(1) / wt.sum(1, keepdim=True)
        r = f12[s] + bhat
        out.append((r ** 2).sum(-1).mean())
        res.append(r)
        bh.append(bhat)
    return torch.stack(out), torch.stack(res), torch.stack(bh)


def case(s, b, n, m, seed, shift=0.0, scale=4.0, dup=False):
    g = torch.Generator().manual_seed(seed)
    p1, p2 = torch.rand(s, n, 3, generator=g) * scale + shift, torch.rand(b, m, 3, generator=g) * scale + shift
    f12, f21 = torch.randn(s, n, 3, generator=g) * 0.1, torch.randn(s, m, 3, generator=g) * 0.1
    if dup:
        p2[:, m // 2:m // 2 + 100] = p2[:, :100]
        p1[:, :60] = p2[0, 200:260] - f12[:, :60]     # W on points of P2, some of them duplicated
        p1[:, 60:80] = p2[0, m // 2:m // 2 + 20] - f12[:, 60:80]
    w = p1 + f12
    return w, f12, p2, f21


def run(dev, w, f12, p2, f21, k, alpha=0.01, beta=0.0025, use_grid=None):
    from pvraft_b200 import ops
    t = [x.to(dev).contiguous() for x in (w, f12, p2, f21)]
    return ops.flow_consistency(*t, k, alpha, beta, use_grid=use_grid)


@pytest.mark.parametrize('k', [1, 3, 8])
@pytest.mark.parametrize('s,b,n,m,shift,dup', [(4, 2, 1000, 1537, 0.0, False), (2, 1, 64, 65, 0.0, False),
                                               (2, 2, 3000, 2500, 1e3, False), (2, 1, 900, 700, 0.0, True)])
def test_search_bit_exact_and_grid_equals_brute_force(dev, s, b, n, m, shift, dup, k):
    w, f12, p2, f21 = case(s, b, n, m, seed=n + m + k, shift=shift, dup=dup)
    a = run(dev, w, f12, p2, f21, k, use_grid=False)
    g = run(dev, w, f12, p2, f21, k, use_grid=True)
    nn = a[1].cpu().numpy()
    for i in range(s):
        assert np.array_equal(nn[i], knearest_host(w[i].numpy(), p2[i % b].numpy(), k)), i
    for x, y in zip(a[1:], g[1:]):
        assert same_bits(x, y)


def test_exact_ties(dev):
    """Integer coordinates: many exactly equal distances; duplicated points and queries."""
    g = torch.Generator().manual_seed(3)
    w = torch.randint(-6, 7, (2, 700, 3), generator=g).float()
    p2 = torch.randint(-6, 7, (1, 900, 3), generator=g).float()
    p2[0, 450:600] = p2[0, 0:150]
    w[1, 400:] = w[1, :300].clone()
    f12, f21 = torch.randn(2, 700, 3, generator=g), torch.randn(2, 900, 3, generator=g)
    for k in (1, 3, 8):
        a = run(dev, w, f12, p2, f21, k, use_grid=False)
        b = run(dev, w, f12, p2, f21, k, use_grid=True)
        for s in range(2):
            assert np.array_equal(a[1][s].cpu().numpy(), knearest_host(w[s].numpy(), p2[0].numpy(), k))
        assert all(same_bits(x, y) for x, y in zip(a[1:], b[1:]))


@pytest.mark.parametrize('n', [8192, 32768, 131072])
def test_grid_equals_brute_force_large(dev, n):
    w, f12, p2, f21 = case(1, 1, n, n, seed=n, scale=50.0)
    a = run(dev, w, f12, p2, f21, 3, use_grid=False)
    g = run(dev, w, f12, p2, f21, 3, use_grid=True)
    assert all(same_bits(x, y) for x, y in zip(a[1:], g[1:]))


@pytest.mark.parametrize('dup', [False, True])
def test_values_and_gradients_against_float64(dev, dup):
    from pvraft_b200.loss import ConsistencyFn
    w, f12, p2, f21 = case(6, 2, 1200, 1100, seed=11, dup=dup)
    k, alpha, beta = 3, 0.01, 0.0025
    acc, nn_idx, res, ok = run(dev, w, f12, p2, f21, k, alpha, beta)
    f64, r64, b64 = consistency64(w.double(), f12.double(), p2.double(), f21.double(), nn_idx.cpu())
    assert torch.allclose(acc.cpu() / w.shape[1], f64, rtol=1e-5, atol=1e-9)
    assert torch.allclose(res.cpu().double(), r64, rtol=1e-4, atol=1e-6)
    rr, lim = (r64 ** 2).sum(-1), alpha * ((f12.double() ** 2).sum(-1) + (b64 ** 2).sum(-1)) + beta
    clear = (rr - lim).abs() > 1e-6 * lim
    assert clear.float().mean() > 0.99
    assert torch.equal(ok.cpu().bool()[clear], (rr < lim)[clear])

    gw = torch.randn(6, generator=torch.Generator().manual_seed(1)).float()
    xs = [t.to(dev).requires_grad_(True) for t in (w, f12, p2, f21)]
    (ConsistencyFn.apply(*xs, k) * gw.to(dev)).sum().backward()
    ys = [t.double().requires_grad_(True) for t in (w, f12, p2, f21)]
    (consistency64(*ys, nn_idx.cpu())[0] * gw.double()).sum().backward()
    for x, y, name in zip(xs, ys, ('d_w', 'd_f12', 'd_p2', 'd_f21')):
        err = (x.grad.cpu().double() - y.grad).norm() / y.grad.norm().clamp_min(1e-30)
        assert err < 2e-4, (name, float(err))


def test_deterministic_bitwise_repeatable_and_batching(dev, det):
    from pvraft_b200 import ops
    w, f12, p2, f21 = case(6, 2, 3000, 2600, seed=5)
    t = [x.to(dev).contiguous() for x in (w, f12, p2, f21)]
    for grid in (False, True):
        a = ops.flow_consistency(*t, 3, 0.01, 0.0025, use_grid=grid)
        b = ops.flow_consistency(*t, 3, 0.01, 0.0025, use_grid=grid)
        assert all(same_bits(x, y) for x, y in zip(a, b))
        parts = [ops.flow_consistency(t[0][i:i + 2].contiguous(), t[1][i:i + 2].contiguous(), t[2], t[3][i:i + 2].contiguous(), 3, 0.01,
                                      0.0025, use_grid=grid) for i in (0, 2, 4)]
        for j in range(4):
            assert same_bits(a[j], torch.cat([q[j] for q in parts]))
    g = torch.rand(6, device=dev)
    d1 = ops.flow_consistency_bwd(t[0], t[2], t[3], a[1], a[2], g)
    d2 = ops.flow_consistency_bwd(t[0], t[2], t[3], a[1], a[2], g)
    assert all(same_bits(x, y) for x, y in zip(d1, d2))
    # the backward over S = 6 against three launches of S = 2: d_w, d_f12 and d_f21 per sample bitwise.  d_p2 sums over the
    # predictions: each launch rounds its exact fixed-point sum to fp32 once, so the one launch's d_p2 and the float64 sum of
    # the three differ by at most half an fp32 ulp of each of the four roundings (terms of opposite sign cancel, so no
    # relative bound on the total holds)
    parts = [ops.flow_consistency_bwd(t[0][i:i + 2].contiguous(), t[2], t[3][i:i + 2].contiguous(), a[1][i:i + 2].contiguous(),
                                      a[2][i:i + 2].contiguous(), g[i:i + 2].contiguous()) for i in (0, 2, 4)]
    for j in (0, 1, 3):
        assert same_bits(d1[j], torch.cat([q[j] for q in parts]))
    dp2 = sum(q[2].double() for q in parts)
    bound = 2.0 ** -24 * (d1[2].double().abs() + sum(q[2].double().abs() for q in parts))
    assert bool(((d1[2].double() - dp2).abs() <= bound).all())
    assert float(d1[2].abs().max()) > 0


def test_public_function(dev):
    import pvraft_b200
    g = torch.Generator().manual_seed(0)
    p1 = (torch.rand(2, 2048, 3, generator=g) * 10).to(dev)
    f = torch.tensor([0.3, -0.1, 0.05], device=dev).expand(2, 2048, 3).contiguous()
    p2 = p1 + f
    out = pvraft_b200.flow_consistency(p1, f, p2, -f)            # a rigid translation and its inverse: consistent everywhere
    assert out.consistent_12.dtype == torch.bool and out.consistent_12.shape == (2, 2048)
    assert out.consistent_12.all() and out.consistent_21.all()
    assert out.res_12.abs().max() < 1e-5 and out.res_21.shape == (2, 2048, 3)
    bad = -f.clone()
    bad[:, :100] = 1.0                                           # the reverse flow disagrees on 100 points
    out = pvraft_b200.flow_consistency(p1, f, p2, bad)
    assert (~out.consistent_21[:, :100]).all() and out.consistent_21[:, 200:].float().mean() > 0.9
