"""The SetConv edge kernel's shared-memory row table (csrc/setconv_edge.cu): every processing order, tiles that overflow the
table, ragged last tiles and the deterministic form give the same per-point maxima and minima, to the bit, and GroupNorm sums
within float64 bounds of a float64 reference."""
import pytest
import torch

from oracle import pvraft_oracle as O

pytestmark = pytest.mark.gpu

TABLE_FLOATS = 22528   # one table buffer (csrc/setconv_edge.cu): rows = min(32 * 33, TABLE_FLOATS / C)


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def graph(pc):
    from pvraft_b200 import ops
    nbr, rel = ops.knn(pc, pc, 32, mode=0, want_rel=True)
    return nbr, rel, ops.point_order(pc)


def inputs(b, n, c, cin, seed, dev):
    g = torch.Generator().manual_seed(seed)
    p = (torch.randn(b, n, c, generator=g) * (1 + torch.arange(b).view(b, 1, 1))).to(dev)
    w = torch.randn(c, cin + 3, generator=g).to(dev)
    return p, w


def edge(p, nbr, rel, w, cin, order=None):
    from pvraft_b200 import ops
    stats = torch.zeros(p.shape[0], 8, 2, dtype=torch.float64, device=p.device)
    ymax, ymin = ops.setconv_edge(p, nbr, rel, w, cin, stats, order=order)
    return ymax, ymin, stats


def check_fp64(p, nbr, rel, w, cin, got):
    """ymax / ymin within 1e-6 of the float64 maxima and minima; GroupNorm sums within the bounds of the bench-batch test."""
    ymax, ymin, stats = got
    b, n, c = p.shape
    we = w[:, cin:].double()
    for s in range(b):
        ps = p[s].double()
        y = ps[nbr[s].long()] - ps.unsqueeze(1) + rel[s].double() @ we.t()
        scale = y.abs().amax().clamp_min(1e-30)
        assert float((ymax[s].double() - y.amax(1)).abs().max() / scale) < 1e-6
        assert float((ymin[s].double() - y.amin(1)).abs().max() / scale) < 1e-6
        ys = y.reshape(-1, 8, c // 8)
        s1, s2, sabs = ys.sum((0, 2)), (ys ** 2).sum((0, 2)), ys.abs().sum((0, 2))
        assert bool(((stats[s, :, 0] - s1).abs() <= 1e-5 * s1.abs() + 1e-7 * sabs + 1e-30).all()), (stats[s, :, 0], s1)
        assert bool(((stats[s, :, 1] - s2).abs() <= 1e-5 * s2 + 1e-30).all()), (stats[s, :, 1], s2)


def assert_same_maxmin(a, b):
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def assert_stats_close(a, b):
    """Two GroupNorm sums of the same values in another order: equal within double rounding."""
    d = (a - b).abs()
    assert bool((d <= 1e-12 * b.abs() + 1e-300).all()), d


@pytest.mark.parametrize('c', [16, 48, 64, 96, 128])
def test_orders_bitwise(dev, c):
    """Morton order, index order and a random permutation fill different tables (and overflow differently); the per-point
    arithmetic is the same, so ymax / ymin are the same bits, and all three match float64."""
    b, n, cin = 2, 8192, 64
    pc, _ = O.synthetic_clouds(b, n, seed=c)
    pc = pc.to(dev)
    nbr, rel, morton = graph(pc)
    perm = torch.stack([torch.randperm(n, generator=torch.Generator().manual_seed(s)) for s in range(b)]).to(dev, torch.int32)
    p, w = inputs(b, n, c, cin, c, dev)
    res = {name: edge(p, nbr, rel, w, cin, o) for name, o in (('morton', morton), ('index', None), ('random', perm))}
    check_fp64(p, nbr, rel, w, cin, res['morton'])
    for name in ('index', 'random'):
        assert_same_maxmin(res[name], res['morton'])
        assert_stats_close(res[name][2], res['morton'][2])


def test_batched_equals_per_sample(dev):
    b, n, c, cin = 3, 8192, 64, 64
    pc, _ = O.synthetic_clouds(b, n, seed=7)
    pc = pc.to(dev)
    nbr, rel, order = graph(pc)
    p, w = inputs(b, n, c, cin, 7, dev)
    whole = edge(p, nbr, rel, w, cin, order)
    for s in range(b):
        one = edge(p[s:s + 1].contiguous(), nbr[s:s + 1].contiguous(), rel[s:s + 1].contiguous(), w, cin, order[s:s + 1].contiguous())
        assert torch.equal(one[0][0], whole[0][s]) and torch.equal(one[1][0], whole[1][s])
        assert_stats_close(one[2][0], whole[2][s])


def test_overflow_unordered_random_cloud(dev):
    """C = 128 (a 176-row table) over a uniformly random cloud in index order: a tile of 32 points references far more
    distinct rows than the table holds, so its rows come from global memory."""
    b, n, c, cin = 2, 8192, 128, 64
    pc = torch.rand(b, n, 3, generator=torch.Generator().manual_seed(3)).to(dev)
    nbr, rel, morton = graph(pc)
    rows = TABLE_FLOATS // c
    refs = torch.cat([nbr.reshape(b, n // 32, 32 * 32), torch.arange(n, device=dev, dtype=torch.int32).view(1, n // 32, 32).expand(b, -1, -1)], 2)
    distinct = torch.tensor([len(torch.unique(t)) for t in refs.reshape(-1, refs.shape[-1])])
    assert float((distinct > rows).float().mean()) > 0.9   # (most tiles overflow)
    p, w = inputs(b, n, c, cin, 3, dev)
    plain, ordered = edge(p, nbr, rel, w, cin, None), edge(p, nbr, rel, w, cin, morton)
    check_fp64(p, nbr, rel, w, cin, plain)
    assert_same_maxmin(plain, ordered)
    assert_stats_close(plain[2], ordered[2])


def test_single_row_table(dev):
    """Every reference of a tile is the same row: one point whose 32 neighbours are itself, and a cloud of one repeated
    point (32 distinct ids, all edge vectors zero)."""
    from pvraft_b200 import ops
    c, cin = 64, 64
    p, w = inputs(2, 1, c, cin, 11, dev)
    nbr = torch.zeros(2, 1, 32, dtype=torch.int32, device=dev)
    rel = torch.randn(2, 1, 32, 3, generator=torch.Generator().manual_seed(11)).to(dev)
    got = edge(p, nbr, rel, w, cin)
    check_fp64(p, nbr, rel, w, cin, got)
    pc = torch.full((2, 256, 3), 0.25, device=dev)
    nbr, rel = ops.knn(pc, pc, 32, mode=0, want_rel=True)
    p, w = inputs(2, 256, c, cin, 12, dev)
    check_fp64(p, nbr, rel, w, cin, edge(p, nbr, rel, w, cin))


@pytest.mark.parametrize('c', [64, 96])
def test_ragged_last_tile(dev, c):
    """N = 1000 is not a multiple of the 32-point tile, B = 3: the last tile of every sample is short."""
    b, n, cin = 3, 1000, 32
    pc, _ = O.synthetic_clouds(b, n, seed=5)
    pc = pc.to(dev)
    nbr, rel, order = graph(pc)
    p, w = inputs(b, n, c, cin, 5, dev)
    ordered, plain = edge(p, nbr, rel, w, cin, order), edge(p, nbr, rel, w, cin, None)
    check_fp64(p, nbr, rel, w, cin, ordered)
    assert_same_maxmin(plain, ordered)
    assert_stats_close(plain[2], ordered[2])


@pytest.mark.parametrize('c', [48, 64, 128])
def test_deterministic_form(dev, c):
    """Under torch.use_deterministic_algorithms(True): two runs are the same bits, maxima and minima are those of the
    default form, and the sums equal the default form's within double rounding."""
    b, n, cin = 4, 8192, 64
    pc, _ = O.synthetic_clouds(b, n, seed=c + 1)
    pc = pc.to(dev)
    nbr, rel, order = graph(pc)
    p, w = inputs(b, n, c, cin, c + 1, dev)
    default = edge(p, nbr, rel, w, cin, order)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        r1, r2, r3 = edge(p, nbr, rel, w, cin, order), edge(p, nbr, rel, w, cin, order), edge(p, nbr, rel, w, cin, None)
    finally:
        torch.use_deterministic_algorithms(prev)
    for r in (r2, r3):   # (the index order fills other tables: the sums do not depend on that either)
        assert_same_maxmin(r, r1)
        assert torch.equal(r[2], r1[2])
    assert_same_maxmin(r1, default)
    assert_stats_close(r1[2], default[2])
