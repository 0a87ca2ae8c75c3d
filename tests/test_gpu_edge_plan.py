"""The SetConv edge kernel's gather plan (csrc/edge_plan.cu, layout in csrc/edge_plan.cuh): each tile's distinct rows and
reference slots against a numpy construction, at every table capacity, for short last tiles and for a plan sliced out of a
larger batch; and the edge kernel run from the plan's tables against the same kernel gathering every tile from global
memory."""
import numpy as np
import pytest
import torch

from oracle import pvraft_oracle as O

pytestmark = pytest.mark.gpu

TILE = 32
REFS = TILE * 33
SLOTS, COUNT = REFS * 4, REFS * 6          # byte offsets in a tile's record (csrc/edge_plan.cuh)
TABLE_FLOATS = 22528                        # one table buffer (csrc/setconv_edge.cu): rows = min(REFS, TABLE_FLOATS / C)


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def decode(plan):
    """uint8 [B,T,record] -> numpy count [B,T], ids [B,T,REFS], slots [B,T,REFS]."""
    a = plan.cpu().numpy()
    ids = a[..., :SLOTS].copy().view(np.int32)
    slots = a[..., SLOTS:COUNT].copy().view(np.uint16).astype(np.int64)
    count = a[..., COUNT:COUNT + 4].copy().view(np.int32)[..., 0]
    return count, ids, slots


def tile_refs(nbr, order, b, t, n):
    """Row ids a tile references, in the plan's reference order (neighbour e of point p at p * 32 + e, then the centres);
    -1 for the missing points of a short tile."""
    start = t * TILE
    length = min(TILE, n - start)
    pts = order[b, start:start + length] if order is not None else np.arange(start, start + length)
    refs = np.full(REFS, -1, dtype=np.int64)
    for p, i in enumerate(pts):
        refs[p * 32:(p + 1) * 32] = nbr[b, i]
        refs[TILE * 32 + p] = i
    return refs


def check_plan(plan, nbr, order):
    """The plan of (nbr, order), tile by tile: its count is the number of distinct references, its ids are those rows once
    each, and every reference's slot holds its own row.  Returns the distinct counts [B,T]."""
    b, n, _ = nbr.shape
    tps = (n + TILE - 1) // TILE
    assert tuple(plan.shape[:2]) == (b, tps)
    count, ids, slots = decode(plan)
    nbr_np = nbr.cpu().numpy()
    order_np = None if order is None else order.cpu().numpy()
    for s in range(b):
        for t in range(tps):
            refs = tile_refs(nbr_np, order_np, s, t, n)
            valid = refs >= 0
            distinct = np.unique(refs[valid])
            c = int(count[s, t])
            assert c == len(distinct), (s, t)
            assert np.array_equal(np.sort(ids[s, t, :c]), distinct), (s, t)   # each distinct row once, all within sample s
            assert (slots[s, t, valid] < c).all()
            assert np.array_equal(ids[s, t, slots[s, t, valid]], refs[valid]), (s, t)
    return count


def graph(pc):
    from pvraft_b200 import ops
    nbr, rel = ops.knn(pc, pc, 32, mode=0, want_rel=True)
    return nbr, rel, ops.point_order(pc)


@pytest.mark.parametrize('order_kind', ['morton', 'index'])
def test_plan_against_numpy(dev, order_kind):
    from pvraft_b200 import ops
    b, n = 2, 8192
    pc, _ = O.synthetic_clouds(b, n, seed=21)
    nbr, _, morton = graph(pc.to(dev))
    order = morton if order_kind == 'morton' else None
    check_plan(ops.edge_plan(nbr, order), nbr, order)


def test_ragged_last_tile_within_sample(dev):
    """N = 7999: the last tile of each sample holds 31 points and references rows of its own sample only."""
    from pvraft_b200 import ops
    b, n = 3, 7999
    pc, _ = O.synthetic_clouds(b, n, seed=22)
    nbr, _, order = graph(pc.to(dev))
    plan = ops.edge_plan(nbr, order)
    assert plan.shape[1] == 250
    check_plan(plan, nbr, order)
    _, ids, slots = decode(plan)
    assert (slots[:, -1, 31 * 32:TILE * 32] == 0).all() and (slots[:, -1, TILE * 32 + 31:] == 0).all()


def test_sliced_plan_equals_own_plan(dev):
    """The plan of a 2B graph sliced to its first B samples names, for every reference, the same row as the plan of those
    B samples built alone (slot numbers may differ: they follow the hash's insertion order)."""
    from pvraft_b200 import ops
    b, n = 2, 8192
    pc1, pc2 = O.synthetic_clouds(b, n, seed=23)
    nbr, _, order = graph(torch.cat([pc1, pc2], 0).to(dev))
    whole = ops.edge_plan(nbr, order)[:b]
    own = ops.edge_plan(nbr[:b].contiguous(), order[:b].contiguous())
    cw, iw, sw = decode(whole)
    co, io, so = decode(own)
    assert np.array_equal(cw, co)
    assert np.array_equal(np.take_along_axis(iw, sw, 2), np.take_along_axis(io, so, 2))


def all_overflow(plan):
    """The same plan with every tile's count past any table: the edge kernel then gathers every tile from global memory."""
    forced = plan.clone()
    forced.view(torch.int32)[..., COUNT // 4] = REFS + 1
    return forced


@pytest.mark.parametrize('c', [16, 48, 64, 96, 128])
def test_table_equals_global_gather(dev, c):
    """A cloud whose Morton half fits the tables and whose shuffled half mostly does not: the plan's counts give the right
    overflow decision at this C's capacity, and the kernel's results from the tables are the bits of the all-global run,
    in the default form (maxima and minima; sums within double rounding) and in the deterministic form (everything)."""
    from pvraft_b200 import ops
    b, n, cin = 2, 8192, 32
    pc = torch.cat([O.synthetic_clouds(1, n, seed=c)[0], torch.rand(1, n, 3, generator=torch.Generator().manual_seed(c))]).to(dev)
    nbr, rel, order = graph(pc)
    order = order.clone()
    order[1] = torch.arange(n, dtype=torch.int32, device=dev)   # the random cloud in index order: most tiles overflow
    plan = ops.edge_plan(nbr, order)
    count = check_plan(plan, nbr, order)
    rows = min(REFS, TABLE_FLOATS // c)
    if c == 64:
        assert (count[0] <= rows).mean() > 0.9 and (count[1] > rows).mean() > 0.5
    g = torch.Generator().manual_seed(c)
    p = torch.randn(b, n, c, generator=g).to(dev)
    w = torch.randn(c, cin + 3, generator=g).to(dev)

    def run(pl, det):
        stats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            ymax, ymin = ops.setconv_edge(p, nbr, rel, w, cin, stats, order=order, plan=pl)
        finally:
            torch.use_deterministic_algorithms(prev)
        return ymax, ymin, stats

    forced = all_overflow(plan)
    for det in (False, True):
        a, z = run(plan, det), run(forced, det)
        assert torch.equal(a[0], z[0]) and torch.equal(a[1], z[1])
        if det:
            assert torch.equal(a[2], z[2])
        else:
            assert bool(((a[2] - z[2]).abs() <= 1e-12 * z[2].abs() + 1e-300).all())
    y = p.double()
    for s in range(b):
        ys = y[s][nbr[s].long()] - y[s].unsqueeze(1) + rel[s].double() @ w[:, cin:].double().t()
        assert float((a[0][s].double() - ys.amax(1)).abs().max() / ys.abs().amax()) < 1e-6


def test_plan_shape_mismatch_rejected(dev):
    from pvraft_b200 import ops
    pc, _ = O.synthetic_clouds(2, 1024, seed=24)
    nbr, rel, order = graph(pc.to(dev))
    plan = ops.edge_plan(nbr, order)
    p = torch.randn(2, 1024, 64, device=dev)
    w = torch.randn(64, 67, device=dev)
    stats = torch.zeros(2, 8, 2, dtype=torch.float64, device=dev)
    with pytest.raises(ValueError):
        ops.setconv_edge(p, nbr, rel, w, 64, stats, order=order, plan=plan[:1])
