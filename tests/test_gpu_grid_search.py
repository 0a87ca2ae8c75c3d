"""The uniform-grid searches against the brute-force forms of the same entry points: ops.chamfer, ops.laplacian and
ops.flow_propagate with use_grid=True / False, and ops.knn beyond 16 384 points against use_sweep=False.  The neighbours, and
their order, must be the same bits; so must every per-point value computed from them.  Sample sums may differ in summation
order only.  Then the deterministic forms, a captured loss step, a warm-started stream and a whole RSF forward at 20 000
points, each against its brute-force run."""
import contextlib
import math

import pytest
import torch

from test_gpu_input_grads import deterministic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def cloud(n, kind, g, dev):
    """[1,n,3] float32 clouds of the named distribution."""
    def r(*s):
        return torch.rand(*s, generator=g, device=dev)
    if kind == 'uniform':
        x = r(n, 3) * 40 - 20
    elif kind == 'lidar':   # rings on a ground plane, dense clusters, a sparse far range
        n1, n2 = n // 2, n // 4
        n3 = n - n1 - n2
        ring = torch.randint(0, 32, (n1,), generator=g, device=dev).float()
        rad = 3 + ring * 1.5 + r(n1) * 0.02
        th = r(n1) * 2 * math.pi
        ground = torch.stack([rad * torch.cos(th), rad * torch.sin(th), -1.7 + r(n1) * 0.05], 1)
        ctr = (r(8, 3) * 30 - 15)[torch.randint(0, 8, (n2,), generator=g, device=dev)]
        clusters = ctr + torch.randn(n2, 3, generator=g, device=dev) * 0.3
        far = torch.cat([r(n3, 2) * 160 - 80, r(n3, 1) * 6 - 2], 1)
        x = torch.cat([ground, clusters, far])[torch.randperm(n, generator=g, device=dev)]
    elif kind == 'flat':
        x = torch.cat([r(n, 2) * 30 - 15, torch.zeros(n, 1, device=dev)], 1)
    elif kind == 'collinear':
        t = r(n, 1) * 50 - 25
        x = torch.cat([t, 0.5 * t + 1, -t], 1)
    elif kind == 'one_cell':
        x = 3.0 + r(n, 3) * 1e-6
    elif kind == 'duplicated':
        base = r(max(1, n // 8), 3) * 10
        x = base[torch.randint(0, base.shape[0], (n,), generator=g, device=dev)]
    elif kind == 'int_ties':   # exact distance ties everywhere
        x = torch.randint(-6, 7, (n, 3), generator=g, device=dev).float()
    elif kind == 'shift1e3':
        x = r(n, 3) * 20 + 1e3
    elif kind == 'shift1e4':
        x = r(n, 3) * 20 + 1e4
    else:
        raise ValueError(kind)
    return x.reshape(1, n, 3).contiguous()


KINDS = ['uniform', 'lidar', 'flat', 'collinear', 'one_cell', 'duplicated', 'int_ties', 'shift1e3', 'shift1e4', 'outside']
SIZES = [(64, 65), (1000, 1537), (16385, 16385), (20000, 5000), (40000, 60000)]


def pair(n, m, kind, seed, dev):
    """(queries [1,n,3], searched [1,m,3]); 'outside': uniform searched points, queries spread far beyond their box."""
    g = torch.Generator(device=dev).manual_seed(seed)
    if kind == 'outside':
        return (torch.rand(1, n, 3, generator=g, device=dev) * 200 - 100).contiguous(), cloud(m, 'uniform', g, dev)
    return cloud(n, kind, g, dev), cloud(m, kind, g, dev)


def same(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.uint8) if a.dtype == torch.float64 else a, b.view(torch.uint8)
                                              if b.dtype == torch.float64 else b)


def close_sums(a, b, rel=1e-12):
    return torch.allclose(a, b, rtol=rel, atol=0.0)


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('n, m', SIZES, ids=[f'{n}x{m}' for n, m in SIZES])
def test_neighbours_match_brute_force(dev, n, m, kind):
    from pvraft_b200 import ops
    q, x = pair(n, m, kind, n + m, dev)
    flow = (torch.randn(1, m, 3, generator=torch.Generator(device=dev).manual_seed(1), device=dev) * 0.05).contiguous()
    for k in (1, 3, 5, 8):
        fg, ig = ops.flow_propagate(x, flow, q, k, want_idx=True, use_grid=True)
        fb, ib = ops.flow_propagate(x, flow, q, k, want_idx=True, use_grid=False)
        assert same(ig, ib), f'propagation neighbours, k={k}'
        assert same(fg, fb), f'propagated flow, k={k}'
    acc_g, ab_g, ba_g = ops.chamfer(q, x, use_grid=True)
    acc_b, ab_b, ba_b = ops.chamfer(q, x, use_grid=False)
    assert same(ab_g, ab_b) and same(ba_g, ba_b)
    assert close_sums(acc_g, acc_b)


@pytest.mark.parametrize('kind', ['uniform', 'lidar', 'int_ties', 'duplicated', 'shift1e4', 'outside'])
@pytest.mark.parametrize('k_int', [1, 3, 5, 8])
def test_laplacian_matches_brute_force(dev, kind, k_int):
    from pvraft_b200 import ops
    n, m, b, preds = 20000, 12000, 2, 2
    clouds = [pair(n, m, kind, 7 + i, dev) for i in range(b)]
    p1, p2 = torch.cat([c[0] for c in clouds]).contiguous(), torch.cat([c[1] for c in clouds]).contiguous()
    w = (p1.repeat(preds, 1, 1) + torch.randn(preds * b, n, 3, device=dev) * 0.05).contiguous()
    g1, g2 = ops.knn(p1, p1, 10, mode=0), ops.knn(p2, p2, 10, mode=0)
    l2 = ops.cloud_laplacian(p2, g2)
    acc_g, idx_g, res_g = ops.laplacian(w, p2, l2, g1, k_int, use_grid=True)
    acc_b, idx_b, res_b = ops.laplacian(w, p2, l2, g1, k_int, use_grid=False)
    assert same(idx_g, idx_b) and same(res_g, res_b)
    assert close_sums(acc_g, acc_b)


def test_largest_clouds_match_brute_force(dev):
    """131 072 x 131 072: every grid row, brute force on every row (the propagation and Chamfer kernels take it whole)."""
    from pvraft_b200 import ops
    for kind in ('uniform', 'lidar'):
        q, x = pair(131072, 131072, kind, 3, dev)
        flow = torch.zeros_like(x)
        fg, ig = ops.flow_propagate(x, flow, q, 8, want_idx=True, use_grid=True)
        fb, ib = ops.flow_propagate(x, flow, q, 8, want_idx=True, use_grid=False)
        assert same(ig, ib) and same(fg, fb), kind
        acc_g, ab_g, ba_g = ops.chamfer(q, x, use_grid=True)
        acc_b, ab_b, ba_b = ops.chamfer(q, x, use_grid=False)
        assert same(ab_g, ab_b) and same(ba_g, ba_b) and close_sums(acc_g, acc_b), kind


@pytest.mark.parametrize('mode', [0, 1])
@pytest.mark.parametrize('k', [9, 10, 32])
@pytest.mark.parametrize('n', [16385, 40000, 100000])
def test_knn_graph_beyond_sort_limit(dev, n, k, mode):
    """ops.knn on the counting-sort index == the brute-force kernel, indices and rel bitwise (all of a 2-sample batch's
    points as queries up to 40 000; 4096 of them at 100 000)."""
    from pvraft_b200 import ops
    g = torch.Generator(device=dev).manual_seed(n + k)
    b = 2 if n <= 40000 else 1
    xyz = torch.cat([cloud(n, 'lidar', g, dev), cloud(n, 'uniform', g, dev)])[:b].contiguous()
    q = xyz if n <= 40000 else xyz[:, torch.randperm(n, generator=g, device=dev)[:4096]].contiguous()
    assert ops.lib().pvraft_knn_workspace_bytes(b, n) == ops.lib().pvraft_grid_index_workspace_bytes(b, n)
    ig, rg = ops.knn(xyz, q, k, mode=mode, want_rel=True)
    ib, rb = ops.knn(xyz, q, k, mode=mode, want_rel=True, use_sweep=False)
    assert same(ig, ib) and same(rg, rb)


def test_index_is_a_permutation_and_repeatable(dev):
    """The index holds every point once, in cells of non-decreasing id; searches on it are the same bits from run to run
    even though the order inside a cell may differ."""
    from pvraft_b200 import ops
    q, x = pair(30000, 50000, 'lidar', 11, dev)
    s, n = 1, x.shape[1]
    ws = torch.empty(int(ops.lib().pvraft_grid_index_workspace_bytes(s, n)), dtype=torch.uint8, device=dev)
    ops.check(ops.lib().pvraft_grid_index_fwd(x.data_ptr(), None, s, n, ws.data_ptr(), ops._stream()), 'grid_index')
    ids = ws[16 * n:20 * n].view(torch.int32)
    assert torch.equal(ids.sort().values, torch.arange(n, dtype=torch.int32, device=dev))
    pts = ws[:16 * n].view(torch.float32).view(n, 4)[:, :3]
    assert torch.equal(pts, x[0][ids.long()])
    runs = [ops.flow_propagate(x, torch.zeros_like(x), q, 8, want_idx=True, use_grid=True) for _ in range(3)]
    runs += [ops.chamfer(q, x, use_grid=True) for _ in range(2)]
    assert all(same(a, b) for a, b in zip(runs[0], runs[1])) and all(same(a, b) for a, b in zip(runs[0], runs[2]))
    with deterministic(True):
        c1, c2 = ops.chamfer(q, x, use_grid=True), ops.chamfer(q, x, use_grid=True)
    assert all(same(a, b) for a, b in zip(c1, c2))


def test_deterministic_forms_batch_and_repeat(dev):
    """DET: one launch over S = n B equals n single-prediction calls, and repeats, for Chamfer and the Laplacian term."""
    from pvraft_b200 import ops
    b, preds, n, m = 2, 3, 20000, 17000
    g = torch.Generator(device=dev).manual_seed(5)
    p1 = torch.cat([cloud(n, 'lidar', g, dev) for _ in range(b)]).contiguous()
    p2 = torch.cat([cloud(m, 'lidar', g, dev) for _ in range(b)]).contiguous()
    w = (p1.repeat(preds, 1, 1) + torch.randn(preds * b, n, 3, generator=g, device=dev) * 0.1).contiguous()
    g1, g2 = ops.knn(p1, p1, 10, mode=0), ops.knn(p2, p2, 10, mode=0)
    l2 = ops.cloud_laplacian(p2, g2)
    with deterministic(True):
        ch = ops.chamfer(w, p2, use_grid=True)
        lp = ops.laplacian(w, p2, l2, g1, 5, use_grid=True)
        assert all(same(a, c) for a, c in zip(ch, ops.chamfer(w, p2, use_grid=True)))
        assert all(same(a, c) for a, c in zip(lp, ops.laplacian(w, p2, l2, g1, 5, use_grid=True)))
        for i in range(preds):
            wi = w[i * b:(i + 1) * b].contiguous()
            chi, lpi = ops.chamfer(wi, p2, use_grid=True), ops.laplacian(wi, p2, l2, g1, 5, use_grid=True)
            assert same(chi[0], ch[0][i * b:(i + 1) * b]) and same(chi[1], ch[1][i * b:(i + 1) * b])
            assert same(lpi[0], lp[0][i * b:(i + 1) * b]) and same(lpi[2], lp[2][i * b:(i + 1) * b])
        brute = ops.chamfer(w, p2, use_grid=False)
    assert same(ch[1], brute[1]) and same(ch[2], brute[2]) and close_sums(ch[0], brute[0])


@contextlib.contextmanager
def forced(ops, grid):
    """Every op picks the grid form (grid=True) or the brute-force form at every size, as the models and losses call them."""
    saved = dict(ops.GRID_SEARCH_MIN_POINTS)
    ops.GRID_SEARCH_MIN_POINTS.update({k: 1 if grid else 1 << 40 for k in saved})
    try:
        yield
    finally:
        ops.GRID_SEARCH_MIN_POINTS.update(saved)


def loss_grads(flow, pc1, pc2, grid, det):
    """Gradient of the three-term self-supervised loss w.r.t. the flow (and the loss), with the grid forms on or off."""
    from pvraft_b200 import ops
    from pvraft_b200.loss import self_supervised_loss
    with forced(ops, grid), deterministic(det):
        f = flow.clone().requires_grad_(True)
        loss = self_supervised_loss(f, {'sequence': [pc1, pc2]}, w_laplacian=0.3)
        loss.backward()
    return loss.detach(), f.grad


def test_loss_gradients_grid_vs_brute(dev):
    g = torch.Generator(device=dev).manual_seed(9)
    pc1 = torch.cat([cloud(20000, 'lidar', g, dev) for _ in range(2)]).contiguous()
    pc2 = (pc1 + torch.randn(pc1.shape, generator=g, device=dev) * 0.2).contiguous()
    flow = torch.randn(pc1.shape, generator=g, device=dev) * 0.1
    lg, gg = loss_grads(flow, pc1, pc2, True, True)
    lb, gb = loss_grads(flow, pc1, pc2, False, True)
    assert same(gg, gb), 'DET gradients: same indices, unchanged backward kernels'
    assert torch.allclose(lg, lb, rtol=1e-6, atol=0)
    # default mode: fp32 atomics in a varying order, against the exact (fixed-point) sums of the DET form
    lg, gg = loss_grads(flow, pc1, pc2, True, False)
    assert float((gg - gb).abs().max()) <= 1e-5 * float(gb.abs().max())
    assert torch.allclose(lg, lb, rtol=1e-6, atol=0)


def test_captured_loss_step_equals_eager(dev):
    """Forward (the flow moves the first cloud) + three-term loss + backward, on the grid forms, captured into one CUDA graph:
    bitwise the eager step under deterministic algorithms."""
    from pvraft_b200 import ops
    from pvraft_b200.loss import self_supervised_loss
    g = torch.Generator(device=dev).manual_seed(4)
    pc1 = torch.cat([cloud(16400, 'lidar', g, dev) for _ in range(2)]).contiguous()
    pc2 = (pc1 + torch.randn(pc1.shape, generator=g, device=dev) * 0.2).contiguous()
    f = (torch.randn(pc1.shape, generator=g, device=dev) * 0.1).requires_grad_(True)
    assert ops.use_grid_search('chamfer', pc1.shape[1]) and ops.use_grid_search('laplacian', pc1.shape[1])

    def step():
        f.grad = None
        loss = self_supervised_loss(f * 1.0, {'sequence': [pc1, pc2]}, w_laplacian=0.3)
        loss.backward()
        return loss.detach().clone(), f.grad.clone()

    with deterministic(True):
        want = step()
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            step()
        torch.cuda.current_stream(dev).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loss = self_supervised_loss(f * 1.0, {'sequence': [pc1, pc2]}, w_laplacian=0.3)
            loss.backward()
        f.grad.zero_()
        graph.replay()
        torch.cuda.synchronize()
    assert same(loss.detach(), want[0]) and same(f.grad, want[1])


def test_stream_warm_start_at_20000_points(dev):
    """SceneFlowStream at 20 000-point scans: its grid propagation equals the brute-force one, bitwise under the flag."""
    from pvraft_b200 import ops, SceneFlowStream
    from test_gpu_flow_stream import ITERS, make_model
    from test_gpu_flow_stream import same as stream_same
    m = make_model(dev)
    g = torch.Generator(device=dev).manual_seed(2)
    base = cloud(20000, 'lidar', g, dev)
    scans = [(base + 0.3 * t + torch.randn(base.shape, generator=g, device=dev) * 0.01).contiguous() for t in range(3)]
    outs = {}
    for grid in (True, False):
        with forced(ops, grid), torch.no_grad(), deterministic(True):
            st = SceneFlowStream(m, ITERS, warm_start=True)
            outs[grid] = [st.step(s) for s in scans]
    assert all(stream_same(a, b) for a, b in zip(outs[True][1:], outs[False][1:]))


def test_rsf_forward_at_20000_points_equals_brute_force_graphs(dev, monkeypatch):
    """An RSF forward at N1 = N2 = 20 000 (its kNN graphs beyond the shared-memory sort) under deterministic algorithms is
    bitwise the forward whose ops.knn is forced to the brute-force kernel."""
    from pvraft_b200 import ops
    from test_gpu_flow_stream import ITERS, make_model
    from test_gpu_flow_stream import same as stream_same
    m = make_model(dev)
    g = torch.Generator(device=dev).manual_seed(8)
    pc1 = cloud(20000, 'lidar', g, dev)
    pc2 = (pc1 + torch.randn(pc1.shape, generator=g, device=dev) * 0.1).contiguous()
    with torch.no_grad(), deterministic(True):
        grid = m([pc1, pc2], ITERS)
        real_knn = ops.knn
        monkeypatch.setattr(ops, 'knn', lambda *a, **kw: real_knn(*a, **{**kw, 'use_sweep': False}))
        brute = m([pc1, pc2], ITERS)
    assert stream_same(grid, brute)
