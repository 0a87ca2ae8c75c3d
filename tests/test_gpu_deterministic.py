"""Deterministic mode: while torch.use_deterministic_algorithms(True) is on, every reduction of the library runs in a fixed
order (exact fixed-point accumulation of values whose own order depends on the shapes only), so kernels, training steps and
forwards give the same bits on every run, eager or replayed, and a sample's forward does not depend on its batch (N % 128 == 0).
Inputs are built so that summation order matters: magnitudes log-uniform over 1e-6..1e2 with random signs, and hubs (many
rows adding into the same few destinations)."""
import types

import pytest
import torch

from conftest import default_weights
from oracle import pvraft_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture
def det():
    """Deterministic mode for one test; the flag and warn_only are restored afterwards."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def wild(*shape, g, dev):
    """Magnitudes log-uniform over 1e-6..1e2, random signs."""
    mag = 10.0 ** (torch.rand(*shape, generator=g) * 8 - 6)
    sign = torch.where(torch.rand(*shape, generator=g) < 0.5, -1.0, 1.0)
    return (mag * sign).float().to(dev)


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int64 if t.element_size() == 8 else torch.int32) if t.is_floating_point() else t


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


def three_runs(fn):
    """fn() -> tuple of tensors; asserts three calls give identical bits and returns the first."""
    outs = [tuple(t.clone() for t in fn()) for _ in range(3)]
    for o in outs[1:]:
        for x, y in zip(outs[0], o):
            assert same_bits(x, y)
    return outs[0]


def off(fn):
    """fn() with the flag off (the default, atomic path)."""
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        return tuple(t.clone() for t in fn())
    finally:
        torch.use_deterministic_algorithms(was)


def close(a, b, tol):
    a, b = a.double().cpu(), b.double().cpu()
    assert float((a - b).abs().max()) <= tol * float(b.abs().max().clamp_min(1e-30)), (float((a - b).abs().max()), float(b.abs().max()))


# ---- kernel level --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('b,n,cin,cout', [(2, 8192 * 32, 3, 64), (2, 8192, 128, 128), (1, 3001, 81, 48)])
def test_linear_wgrad(det, dev, b, n, cin, cout):
    from pvraft_b200 import ops
    g = torch.Generator().manual_seed(cin + cout)
    x, dy = wild(b, n, cin, g=g, dev=dev), wild(b, n, cout, g=g, dev=dev)

    def run():
        dw, db = torch.zeros(cout, cin, device=dev), torch.zeros(cout, device=dev)
        ops.linear_wgrad(x, dy, dw, db)
        return dw, db
    dw, db = three_runs(run)
    xd, dyd = x.double().reshape(-1, cin), dy.double().reshape(-1, cout)
    close(dw, dyd.t() @ xd, 2e-5)
    close(db, dyd.sum(0), 2e-5)
    aw, ab = off(run)
    close(dw, aw, 2e-5)
    close(db, ab, 2e-5)


@pytest.mark.parametrize('cin,cout', [(3, 64), (4, 64), (3, 128), (4, 32)])
def test_linear_bwd_small(det, dev, cin, cout):
    from pvraft_b200 import ops
    g = torch.Generator().manual_seed(7 * cin + cout)
    b, r = 2, 8192 * 32                                   # edge-level rows
    x, dy = wild(b, r, cin, g=g, dev=dev), wild(b, r, cout, g=g, dev=dev)
    w = wild(cout, cin, g=g, dev=dev)

    def run():
        dw, db = torch.zeros(cout, cin, device=dev), torch.zeros(cout, device=dev)
        dx = ops.linear_bwd_small(x, dy, w, dw, db, want_dx=True)
        return dw, db, dx
    dw, db, dx = three_runs(run)
    xd, dyd = x.double().reshape(-1, cin), dy.double().reshape(-1, cout)
    close(dw, dyd.t() @ xd, 2e-5)
    close(db, dyd.sum(0), 2e-5)
    close(dx.reshape(-1, cin), dyd @ w.double(), 1e-5)
    for a, o in zip((dw, db, dx), off(run)):
        close(a, o, 2e-5)


@pytest.mark.parametrize('arg', [False, True])
def test_gn_act_bwd(det, dev, arg):
    from pvraft_b200 import ops
    from pvraft_b200._lib import ACT_LRELU
    g = torch.Generator().manual_seed(5 + arg)
    b, rows, c = 2, 8192 * 32, 64
    x = torch.randn(b, rows, c, generator=g).to(dev)
    xs = x.double().reshape(b, rows, 8, c // 8)
    stats = torch.stack([xs.sum((1, 3)), (xs * xs).sum((1, 3))], -1).contiguous()
    gamma, beta = torch.randn(c, generator=g).to(dev), torch.randn(c, generator=g).to(dev)
    if arg:
        dy = wild(b, rows // 32, c, g=g, dev=dev)
        am = torch.randint(0, 32, (b, rows // 32, c), generator=g).to(torch.uint8).to(dev)
    else:
        dy, am = wild(b, rows, c, g=g, dev=dev), None

    def run():
        dx, dg, dbt, ds = ops.gn_act_bwd(x, dy, stats, gamma, beta, float(rows * c // 8), ACT_LRELU, 0.1, want_dslope=True, arg=am)
        return dx, dg, dbt, ds
    outs = three_runs(run)
    for a, o in zip(outs, off(run)):
        close(a, o, 1e-4)
    # float64 autograd reference: GroupNorm (statistics of x itself) + LeakyReLU with a learnable slope; in the arg form dy
    # reaches only row 32 * point + arg of each (point, channel)
    if arg:
        dyd = torch.zeros(b, rows // 32, 32, c, dtype=torch.float64, device=dev)
        dyd.scatter_(2, am.long().unsqueeze(2), dy.double().unsqueeze(2))
        dyd = dyd.reshape(b, rows, c)
    else:
        dyd = dy.double()
    xr = x.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    sl = torch.tensor(0.1, dtype=torch.float64, device=dev, requires_grad=True)
    xs = xr.reshape(b, rows, 8, c // 8)
    mean = xs.mean((1, 3), keepdim=True)
    var = ((xs - mean) ** 2).mean((1, 3), keepdim=True)
    t = ((xs - mean) / torch.sqrt(var + 1e-5)).reshape(b, rows, c) * gr + br
    y = torch.where(t >= 0, t, sl * t)
    (y * dyd).sum().backward()
    dx, dg, dbt, ds = outs
    close(dx, xr.grad, 1e-4)
    close(dg, gr.grad, 1e-4)
    close(dbt, br.grad, 1e-4)
    scale = float((dyd * t.detach()).abs()[t.detach() < 0].sum())   # dslope = sum over t < 0 of dy * t: may cancel
    assert abs(float(ds) - float(sl.grad)) <= 1e-6 * scale, (float(ds), float(sl.grad), scale)


def test_edge_fwd_and_bwd_with_hubs(det, dev):
    from pvraft_b200 import ops
    g = torch.Generator().manual_seed(3)
    b, n, c = 2, 8192, 64
    p = wild(b, n, c, g=g, dev=dev)
    nbr = torch.randint(0, 4, (b, n, 32), generator=g).to(torch.int32).to(dev)   # every point lists the same few neighbours
    e0 = wild(b, n * 32, c, g=g, dev=dev)
    dt = wild(b, n * 32, c, g=g, dev=dev)

    def fwd():
        stats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
        e = ops.edge_fwd(p, nbr, e0.clone(), stats)
        return e, stats

    def bwd():
        return (ops.edge_bwd(dt, nbr, torch.zeros(b, n, c, device=dev)),)
    e, stats = three_runs(fwd)
    ed = e.double().reshape(b, n * 32, 8, c // 8)
    close(stats, torch.stack([ed.sum((1, 3)), (ed * ed).sum((1, 3))], -1), 1e-6)
    (dp,) = three_runs(bwd)
    dtd = dt.double().reshape(b, n, 32, c)
    ref = torch.zeros(b, n, c, dtype=torch.float64, device=dev)
    ref.scatter_add_(1, nbr.long().reshape(b, n * 32, 1).expand(b, n * 32, c), dtd.reshape(b, n * 32, c))
    ref -= dtd.sum(2)
    close(dp, ref, 1e-5)
    close(dp, off(bwd)[0], 1e-5)
    close(stats, off(fwd)[1], 1e-6)


def test_corr_init_bwd_with_hubs(det, dev):
    from pvraft_b200 import ops
    g = torch.Generator().manual_seed(4)
    b, n, c, k = 2, 4096, 128, 64
    f1, f2 = wild(b, n, c, g=g, dev=dev), wild(b, n, c, g=g, dev=dev)
    idx = torch.randint(0, n, (b, n, k), generator=g)
    idx[:, :, :16] = torch.arange(16)                     # most rows keep the same 16 columns
    idx = idx.to(torch.int32).to(dev)
    gr = wild(b, n, k, g=g, dev=dev)

    def run():
        return ops.corr_init_bwd(gr, idx, f1, f2)
    d1, d2 = three_runs(run)
    s = c ** -0.5
    gd = gr.double()
    ref2 = torch.zeros(b, n, c, dtype=torch.float64, device=dev)
    ref2.scatter_add_(1, idx.long().reshape(b, n * k, 1).expand(b, n * k, c),
                      (gd.unsqueeze(-1) * f1.double().unsqueeze(2) * s).reshape(b, n * k, c))
    close(d2, ref2, 1e-5)
    a1, a2 = off(run)
    close(d2, a2, 1e-5)
    assert same_bits(d1, a1)                               # d f1 is a per-row gather: the same kernel arithmetic in both modes


def test_flow_metrics(det, dev):
    from pvraft_b200 import loss
    g = torch.Generator().manual_seed(6)
    b, n = 4, 8192
    est, gt = wild(b, n, 3, g=g, dev=dev), wild(b, n, 3, g=g, dev=dev)
    mask = (torch.rand(b, n, 1, generator=g) > 0.3).float().to(dev)
    batch = {'ground_truth': [mask, gt]}
    a = three_runs(lambda: (loss._metrics(est, gt, mask[..., 0].contiguous()),))[0]
    o = off(lambda: (loss._metrics(est, gt, mask[..., 0].contiguous()),))[0]
    close(a[:6], o[:6], 1e-6)
    e = (est - gt).double()[mask[..., 0] > 0]
    close(a[0], e.abs().sum(), 1e-6)
    assert float(a[1]) == e.shape[0]
    close(a[2], e.norm(dim=-1).sum(), 1e-6)
    ests = [wild(b, n, 3, g=g, dev=dev) for _ in range(3)]
    for fn in (lambda: loss.compute_loss(est, batch), lambda: loss.sequence_loss(ests, batch), lambda: loss.compute_epe_train(est, batch),
               lambda: torch.tensor(loss.compute_epe(est, batch), dtype=torch.float64)):
        three_runs(lambda: (fn(),))


# ---- statistics producers: repeatable and batch-invariant --------------------------------------------------------------------------
def knn_moments(sel):
    """[B,N,32,4] (c, dx, dy, dz) of the selected neighbours -> [B,15] float64 moments as the lookup accumulates them."""
    b = sel.shape[0]
    f = sel.double().reshape(b, -1, 4)
    iu = torch.triu_indices(4, 4)
    m = torch.zeros(b, 15, dtype=torch.float64, device=sel.device)
    m[:, :4] = f.sum(1)
    m[:, 4:14] = torch.einsum('bni,bnj->bij', f, f)[:, iu[0], iu[1]]
    m[:, 14] = f.shape[1]
    return m


@pytest.mark.parametrize('state_dtype', [torch.float32, torch.bfloat16])
def test_lookup_moments(det, dev, state_dtype):
    from pvraft_b200 import CorrBlock
    b, n, k = 4, 4096, 256
    state, coords, xyz2 = O.synthetic_state(b, n, k, seed=12, box=3.0)
    coords = coords.to(dev)

    def block(s0, s1):
        cb = CorrBlock(num_levels=3, base_scale=0.25, truncate_k=k).to(dev)
        cb.state_dtype = state_dtype
        cb.set_state(state.truncated_corr[s0:s1].to(dev), state.indices[s0:s1].to(torch.int32).to(dev), xyz2[s0:s1].to(dev))
        return cb
    cb = block(0, b)

    def run(cb=cb, s0=0, s1=b):
        out = cb.lookup(coords[s0:s1])
        return out['moments'], out['knn_sel']
    mom, sel = three_runs(run)
    close(mom[:, :15], knn_moments(sel), 1e-9)
    close(mom[:, :15], off(run)[0][:, :15], 1e-9)
    for i in range(b):                                     # a sample's moments do not depend on its batch
        assert same_bits(run(block(i, i + 1), i, i + 1)[0][0, :15], mom[i, :15]), i


def test_setconv_edge_stats(det, dev):
    from pvraft_b200 import ops
    b, n, c, cin = 4, 4096, 96, 64
    g = torch.Generator().manual_seed(c)
    pc, _ = O.synthetic_clouds(b, n, seed=c)
    pcd = pc.to(dev)
    nbr, rel = ops.knn(pcd, pcd, 32, mode=0, want_rel=True)
    P = wild(b, n, c, g=g, dev=dev)
    w = torch.randn(c, cin + 3, generator=g).to(dev)

    def run(s0=0, s1=b):
        stats = torch.zeros(s1 - s0, 8, 2, dtype=torch.float64, device=dev)
        ymax, ymin = ops.setconv_edge(P[s0:s1].contiguous(), nbr[s0:s1].contiguous(), rel[s0:s1].contiguous(), w, cin, stats)
        return stats, ymax, ymin
    stats, ymax, ymin = three_runs(run)
    we = w[:, cin:].double()
    for s in range(b):   # float64 reference, one sample at a time
        p = P[s].double()
        y = (p[nbr[s].long()] - p.unsqueeze(1) + rel[s].double() @ we.t()).reshape(n * 32, 8, c // 8)
        s1, s2, sabs = y.sum((0, 2)), (y ** 2).sum((0, 2)), y.abs().sum((0, 2))
        assert bool(((stats[s, :, 0] - s1).abs() <= 1e-5 * s1.abs() + 1e-7 * sabs).all()), (stats[s, :, 0], s1)
        assert bool(((stats[s, :, 1] - s2).abs() <= 1e-5 * s2).all()), (stats[s, :, 1], s2)
    a_stats, a_max, a_min = off(run)
    assert same_bits(ymax, a_max) and same_bits(ymin, a_min)   # max / min are not reductions: the same bits in both modes
    sabs = torch.stack([(a_stats[..., 0]).abs(), a_stats[..., 1].abs()], -1)
    assert bool(((stats - a_stats).abs() <= 1e-5 * sabs + 1e-9 * sabs.amax()).all())
    for i in range(b):                                     # a sample's statistics do not depend on its batch
        assert same_bits(run(i, i + 1)[0][0], stats[i]), i


def test_stats_producers_batch_invariant(det, dev):
    from pvraft_b200 import ops
    g = torch.Generator().manual_seed(8)
    n, c = 4096, 128
    x = wild(4, n, 64, g=g, dev=dev)
    w = (torch.randn(c, 64, generator=g) / 8).to(dev)
    bias = torch.randn(c, generator=g).to(dev)
    tw = ops.tc_weights(w)

    def producers(xb):
        bb = xb.shape[0]
        s_tc, s_lin = ops.new_stats(bb, dev)[0], ops.new_stats(bb, dev)[0]
        ops.tc_linear([xb], tw, bias, out_stats=s_tc)
        ops.linear(xb, w, bias, out_stats=s_lin)
        return s_tc, s_lin
    s_tc, s_lin = three_runs(lambda: producers(x))
    a_tc, a_lin = off(lambda: producers(x))
    close(s_tc, a_tc, 1e-6)
    close(s_lin, a_lin, 1e-6)
    for i in range(4):
        one_tc, one_lin = producers(x[i:i + 1].contiguous())
        assert same_bits(one_tc[0], s_tc[i]) and same_bits(one_lin[0], s_lin[i])


# ---- whole model -------------------------------------------------------------------------------------------------------------------
def _args(k=128):
    return types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)


def _step(dev, n, seed=0, iters=3):
    """One stage-1 step from fixed weights, inputs and a fresh Adam state -> (loss, grads, params after the step)."""
    from pvraft_b200 import RSF, loss
    W = default_weights(args=_args(), seed=2)
    pc1, pc2 = O.synthetic_clouds(2, n, seed=11 + seed)
    pc1, pc2 = (pc1 * 0.4).to(dev), (pc2 * 0.4).to(dev)
    m = RSF(_args())
    m.load_state_dict(W)
    m = m.to(dev).train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    batch = {'ground_truth': [torch.ones(2, n, 1, device=dev), pc2 - pc1]}
    flows = m([pc1, pc2], num_iters=iters)
    lo = loss.sequence_loss(flows, batch)
    lo.backward()
    grads = {k: p.grad.clone() for k, p in m.named_parameters()}
    opt.step()
    return lo.detach().clone(), grads, {k: p.detach().clone() for k, p in m.named_parameters()}


def _assert_steps_equal(a, b):
    assert same_bits(a[0], b[0])
    assert len(a[1]) == 95
    for k in a[1]:
        assert same_bits(a[1][k], b[1][k]), k
        assert same_bits(a[2][k], b[2][k]), k


@pytest.mark.parametrize('n,tc', [(1024, False), (1024, True), (1000, False)])
def test_stage1_step_is_bitwise_reproducible(det, dev, n, tc):
    from pvraft_b200 import train as T
    was = T._TC_TRAIN
    if tc:
        T._TC_TRAIN = '1'
    try:
        _assert_steps_equal(_step(dev, n), _step(dev, n))
    finally:
        T._TC_TRAIN = was


def test_refine_step_is_bitwise_reproducible(det, dev):
    from pvraft_b200 import RSF_refine
    W = default_weights(refine=True, args=_args(64), seed=4)
    pc1, pc2 = O.synthetic_clouds(2, 512, seed=21)
    pc1, pc2 = (pc1 * 0.4).to(dev), (pc2 * 0.4).to(dev)

    def run():
        m = RSF_refine(_args(64))
        m.load_state_dict(W)
        m = m.to(dev).train()
        refined = m([pc1, pc2], 4)
        (refined - (pc2 - pc1)).abs().sum(-1).mean().backward()
        return {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    a, b = run(), run()
    assert len(a) == 29
    for k in a:
        assert same_bits(a[k], b[k]), k


def test_gradients_match_oracle_in_deterministic_mode(det, dev):
    import test_gpu_train as TT
    TT.test_rsf_gradients_match_oracle(dev)


def _model(dev, refine=False, k=128):
    from pvraft_b200 import RSF, RSF_refine
    W = default_weights(refine=refine, args=_args(k), seed=1)
    m = (RSF_refine if refine else RSF)(_args(k))
    m.load_state_dict(W)
    return m.to(dev).eval()


@pytest.mark.parametrize('refine', [False, True])
def test_inference_eager_and_replay_bitwise(det, dev, refine):
    from pvraft_b200 import ops
    m = _model(dev, refine)
    if refine:                                             # the bf16 state mode: bf16 values + uint16 ids in the lookup
        m.set_precision('bf16')
        assert m.corr_block.state_dtype == torch.bfloat16
    pc1, pc2 = (t.to(dev) for t in O.synthetic_clouds(2, 1024, seed=3))
    with torch.no_grad():
        m.use_cuda_graph = False
        e1, e2 = m([pc1, pc2], 8), m([pc1, pc2], 8)
        m.use_cuda_graph = True
        r1, r2 = m([pc1, pc2], 8), m([pc1, pc2], 8)
    last = (lambda o: o) if refine else (lambda o: o[-1])
    assert same_bits(last(e1), last(e2)) and same_bits(last(r1), last(r2)) and same_bits(last(e1), last(r1))
    assert all(key[-1] is True for key in m._graphs)
    assert ops.deterministic()


def test_inference_batch_invariant(det, dev):
    m = _model(dev)
    m.use_cuda_graph = False
    pc1, pc2 = (t.to(dev) for t in O.synthetic_clouds(4, 1024, seed=9))
    with torch.no_grad():
        whole = m([pc1, pc2], 8)[-1]
        for i in range(4):
            assert same_bits(m([pc1[i:i + 1], pc2[i:i + 1]], 8)[-1][0], whole[i]), i


def test_windowed_build_forward_repeatable(det, dev):
    m = _model(dev, k=512)
    m.use_cuda_graph = False
    pc1, pc2 = (t.to(dev) for t in O.synthetic_clouds(1, 65536, seed=5))
    with torch.no_grad():
        a, b = m([pc1, pc2], 2)[-1], m([pc1, pc2], 2)[-1]
    assert same_bits(a, b)


def test_switching_takes_each_path_and_never_replays_across(dev):
    from pvraft_b200 import ops
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    m = _model(dev)
    m.use_cuda_graph = True
    pc1, pc2 = (t.to(dev) for t in O.synthetic_clouds(2, 1024, seed=3))
    outs, counts = [], []
    try:
        with torch.no_grad():
            for flag in (False, True, False):
                torch.use_deterministic_algorithms(flag)
                m([pc1, pc2], 8)                           # captures the setting's graph, or replays it
                n0 = ops.launch_count
                outs.append(m([pc1, pc2], 8)[-1])          # a replay
                counts.append(ops.launch_count - n0)
                assert (tuple(pc1.shape), pc1.device, 8, flag) in m._graphs
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    assert len(m._graphs) == 2                             # one graph per setting, the first re-used on the way back
    assert counts[0] == counts[1] == counts[2] > 0         # every deterministic entry point is one library call, as its default
    close(outs[1], outs[0], 1e-4)
