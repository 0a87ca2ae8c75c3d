"""Scan sequences: the flow propagation kernel, RAFT's warm start (`forward(..., flow_init=)`) on every path of the model, and
`SceneFlowStream`.

Bounds: the kernel's neighbour sets are bit-exact against a numpy float32 restatement of the difference form and the tie
rule, its flows within 1e-6 (max-abs / max-abs) of a float64 inverse-distance weighting over those neighbours.  A warm-started
forward is held to test_gpu_parity.py's free-running bound against the oracle loop started at xyz1 + flow_init (mean-abs error
< 2e-3 of the mean |flow| at every iteration), a warm-started training step to test_gpu_train.py's gradient bounds.  Streams
are compared with per-pair calls bit for bit, under torch.use_deterministic_algorithms(True) at N % 128 == 0.
"""
import types

import numpy as np
import pytest
import torch

from conftest import default_weights
from oracle import pvraft_oracle as O
from test_gpu_deterministic import same_bits
from test_gpu_input_grads import deterministic
from test_gpu_train import leaf
from train_helpers import compare_grads, oracle_adjacency, sequence_loss

pytestmark = pytest.mark.gpu
K, ITERS = 128, 3


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module', autouse=True)
def _cpu_threads():
    old = torch.get_num_threads()
    torch.set_num_threads(min(16, old))
    yield
    torch.set_num_threads(old)


def args(k=K):
    return types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)


def make_model(dev, refine=False, seed=0, k=K):
    from pvraft_b200 import RSF, RSF_refine
    torch.manual_seed(seed)
    return (RSF_refine if refine else RSF)(args(k)).to(dev).eval()


def same(a, b):
    """Bitwise equality of two outputs (a tensor or a list of tensors)."""
    if torch.is_tensor(a):
        return torch.is_tensor(b) and a.shape == b.shape and same_bits(a, b)
    return len(a) == len(b) and all(x.shape == y.shape and same_bits(x, y) for x, y in zip(a, b))


def final(out):
    return out if torch.is_tensor(out) else out[-1]


def scan_sequence(b, sizes, seed=0):
    """Synthetic scans of one scene: every scan samples the scene anew (points do not correspond), the scene moves rigidly
    (a turn about z and a translation per scan) and a box in it moves on its own; 1 cm of noise."""
    g = torch.Generator().manual_seed(seed)
    scans = []
    for t, n in enumerate(sizes):
        pts = 10.0 * torch.rand(b, n, 3, generator=g)
        in_box = ((pts[..., 0] < 3) & (pts[..., 1] < 3)).unsqueeze(-1)
        a = 0.02 * t
        rot = torch.tensor([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
        pts = pts @ rot.T + torch.tensor([0.15, 0.05, 0.0]) * t + in_box * torch.tensor([0.0, 0.2, 0.0]) * t
        scans.append((pts + 0.01 * torch.randn(b, n, 3, generator=g)).contiguous())
    return scans


# ----------------------------------------------------------------------------------------------------------------------
# the propagation kernel
# ----------------------------------------------------------------------------------------------------------------------
def np_neighbours(xyz_prev, flow_prev, xyz, k):
    """float32 restatement: W = xyz_prev + flow_prev, d = (dx*dx + dy*dy) + dz*dz of q - W rounded at every step, the k least
    on (distance, index) -> [N,k] int64."""
    w = (xyz_prev + flow_prev).astype(np.float32)
    n, m = xyz.shape[0], w.shape[0]
    out = np.empty((n, k), dtype=np.int64)
    chunk = max(1, (1 << 22) // m)
    for q0 in range(0, n, chunk):
        q = xyz[q0:q0 + chunk]
        dx, dy, dz = (q[:, None, c] - w[None, :, c] for c in range(3))
        d = (dx * dx + dy * dy) + dz * dz
        out[q0:q0 + chunk] = np.argsort(d, axis=1, kind='stable')[:, :k]   # stable: equal distances keep index order
    return out


def np_idw(xyz_prev, flow_prev, xyz, idx):
    """float64 inverse-distance weighting over given neighbours."""
    w = (xyz_prev + flow_prev).astype(np.float32).astype(np.float64)
    d = ((xyz.astype(np.float64)[:, None, :] - w[idx]) ** 2).sum(-1)
    wt = 1.0 / (np.sqrt(d) + 1e-8)
    return (wt[..., None] * flow_prev.astype(np.float64)[idx]).sum(1) / wt.sum(1, keepdims=True)


def propagation_clouds(b, n, m, kind, seed):
    g = np.random.default_rng(seed)
    if kind == 'grid':      # integer coordinates and flows: many exact distance ties
        xyz_prev = g.integers(0, 6, (b, m, 3)).astype(np.float32)
        flow_prev = g.integers(-1, 2, (b, m, 3)).astype(np.float32)
        xyz = (g.integers(0, 12, (b, n, 3)) * 0.5).astype(np.float32)
        return xyz_prev, flow_prev, xyz
    xyz_prev = (10.0 * g.random((b, m, 3))).astype(np.float32)
    flow_prev = (0.3 * g.standard_normal((b, m, 3))).astype(np.float32)
    xyz = (10.0 * g.random((b, n, 3))).astype(np.float32)
    if kind == 'dup':       # every point twice, with the same flow; queries on some of the moved points
        xyz_prev[:, 1::2] = xyz_prev[:, :m // 2 * 2:2][:, :xyz_prev[:, 1::2].shape[1]]
        flow_prev[:, 1::2] = flow_prev[:, :m // 2 * 2:2][:, :flow_prev[:, 1::2].shape[1]]
        xyz[:, ::3] = (xyz_prev + flow_prev)[:, g.integers(0, m, xyz[:, ::3].shape[1])]
    if kind == 'shift':     # far from the origin, where the expanded form |q|^2 + |x|^2 - 2 q.x cancels
        xyz_prev += np.float32(1e3)
        xyz += np.float32(1e3)
    return xyz_prev, flow_prev, xyz


@pytest.mark.parametrize('b,n,m,k,kind', [
    (1, 32, 33, 1, 'random'), (2, 32, 33, 3, 'grid'), (1, 32, 33, 8, 'dup'),
    (2, 1000, 1537, 3, 'shift'), (1, 1000, 1537, 8, 'grid'), (1, 1000, 1537, 1, 'dup'),
    (1, 8192, 8192, 3, 'random'), (1, 20000, 5000, 8, 'shift'),
    (2, 40, 5, 5, 'random'), (1, 100, 8, 8, 'grid'),     # k = M
])
def test_propagation_against_numpy(dev, b, n, m, k, kind):
    from pvraft_b200 import ops
    xyz_prev, flow_prev, xyz = propagation_clouds(b, n, m, kind, seed=n + m + k)
    t = [torch.from_numpy(a).to(dev) for a in (xyz_prev, flow_prev, xyz)]
    flow, idx = ops.flow_propagate(*t, k=k, want_idx=True)
    assert flow.shape == (b, n, 3) and idx.shape == (b, n, k) and idx.dtype == torch.int32
    for s in range(b):
        want = np_neighbours(xyz_prev[s], flow_prev[s], xyz[s], k)
        assert np.array_equal(idx[s].cpu().numpy(), want), f'sample {s}: {(idx[s].cpu().numpy() != want).any(1).sum()} rows differ'
        ref = np_idw(xyz_prev[s], flow_prev[s], xyz[s], want)
        err = np.abs(flow[s].cpu().numpy() - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err < 1e-6, err
        one, one_idx = ops.flow_propagate(*(x[s:s + 1] for x in t), k=k, want_idx=True)   # a batch = its samples one by one
        assert same_bits(one[0], flow[s]) and torch.equal(one_idx[0], idx[s])
    assert same_bits(ops.flow_propagate(*t, k=k), flow)                  # with or without idx_out; reproducible


# ----------------------------------------------------------------------------------------------------------------------
# flow_init
# ----------------------------------------------------------------------------------------------------------------------
def pair(dev, b=2, n=1024, seed=5):
    pc1, pc2 = O.synthetic_clouds(b, n, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    init = 0.7 * (pc2 - pc1) + 0.02 * torch.randn(b, n, 3, generator=g)
    return pc1, pc2, init, [pc1.to(dev), pc2.to(dev)], init.to(dev)


@pytest.mark.parametrize('refine', [False, True])
@pytest.mark.parametrize('graphed', [False, True])
def test_zero_flow_init_is_none(dev, refine, graphed):
    m = make_model(dev, refine)
    m.use_cuda_graph = graphed
    _, _, init, p, _ = pair(dev)
    with torch.no_grad(), deterministic(True):
        cold = m(p, ITERS)
        zero = m(p, ITERS, flow_init=torch.zeros_like(p[0]))
    assert same(cold, zero)
    if graphed:
        assert len(m._graphs) == 2      # the warm start is a graph of its own


@pytest.mark.parametrize('refine', [False, True])
def test_replay_takes_new_flow_init(dev, refine):
    """flow_init is a static input of the graph: a new value replays the same capture and equals the eager forward."""
    m = make_model(dev, refine)
    _, _, init, p, f1 = pair(dev)
    f2 = 0.5 * f1.flip(1)
    with torch.no_grad(), deterministic(True):
        m.use_cuda_graph = True
        g1 = m(p, ITERS, flow_init=f1)
        captured = next(iter(m._graphs.values()))[0]
        g2 = m(p, ITERS, flow_init=f2)
        assert len(m._graphs) == 1 and next(iter(m._graphs.values()))[0] is captured
        m.use_cuda_graph = False
        e1, e2 = m(p, ITERS, flow_init=f1), m(p, ITERS, flow_init=f2)
        cold = m(p, ITERS)
    assert same(g1, e1) and same(g2, e2)
    assert not same(e1, e2) and not same(e1, cold)


def oracle_warm(P, xyz1, xyz2, flow_init, iters, refine=False, k=K):
    """model/RAFTSceneFlow.py:22-50 with the loop started at coords2 = xyz1 + flow_init (a constant), restated from the
    oracle's pieces."""
    li = O.prepare(P, xyz1, xyz2, k)
    coords1, coords2, net = xyz1, xyz1 + flow_init.detach(), li.net
    flows = []
    for _ in range(iters):
        coords2 = coords2.detach()
        corr = O.corr_lookup(P, li.state, coords2, 3, 0.25)
        flow = coords2 - coords1
        net, delta = O.update_block(P, net, li.inp, corr, flow, li.graph)
        coords2 = coords2 + delta
        flows.append(coords2 - coords1)
    return O.flot_refine(P, 'refine_block', flows[-1], li.feat_graph) if refine else flows


@pytest.mark.parametrize('refine', [False, True])
def test_warm_start_matches_oracle(dev, refine):
    m = make_model(dev, refine)
    W = {kk: v.detach().cpu() for kk, v in m.state_dict().items()}
    pc1, pc2, init, p, f = pair(dev, seed=13)
    with torch.no_grad():
        want = oracle_warm(W, pc1, pc2, init, ITERS, refine)
        got = m(p, ITERS, flow_init=f)
        cold = m(p, ITERS)
    for g, w in ([(got, want)] if refine else zip(got, want)):
        err = float((g.cpu() - w).abs().mean() / w.abs().mean())
        print(f'warm start vs oracle: {err:.2e}')
        assert err < 2e-3
    assert float((final(got) - final(cold)).abs().mean()) > 1e-3     # the start matters


def test_training_step_with_flow_init_matches_oracle(dev):
    """A 3-iteration stage-1 step from a warm start: the 95 parameter gradients and both input gradients against autograd
    through the warm-started oracle; flow_init itself receives none."""
    from pvraft_b200 import RSF
    b, n = 2, 1024
    W = default_weights(args=args(), seed=2)
    pc1, pc2 = O.synthetic_clouds(b, n, seed=11)
    pc1, pc2 = pc1 * 0.4, pc2 * 0.4
    gt = pc2 - pc1
    init = 0.6 * gt + 0.01 * torch.randn(b, n, 3, generator=torch.Generator().manual_seed(3))
    Wr = {kk: leaf(v) for kk, v in W.items()}
    x1r, x2r = leaf(pc1), leaf(pc2)
    flows_ref = oracle_warm(Wr, x1r, x2r, init, ITERS)
    sequence_loss(flows_ref, gt).backward()
    want = dict({kk: v.grad for kk, v in Wr.items()}, xyz1=x1r.grad, xyz2=x2r.grad)
    m = RSF(args())
    m.load_state_dict(W)
    m = m.to(dev).train()
    x1, x2, fi = leaf(pc1, dev), leaf(pc2, dev), leaf(init, dev)
    with oracle_adjacency():
        flows = m([x1, x2], num_iters=ITERS, flow_init=fi)
    for f, fr in zip(flows, flows_ref):
        assert float((f.detach().cpu() - fr.detach()).abs().mean()) < 1e-4 * float(fr.detach().abs().mean())
    sequence_loss(flows, gt.to(dev)).backward()
    got = {kk: q.grad for kk, q in m.named_parameters()}
    assert len(got) == 95 and all(v is not None for v in got.values())
    compare_grads(dict(got, xyz1=x1.grad, xyz2=x2.grad), want, 2e-2, 5e-2)
    assert fi.grad is None


def test_refine_training_with_flow_init(dev):
    """RSF_refine._forward_train: the loop under no_grad from the warm start, the refiner with gradients."""
    m = make_model(dev, refine=True)
    W = {kk: v.detach().cpu() for kk, v in m.state_dict().items()}
    pc1, pc2, init, p, f = pair(dev, seed=17)
    m.train()
    fi = f.clone().requires_grad_(True)
    with oracle_adjacency():
        refined = m(p, ITERS, flow_init=fi)
    Wr = {kk: leaf(v) for kk, v in W.items()}
    with oracle_adjacency():
        want = oracle_warm(Wr, pc1, pc2, init, ITERS, refine=True)
    assert float((refined.detach().cpu() - want.detach()).abs().mean()) < 2e-3 * float(want.detach().abs().mean())
    gt = pc2 - pc1
    (refined - gt.to(dev)).abs().sum(-1).mean().backward()
    (want - gt).abs().sum(-1).mean().backward()
    got = {kk: q.grad for kk, q in m.named_parameters() if q.grad is not None}
    assert len(got) == 29 and all(kk.startswith('refine_block.') for kk in got)
    compare_grads(got, {kk: Wr[kk].grad for kk in got}, 2e-2, 5e-2)
    assert fi.grad is None


@pytest.mark.parametrize('mode', ['bf16', 'bf16-compute', 'bf16-mixed'])
def test_precision_modes_take_flow_init(dev, mode):
    m = make_model(dev)
    _, _, _, p, f = pair(dev, seed=21)
    with torch.no_grad():
        full = m(p, ITERS, flow_init=f)
        m.set_precision(mode)
        low = m(p, ITERS, flow_init=f)
        with deterministic(True):
            zero = m(p, ITERS, flow_init=torch.zeros_like(f))
            cold = m(p, ITERS)
    err = float((low[-1] - full[-1]).abs().mean() / full[-1].abs().mean())
    print(f'{mode}: warm start vs fp32 {err:.2e}')
    assert err < 2e-2
    assert same(zero, cold)
    if mode == 'bf16-mixed':       # a training step from the warm start
        m.train()
        fi = f.clone().requires_grad_(True)
        flows = m(p, ITERS, flow_init=fi)
        sequence_loss(flows, (p[1] - p[0])).backward()
        assert all(q.grad is not None and bool(torch.isfinite(q.grad).all()) for q in m.parameters())
        assert fi.grad is None


def test_deterministic_warm_start_is_repeatable(dev):
    m = make_model(dev)
    m.use_cuda_graph = False
    _, _, _, p, f = pair(dev, seed=23)
    with deterministic(True):
        with torch.no_grad():
            a, b = m(p, ITERS, flow_init=f), m(p, ITERS, flow_init=f)
        assert same(a, b)
        m.train()
        grads = []
        for _ in range(2):
            m.zero_grad(set_to_none=True)
            sequence_loss(m(p, ITERS, flow_init=f), p[1] - p[0]).backward()
            grads.append([q.grad.clone() for q in m.parameters()])
        assert same(grads[0], grads[1])


def test_data_parallel_scatters_flow_init(dev):
    m = make_model(dev)
    m.use_cuda_graph = False
    _, _, _, p, f = pair(dev, seed=29)
    dp = torch.nn.DataParallel(m, device_ids=list(range(torch.cuda.device_count())))
    with torch.no_grad(), deterministic(True):
        assert same(dp(p, ITERS, flow_init=f), m(p, ITERS, flow_init=f))


# ----------------------------------------------------------------------------------------------------------------------
# SceneFlowStream
# ----------------------------------------------------------------------------------------------------------------------
EQUAL, UNEQUAL = (1024,) * 5, (1024, 1152, 896, 1280, 1024)


def pair_calls(m, scans, warm, k=3):
    """What a stream must return: per-pair model calls, warm-started from the previous pair's final flow."""
    from pvraft_b200 import ops
    outs, last = [None], None
    for t in range(1, len(scans)):
        init = ops.flow_propagate(scans[t - 2], last, scans[t - 1], k) if warm and last is not None else None
        outs.append(m([scans[t - 1], scans[t]], ITERS, flow_init=init))
        last = final(outs[-1])
    return outs


@pytest.mark.parametrize('refine', [False, True])
@pytest.mark.parametrize('sizes', [EQUAL, UNEQUAL], ids=['equal', 'unequal'])
@pytest.mark.parametrize('warm', [False, True], ids=['cold', 'warm'])
def test_stream_equals_pair_calls(dev, refine, sizes, warm):
    from pvraft_b200 import SceneFlowStream
    m = make_model(dev, refine)
    scans = [s.to(dev) for s in scan_sequence(2, sizes)]
    with torch.no_grad(), deterministic(True):
        want = pair_calls(m, scans, warm)
        st = SceneFlowStream(m, ITERS, warm_start=warm)
        got = [st.step(s) for s in scans]
    assert got[0] is None
    for t in range(1, len(scans)):
        assert same(got[t], want[t]), f'scan {t}'
    if warm:
        assert not same(want[-1], pair_calls(m, scans, False)[-1])


@pytest.mark.parametrize('refine', [False, True])
@pytest.mark.parametrize('b', [2, 3])
def test_stream_graphed_equals_eager(dev, refine, b):
    """Replayed steps (from the first step at B <= 2, from the second with the same shapes above) equal eager steps bit for
    bit, count the library's replayed kernels, and run the feature encoder once per step."""
    from pvraft_b200 import SceneFlowStream, ops
    m = make_model(dev, refine)
    scans = [s.to(dev) for s in scan_sequence(b, EQUAL, seed=b)]
    calls = []
    hook = m.feature_extractor.register_forward_hook(lambda *a: calls.append(1))
    try:
        with torch.no_grad(), deterministic(True):
            m.use_cuda_graph = False
            st = SceneFlowStream(m, ITERS)
            eager, launches = [], []
            for s in scans:
                n0, c0 = ops.launch_count, len(calls)
                eager.append(st.step(s))
                launches.append(ops.launch_count - n0)
                assert len(calls) - c0 == 1            # the new scan only
            m.use_cuda_graph = None
            st = SceneFlowStream(m, ITERS)
            graphed = []
            for t, s in enumerate(scans):
                n0, c0 = ops.launch_count, len(calls)
                graphed.append(st.step(s))
                if t == 4 or (t == 3 and b <= 2):      # replays of an existing capture
                    assert len(calls) == c0 and ops.launch_count - n0 == launches[t]
    finally:
        hook.remove()
    # B <= 2: the first scan, the cold second and the warm third (replayed for the rest); B = 3: the warm step, captured when
    # it came back at the fourth scan and replayed at the fifth
    assert len(m._stream_graphs) == (3 if b <= 2 else 1)
    for t in range(1, len(scans)):
        assert same(graphed[t], eager[t]), f'scan {t}'


def test_stream_follows_weights_and_precision(dev):
    """A weight change re-encodes the cached scan and captures the step again; set_precision drops the stream's graphs."""
    from pvraft_b200 import SceneFlowStream, ops
    m = make_model(dev)
    scans = [s.to(dev) for s in scan_sequence(1, EQUAL[:4], seed=7)]
    with torch.no_grad(), deterministic(True):
        st = SceneFlowStream(m, ITERS)
        outs = [st.step(s) for s in scans[:3]]
        key = st._key(dict(xyz1=scans[1], xyz=scans[2], src_xyz=scans[0]))   # (every warm step of this sequence)
        entry = m._stream_graphs[key]
        m.feature_extractor.feat_conv1.fc1.weight.mul_(1.01)           # a weight changes
        out = st.step(scans[3])
        assert m._stream_graphs[key] is not entry
        m.use_cuda_graph = False
        want = m([scans[2], scans[3]], ITERS, flow_init=ops.flow_propagate(scans[1], outs[2][-1], scans[2], 3))
        assert same(out, want)
        m.set_precision('fp32')
        assert '_stream_graphs' not in m.__dict__
