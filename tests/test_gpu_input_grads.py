"""Gradients into the input clouds (model/RAFTSceneFlow.py:22-50, model/RAFTSceneFlowRefine.py:22-48): `xyz1.requires_grad_()`
/ `xyz2.requires_grad_()` give input gradients through plain autograd, with trainable or frozen weights.
    * the lookup's table gradient (pvraft_corr_lookup_xyz_bwd) and the graph's edge features (pvraft_edge_bwd with C = 3)
      against float64 autograd, in the default and the deterministic mode;
    * the whole model against autograd through the CPU oracle on the oracle's adjacency, with the bounds of
      train_helpers.compare_grads, for RSF (equal and unequal clouds, N % 128 != 0) and RSF_refine;
    * frozen weights, bitwise repeatability in deterministic mode, and a captured frozen-weight step.
"""
import contextlib
import types

import pytest
import torch

from conftest import default_weights, rel_err
import unequal_oracle as U
from oracle import pvraft_oracle as O
from test_gpu_deterministic import same_bits
from test_gpu_train import leaf
from test_gpu_unequal_clouds import unequal_state
from train_helpers import compare_grads, oracle_adjacency, sequence_loss

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module', autouse=True)
def _cpu_threads():
    old = torch.get_num_threads()
    torch.set_num_threads(min(16, old))
    yield
    torch.set_num_threads(old)


@contextlib.contextmanager
def deterministic(flag):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(flag)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def args(k, levels=3, scale=0.25):
    return types.SimpleNamespace(corr_levels=levels, base_scales=scale, truncate_k=k)


# ----------------------------------------------------------------------------------------------------------------------
# single Functions
# ----------------------------------------------------------------------------------------------------------------------
def hub_state(b, n, m, k, dev, seed=3):
    """Every query sits on a cluster of 40 rows of xyz2 that are candidates of every row: all N*32 selections land on them."""
    g = torch.Generator().manual_seed(seed)
    xyz2 = 4.0 * torch.rand(b, m, 3, generator=g)
    xyz2[:, :40] = 5.0 + 0.05 * torch.rand(b, 40, 3, generator=g)
    rest = torch.argsort(torch.rand(b, n, m - 40, generator=g), dim=2)[..., :k - 40] + 40
    idx = torch.cat([torch.arange(40).expand(b, n, 40), rest], 2)
    idx = torch.gather(idx, 2, torch.argsort(torch.rand(b, n, k, generator=g), dim=2))
    coords = 5.0 + 0.05 * torch.rand(b, n, 3, generator=g)
    corr = torch.sort(torch.randn(b, n, k, generator=g) * 5 + 20, dim=2, descending=True).values
    return corr.to(dev), idx.to(dev), coords.to(dev).contiguous(), xyz2.to(dev).contiguous()


@pytest.mark.parametrize('case', ['spread-128', 'spread-512', 'hubs-128', 'hubs-512'])
@pytest.mark.parametrize('det', [False, True])
def test_lookup_table_gradient_against_float64(dev, case, det):
    """d xyz2 of the kNN 4-vectors (knn_xyz = xyz2[corr_idx[slot]] - coords) against float64 autograd, N != M; d corr is the
    same bits with and without it."""
    from pvraft_b200 import CorrBlock, ops, train as T
    kind, k = case.split('-')
    b, n, m, k, levels, scale = 2, 700, 1100, int(k), 3, 0.25
    corr, idx, coords, xyz2 = (hub_state(b, n, m, k, dev) if kind == 'hubs' else unequal_state(b, n, m, k, 7 * k, 3.0, dev))
    cb = CorrBlock(num_levels=levels, base_scale=scale, truncate_k=k).to(dev)
    cb.set_state(corr, idx, xyz2)
    g = torch.Generator().manual_seed(k)
    g_vox, g_sel = torch.randn(b, n, levels * 27, generator=g).to(dev), torch.randn(b, n * 32, 4, generator=g).to(dev)

    def run(with_xyz2):
        cv, x2 = leaf(cb.corr_val), leaf(xyz2)
        vox, sel = T.CorrLookupFn.apply(cv, cb.corr_idx, cb._xyz2p, coords, levels, scale, x2 if with_xyz2 else None)
        ((vox * g_vox).sum() + (sel * g_sel).sum()).backward()
        return cv.grad, x2.grad, sel.detach()

    with deterministic(det):
        d_corr, d_xyz2, sel = run(True)
        d_corr0, none, _ = run(False)
        again = run(True)
    assert none is None and same_bits(d_corr, d_corr0)
    if det:
        assert same_bits(d_xyz2, again[1])
    slots = ops.corr_lookup(cb.corr_val, cb.corr_idx, cb._xyz2p, coords, levels, scale, want_slots=True)['knn_slot'].long()
    ids = torch.gather(cb.corr_idx.long(), 2, slots).cpu()                                   # [B,N,32] rows of xyz2
    if kind == 'hubs':
        assert int(ids.max()) < 40                                                          # every selection is a hub
    x2r = leaf(xyz2.double().cpu())
    want = torch.gather(x2r, 1, ids.reshape(b, -1, 1).expand(b, n * 32, 3)) - coords.double().cpu().repeat_interleave(32, 1)
    assert rel_err(sel[..., 1:].cpu(), want.detach()) < 1e-6
    (want * g_sel[..., 1:].double().cpu()).sum().backward()
    assert rel_err(d_xyz2.cpu(), x2r.grad) < 1e-5


@pytest.mark.parametrize('det', [False, True])
def test_graph_edge_features_backward(dev, det):
    """Graph.construct_graph(pc).edge_feats is differentiable w.r.t. pc (model/flot/graph.py:72), with the kNN kernel's values."""
    from pvraft_b200 import Graph
    b, n = 2, 1000
    g = torch.Generator().manual_seed(5)
    pc = leaf(3.0 * torch.rand(b, n, 3, generator=g), dev)
    gr = torch.randn(b * n * 32, 3, generator=g)
    with deterministic(det):
        graph = Graph.construct_graph(pc, 32)
        assert graph.edge_feats.requires_grad
        graph.edge_feats.backward(gr.to(dev))
        plain = Graph.construct_graph(pc.detach(), 32)
        if det:
            grad0 = pc.grad.clone()
            pc.grad = None
            Graph.construct_graph(pc, 32).edge_feats.backward(gr.to(dev))
            assert same_bits(pc.grad, grad0)
    assert torch.equal(plain.nbr, graph.nbr) and same_bits(plain._rel, graph._rel)
    nbr = graph.nbr.long().cpu()
    pr = leaf(pc.detach().double().cpu())
    rel = torch.gather(pr.unsqueeze(1).expand(b, n, n, 3), 2, nbr.unsqueeze(-1).expand(b, n, 32, 3)) - pr.unsqueeze(2)
    assert rel_err(graph._rel.detach().cpu(), rel.detach()) < 1e-6
    (rel.reshape(-1, 3) * gr.double()).sum().backward()
    assert rel_err(pc.grad.cpu(), pr.grad) < 1e-5


# ----------------------------------------------------------------------------------------------------------------------
# whole model against the oracle
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n1, n2, k', [(1024, 1024, 128), (384, 640, 64), (1000, 1000, 128)])
def test_rsf_input_gradients_match_oracle(dev, n1, n2, k):
    """A 3-iteration step at B = 2: with trainable weights every parameter and both clouds, with frozen weights both clouds
    and no parameter, against autograd through the oracle (equal clouds; unequal clouds; N % 128 != 0, the CUDA-core layers)."""
    from pvraft_b200 import RSF
    b, iters = 2, 3
    W = default_weights(args=args(k), seed=2)
    pc1, pc2 = O.synthetic_clouds(b, n2, seed=11)          # n1 <= n2: xyz2's first n1 points move those of xyz1
    s = 0.4 * (n1 / 1024) ** (1 / 3)                          # the point density of test_gpu_train's 1024-point step
    pc1, pc2 = pc1[:, :n1] * s, pc2 * s
    gt = pc2[:, :n1] - pc1
    Wr = {kk: leaf(v) for kk, v in W.items()}
    x1r, x2r = leaf(pc1), leaf(pc2)
    flows_ref = (O.rsf_forward if n1 == n2 else U.rsf_forward)(Wr, x1r, x2r, iters, 3, 0.25, k)
    sequence_loss(flows_ref, gt).backward()
    want = dict({kk: v.grad for kk, v in Wr.items()}, xyz1=x1r.grad, xyz2=x2r.grad)
    assert float(want['xyz1'].abs().max()) > 0 and float(want['xyz2'].abs().max()) > 0
    m = RSF(args(k))
    m.load_state_dict(W)
    m = m.to(dev).train()
    for frozen in (False, True):
        m.requires_grad_(not frozen)
        m.zero_grad(set_to_none=True)
        x1, x2 = leaf(pc1, dev), leaf(pc2, dev)
        with oracle_adjacency():
            flows = m([x1, x2], num_iters=iters)
        assert len(flows) == iters and all(f.requires_grad for f in flows)
        for f, fr in zip(flows, flows_ref):
            assert float((f.detach().cpu() - fr.detach()).abs().mean()) < 1e-4 * float(fr.detach().abs().mean())
        sequence_loss(flows, gt.to(dev)).backward()
        got = {kk: p.grad for kk, p in m.named_parameters() if p.grad is not None}
        if frozen:
            assert not got
            compare_grads({'xyz1': x1.grad, 'xyz2': x2.grad}, {kk: want[kk] for kk in ('xyz1', 'xyz2')}, 2e-2, 5e-2)
        else:
            assert len(got) == 95
            compare_grads(dict(got, xyz1=x1.grad, xyz2=x2.grad), want, 2e-2, 5e-2)


def test_rsf_refine_input_gradient_matches_oracle(dev):
    """RSF_refine: the loop runs under no_grad, so xyz1 receives minus the refiner's input-flow gradient and xyz2 none."""
    from pvraft_b200 import RSF_refine
    b, n, k, iters = 2, 512, 64, 4
    W = default_weights(refine=True, args=args(k), seed=4)
    pc1, pc2 = O.synthetic_clouds(b, n, seed=21)
    pc1, pc2 = pc1 * 0.4, pc2 * 0.4
    gt = pc2 - pc1
    Wr = {kk: (leaf(v) if kk.startswith('refine_block.') else v.clone()) for kk, v in W.items()}
    x1r, trace = leaf(pc1), []
    with torch.no_grad():
        li = O.prepare(Wr, pc1, pc2, k)
        O.raft_loop(Wr, li, pc1, iters, 3, 0.25, trace=trace)
    coords2 = trace[-1]['coords'] + trace[-1]['delta']
    refined_ref = O.flot_refine(Wr, 'refine_block', coords2 - x1r, li.feat_graph)       # RAFTSceneFlowRefine.py:46
    (refined_ref - gt).abs().sum(-1).mean().backward()
    want = dict({kk: v.grad for kk, v in Wr.items() if kk.startswith('refine_block.')}, xyz1=x1r.grad)
    m = RSF_refine(args(k))
    m.load_state_dict(W)
    m = m.to(dev).train()
    x1, x2 = leaf(pc1, dev), leaf(pc2, dev)
    with oracle_adjacency():
        refined = m([x1, x2], iters)
    assert float((refined.detach().cpu() - refined_ref.detach()).abs().mean()) < 2e-3 * float(refined_ref.detach().abs().mean())
    (refined - gt.to(dev)).abs().sum(-1).mean().backward()
    assert x2.grad is None
    got = {kk: p.grad for kk, p in m.named_parameters() if p.grad is not None}
    assert set(got) == set(want) - {'xyz1'}
    compare_grads(dict(got, xyz1=x1.grad), want, 2e-2, 5e-2)
    with oracle_adjacency(), deterministic(True):             # the refiner's input values do not change
        assert same_bits(m([leaf(pc1, dev), x2.detach()], iters), m([x1.detach(), x2.detach()], iters))


def test_refine_bf16_state_rejects_input_gradients(dev):
    from pvraft_b200 import RSF, RSF_refine
    torch.manual_seed(0)
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(1, 256, seed=3)]
    for cls in (RSF, RSF_refine):
        m = cls(args(64)).to(dev).set_precision('bf16').requires_grad_(False)
        with pytest.raises(NotImplementedError):
            m([pc1.clone().requires_grad_(), pc2], 2)


# ----------------------------------------------------------------------------------------------------------------------
# frozen weights, deterministic mode, capture
# ----------------------------------------------------------------------------------------------------------------------
def test_deterministic_input_gradients(dev):
    """Under torch.use_deterministic_algorithms(True): two identical steps give the same bits of xyz1.grad / xyz2.grad, frozen
    weights give the same bits as trainable ones, and the flows are the same bits with and without input gradients."""
    from pvraft_b200 import RSF
    b, n, k, iters = 2, 1024, 128, 3
    torch.manual_seed(0)
    m = RSF(args(k)).to(dev).train()
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(b, n, seed=41)]
    gt = pc2 - pc1

    def step(frozen, inputs=True):
        m.requires_grad_(not frozen)
        m.zero_grad(set_to_none=True)
        x1, x2 = (leaf(pc1), leaf(pc2)) if inputs else (pc1, pc2)
        flows = m([x1, x2], num_iters=iters)
        sequence_loss(flows, gt).backward()
        return x1.grad, x2.grad, flows[-1].detach()

    with deterministic(True):
        a, b_, c = step(False), step(False), step(True)
        plain = step(False, inputs=False)
    for x, y in ((a, b_), (a, c)):
        assert same_bits(x[0], y[0]) and same_bits(x[1], y[1]) and same_bits(x[2], y[2])
    assert same_bits(a[2], plain[2])
    assert float(a[0].abs().max()) > 0 and float(a[1].abs().max()) > 0


@pytest.mark.parametrize('det', [False, True])
def test_captured_frozen_weight_step(dev, det):
    """A frozen-weight forward and backward into the inputs, captured into one CUDA graph (no host synchronisation): replays
    agree with eager within the oracle bounds, and two replays give the same bits in deterministic mode."""
    from pvraft_b200 import RSF
    b, n, k, iters = 2, 1024, 128, 3
    torch.manual_seed(0)
    m = RSF(args(k)).to(dev).train().requires_grad_(False)
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(b, n, seed=51)]
    gt = pc2 - pc1
    x1, x2 = leaf(pc1), leaf(pc2)

    def step():
        sequence_loss(m([x1, x2], num_iters=iters), gt).backward()

    with deterministic(det):
        step()
        eager = {'xyz1': x1.grad.clone().cpu(), 'xyz2': x2.grad.clone().cpu()}
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                x1.grad = x2.grad = None
                step()
        torch.cuda.current_stream().wait_stream(side)
        x1.grad = x2.grad = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        replays = []
        for _ in range(2):
            graph.replay()
            torch.cuda.synchronize()
            replays.append((x1.grad.clone(), x2.grad.clone()))
    compare_grads({'xyz1': replays[0][0], 'xyz2': replays[0][1]}, eager, 2e-2, 5e-2)
    if det:
        assert same_bits(replays[0][0], replays[1][0]) and same_bits(replays[0][1], replays[1][1])
