"""Gradient contract (SURVEY.md section 8b / 8c item 4): every autograd Function of the training path against PyTorch autograd on
the same op, and the whole model -- all 95 parameters of a stage-1 step, the 29 of `refine_block` in a refine step -- against
autograd through the CPU oracle.  Tolerances (max-abs difference / max-abs reference, per tensor):
    single layers          1e-5 (outputs), 2e-5 .. 1e-4 (gradients: fp32 atomics, other summation orders)
    whole-model gradients  per parameter tensor: relative L2 error < 2e-2, max-abs / max-abs < 5e-2 (measured worst 6.6e-3 stage 1,
                           2.6e-2 refine); cosine similarity of the full gradient vector > 0.99999 (measured 0.99999999 / 0.9999998)
(the per-tensor bound is looser because discrete routing decisions -- arg-max over the 32 neighbours, the sign of the L1 loss at
flow = target, top-K membership at near-ties -- may flip between two fp32 evaluations and move a gradient contribution).
"""
import types

import pytest
import torch
import torch.nn.functional as F

from conftest import default_weights, rel_err
from oracle import pvraft_oracle as O
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


def leaf(t, dev=None):
    t = t.clone().detach()
    if dev is not None:
        t = t.to(dev)
    return t.requires_grad_(True)


# ----------------------------------------------------------------------------------------------------------------------
# single Functions
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('b,r,cin,cout,bias', [(2, 300, 64, 64, True), (1, 1000, 81, 128, True), (2, 257, 3, 16, False),
                                               (1, 4096, 192, 128, True), (2, 130, 128, 3, True), (1, 70, 4, 64, True),
                                               (2, 4099, 3, 32, False), (1, 9000, 3, 128, True), (2, 2500, 4, 64, True), (1, 33, 2, 64, False),
                                               (1, 5000, 3, 16, False), (2, 3001, 3, 48, True), (1, 2777, 4, 96, True)])
def test_linear_fn(dev, b, r, cin, cout, bias):
    from pvraft_b200 import train as T
    g = torch.Generator().manual_seed(cin * 131 + cout)
    x, w = torch.randn(b, r, cin, generator=g), torch.randn(cout, cin, 1, generator=g) / cin ** 0.5
    bv = torch.randn(cout, generator=g) if bias else None
    gy = torch.randn(b, r, cout, generator=g)
    xr, wr, br = leaf(x).double(), leaf(w).double(), (leaf(bv).double() if bias else None)
    xr.retain_grad(); wr.retain_grad()
    if bias:
        br.retain_grad()
    yr = F.linear(xr, wr.reshape(cout, cin), br)
    yr.backward(gy.double())
    xd, wd, bd = leaf(x, dev), leaf(w, dev), (leaf(bv, dev) if bias else None)
    y, stats = T.linear(xd, wd, bd, True) if cout % 8 == 0 else (T.linear(xd, wd, bd), None)
    y.backward(gy.to(dev))
    assert rel_err(y.detach().cpu(), yr.detach()) < 1e-5
    assert rel_err(xd.grad.cpu(), xr.grad) < 2e-5
    assert rel_err(wd.grad.cpu(), wr.grad) < 5e-5 and wd.grad.shape == w.shape
    if bias:
        assert rel_err(bd.grad.cpu(), br.grad) < 5e-5
    if stats is not None:
        gs = yr.detach().reshape(b, r, 8, cout // 8)
        assert torch.allclose(stats[..., 0].cpu(), gs.sum((1, 3)), rtol=1e-5, atol=1e-3)


@pytest.mark.parametrize('b,r,cin,cout,bias,stats', [(2, 1024, 192, 64, True, True), (1, 2048, 64, 96, False, True),
                                                     (2, 512, 128, 61, True, False), (1, 256, 32, 128, True, True)])
def test_linear_fn_on_tensor_cores(dev, b, r, cin, cout, bias, stats):
    """The per-point layers of a CAPTURED training step run on the wgmma kernel (3xTF32), forward and dx (PVRAFT_TC_TRAIN=auto;
    forced here): same Function, same bounds as the CUDA-core path."""
    from pvraft_b200 import ops, train as T
    g = torch.Generator().manual_seed(cin * 7 + cout)
    x, w = torch.randn(b, r, cin, generator=g), torch.randn(cout, cin, 1, generator=g) / cin ** 0.5
    bv = torch.randn(cout, generator=g) if bias else None
    gy = torch.randn(b, r, cout, generator=g)
    xr, wr, br = leaf(x).double(), leaf(w).double(), (leaf(bv).double() if bias else None)
    xr.retain_grad(); wr.retain_grad()
    if bias:
        br.retain_grad()
    yr = F.linear(xr, wr.reshape(cout, cin), br)
    yr.backward(gy.double())
    xd, wd, bd = leaf(x, dev), leaf(w, dev), (leaf(bv, dev) if bias else None)
    was, n0 = T._TC_TRAIN, ops.launch_count
    T._TC_TRAIN = '1'
    try:
        out = T.linear(xd, wd, bd, stats)
        y, st = out if stats else (out, None)
        y.backward(gy.to(dev))
    finally:
        T._TC_TRAIN = was
    assert rel_err(y.detach().cpu(), yr.detach()) < 1e-5
    assert rel_err(xd.grad.cpu(), xr.grad) < 2e-5
    assert rel_err(wd.grad.cpu(), wr.grad) < 5e-5
    if bias:
        assert rel_err(bd.grad.cpu(), br.grad) < 5e-5
    if st is not None:
        gs = yr.detach().reshape(b, r, 8, cout // 8)
        assert torch.allclose(st[..., 0].cpu(), gs.sum((1, 3)), rtol=1e-5, atol=1e-3)
        assert torch.allclose(st[..., 1].cpu(), (gs ** 2).sum((1, 3)), rtol=1e-5, atol=1e-2)


@pytest.mark.parametrize('b,r,c,act', [(2, 512, 64, 'lrelu'), (1, 3000, 16, 'lrelu'), (2, 640, 48, 'lrelu'), (1, 2048, 128, 'prelu'),
                                       (2, 96, 96, 'none')])
def test_gn_act_fn(dev, b, r, c, act):
    from pvraft_b200 import ops, train as T
    g = torch.Generator().manual_seed(c + r)
    x = torch.randn(b, r, c, generator=g) * 1.7 + 0.4
    gamma, beta = torch.randn(c, generator=g), torch.randn(c, generator=g) * 0.2
    slope = torch.tensor([0.25])
    gy = torch.randn(b, r, c, generator=g)
    xr, gr, br, sr = leaf(x).double(), leaf(gamma).double(), leaf(beta).double(), leaf(slope).double()
    for t in (xr, gr, br, sr):
        t.retain_grad()
    n = F.group_norm(xr.transpose(1, 2), 8, gr, br, 1e-5).transpose(1, 2)
    yr = {'lrelu': lambda t: F.leaky_relu(t, 0.1), 'prelu': lambda t: torch.where(t >= 0, t, sr * t), 'none': lambda t: t}[act](n)
    yr.backward(gy.double())
    xd, gd, bd, sd = leaf(x, dev), leaf(gamma, dev), leaf(beta, dev), leaf(slope, dev)
    xs = xd.detach().double().reshape(b, r, 8, c // 8)
    stats = torch.stack([xs.sum((1, 3)), (xs ** 2).sum((1, 3))], -1).contiguous()
    code = ops.ACT_NONE if act == 'none' else ops.ACT_LRELU
    y = T.GnActFn.apply(xd, stats, gd, bd, sd if act == 'prelu' else None, code, 0.25 if act == 'prelu' else 0.1)
    y.backward(gy.to(dev))
    assert rel_err(y.detach().cpu(), yr.detach()) < 1e-5
    assert rel_err(xd.grad.cpu(), xr.grad) < 5e-5
    assert rel_err(gd.grad.cpu(), gr.grad) < 5e-5 and rel_err(bd.grad.cpu(), br.grad) < 5e-5
    if act == 'prelu':
        assert rel_err(sd.grad.cpu(), sr.grad) < 5e-5


@pytest.mark.parametrize('b,pts,c,act', [(2, 64, 64, 'lrelu'), (1, 301, 16, 'lrelu'), (2, 40, 128, 'prelu'), (1, 17, 96, 'none')])
def test_gn_act_max_fn(dev, b, pts, c, act):
    """GroupNorm + activation + max over 32 rows as one Function: values, arg-max routing and every gradient against autograd
    of the unfused float64 chain (the backward never builds the dense gradient of the max)."""
    from pvraft_b200 import ops, train as T
    r = pts * 32
    g = torch.Generator().manual_seed(c + pts)
    x = torch.randn(b, r, c, generator=g) * 1.7 + 0.4
    gamma, beta = torch.randn(c, generator=g), torch.randn(c, generator=g) * 0.2
    slope = torch.tensor([0.25])
    gy = torch.randn(b, pts, c, generator=g)
    xr, gr, br, sr = leaf(x).double(), leaf(gamma).double(), leaf(beta).double(), leaf(slope).double()
    for t in (xr, gr, br, sr):
        t.retain_grad()
    n = F.group_norm(xr.transpose(1, 2), 8, gr, br, 1e-5).transpose(1, 2)
    a = {'lrelu': lambda t: F.leaky_relu(t, 0.1), 'prelu': lambda t: torch.where(t >= 0, t, sr * t), 'none': lambda t: t}[act](n)
    yr = a.view(b, pts, 32, c).max(2).values
    yr.backward(gy.double())
    xd, gd, bd, sd = leaf(x, dev), leaf(gamma, dev), leaf(beta, dev), leaf(slope, dev)
    xs = xd.detach().double().reshape(b, r, 8, c // 8)
    stats = torch.stack([xs.sum((1, 3)), (xs ** 2).sum((1, 3))], -1).contiguous()
    code = ops.ACT_NONE if act == 'none' else ops.ACT_LRELU
    y = T.GnActMaxFn.apply(xd, stats, gd, bd, sd if act == 'prelu' else None, code, 0.25 if act == 'prelu' else 0.1)
    y.backward(gy.to(dev))
    assert y.shape == (b, pts, c)
    assert rel_err(y.detach().cpu(), yr.detach()) < 1e-5
    assert rel_err(xd.grad.cpu(), xr.grad) < 5e-5
    assert rel_err(gd.grad.cpu(), gr.grad) < 5e-5 and rel_err(bd.grad.cpu(), br.grad) < 5e-5
    if act == 'prelu':
        assert rel_err(sd.grad.cpu(), sr.grad) < 5e-5


def test_edge_and_max_fn(dev):
    from pvraft_b200 import train as T
    b, n, c = 2, 200, 48
    g = torch.Generator().manual_seed(3)
    p, e = torch.randn(b, n, c, generator=g), torch.randn(b, n * 32, c, generator=g)
    nbr = torch.randint(0, n, (b, n, 32), generator=g).to(torch.int32)
    gy = torch.randn(b, n, c, generator=g)
    pr, er = leaf(p).double(), leaf(e).double()
    pr.retain_grad(); er.retain_grad()
    gathered = torch.gather(pr.unsqueeze(1).expand(b, n, n, c), 2, nbr.long().unsqueeze(-1).expand(b, n, 32, c))
    tr = gathered - pr.unsqueeze(2) + er.view(b, n, 32, c)
    yr = tr.max(2).values
    yr.backward(gy.double())
    pd, ed = leaf(p, dev), leaf(e, dev)
    t, stats = T.EdgeFn.apply(pd, ed * 1.0, nbr.to(dev))          # (* 1.0: the edge stage works in place on a non-leaf)
    y = T.MaxKFn.apply(t)
    y.backward(gy.to(dev))
    assert rel_err(y.detach().cpu(), yr.detach()) < 1e-6
    assert rel_err(t.detach().cpu().view(b, n, 32, c), tr.detach()) < 1e-6
    assert rel_err(pd.grad.cpu(), pr.grad) < 1e-5 and rel_err(ed.grad.cpu(), er.grad) < 1e-6
    ts = tr.detach().reshape(b, n * 32, 8, c // 8)
    assert torch.allclose(stats[..., 0].cpu(), ts.sum((1, 3)), rtol=1e-5, atol=1e-3)
    assert torch.allclose(stats[..., 1].cpu(), (ts ** 2).sum((1, 3)), rtol=1e-5, atol=1e-3)


@pytest.mark.parametrize('b,n,k,box,levels,scale', [(2, 256, 64, 3.0, 3, 0.25), (1, 1024, 512, 10.0, 3, 0.25), (1, 300, 32, 3.0, 2, 0.3)])
def test_corr_lookup_fn_backward(dev, b, n, k, box, levels, scale):
    """d(voxel means, kNN correlations)/d(truncated correlation) against autograd through the oracle (model/corr.py:47-66,84)."""
    from pvraft_b200 import CorrBlock, ops, train as T
    state, coords, xyz2 = O.synthetic_state(b, n, k, seed=n + k, box=box)
    cb = CorrBlock(num_levels=levels, base_scale=scale, truncate_k=k).to(dev)
    cb.set_state(state.truncated_corr.to(dev), state.indices.to(torch.int32).to(dev), xyz2.to(dev))
    stored = O.CorrState(leaf(cb.corr_val.cpu()), cb.corr_idx.long().cpu(), cb.truncate_xyz2.cpu())
    g = torch.Generator().manual_seed(1)
    g_vox, g_sel = torch.randn(b, n, levels * 27, generator=g), torch.randn(b, n * 32, 4, generator=g)
    cv = leaf(cb.corr_val)
    vox, sel = T.CorrLookupFn.apply(cv, cb.corr_idx, cb._xyz2p, coords.to(dev), levels, scale)
    (vox * g_vox.to(dev)).sum().add((sel * g_sel.to(dev)).sum()).backward()
    # oracle: same slots (ties at the 32nd distance may legitimately pick another slot), its own cells / counts
    slots = ops.corr_lookup(cb.corr_val, cb.corr_idx, cb._xyz2p, coords.to(dev), levels, scale, want_slots=True)['knn_slot'].long().cpu()
    want_vox = O.voxel_means(stored, coords, levels, scale).transpose(1, 2)
    want_sel = O.knn_gather(stored, coords, slots).permute(0, 2, 3, 1).reshape(b, n * 32, 4)
    ((want_vox * g_vox).sum() + (want_sel * g_sel).sum()).backward()
    assert rel_err(vox.detach().cpu(), want_vox.detach()) < 1e-6
    assert rel_err(cv.grad.cpu(), stored.truncated_corr.grad) < 1e-5


@pytest.mark.parametrize('b,n,c,k', [(2, 256, 128, 64), (1, 384, 64, 128)])
def test_corr_init_fn_backward(dev, b, n, c, k):
    """Sparse backward of the truncated correlation against the dense autograd of model/corr.py:31-40,95-100."""
    from pvraft_b200 import CorrBlock, train as T
    g = torch.Generator().manual_seed(n + c)
    f1, f2 = torch.randn(b, n, c, generator=g), torch.randn(b, n, c, generator=g)
    cb = CorrBlock(truncate_k=k)
    a, d = leaf(f1, dev), leaf(f2, dev)
    val, idx = T.CorrInitFn.apply(a, d, k, cb)
    gv = torch.randn(b, n, k, generator=g)
    (val * gv.to(dev)).sum().backward()
    ar, dr = leaf(f1).double(), leaf(f2).double()
    ar.retain_grad(); dr.retain_grad()
    corr = torch.matmul(ar, dr.transpose(1, 2)) / c ** 0.5
    picked = torch.gather(corr, 2, idx.long().cpu())               # the same entries, in the stored order
    assert rel_err(val.detach().cpu(), picked.detach()) < 2e-6
    (picked * gv.double()).sum().backward()
    assert rel_err(a.grad.cpu(), ar.grad) < 2e-5 and rel_err(d.grad.cpu(), dr.grad) < 2e-5


# ----------------------------------------------------------------------------------------------------------------------
# whole model
# ----------------------------------------------------------------------------------------------------------------------
def test_rsf_gradients_match_oracle(dev):
    """SURVEY 8c item 4: a 3-iteration training step, N=1024, B=2 -- every one of the 95 parameters."""
    from pvraft_b200 import RSF
    b, n, k, iters = 2, 1024, 128, 3
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    W = default_weights(args=args, seed=2)
    pc1, pc2 = O.synthetic_clouds(b, n, seed=11)
    pc1, pc2 = pc1 * 0.4, pc2 * 0.4                       # dense enough for non-empty voxel cells at every level
    gt = pc2 - pc1
    Wr = {kk: leaf(v) for kk, v in W.items()}
    flows_ref = O.rsf_forward(Wr, pc1, pc2, iters, 3, 0.25, k)
    sequence_loss(flows_ref, gt).backward()
    want = {kk: v.grad for kk, v in Wr.items()}
    assert all(v is not None and float(v.abs().max()) > 0 for v in want.values())     # all 95 receive gradient (SURVEY 8b)
    m = RSF(args)
    m.load_state_dict(W)
    m = m.to(dev).train()
    with oracle_adjacency():
        flows = m([pc1.to(dev), pc2.to(dev)], num_iters=iters)
    assert isinstance(flows, list) and len(flows) == iters and flows[-1].requires_grad
    for f, fr in zip(flows, flows_ref):
        assert float((f.detach().cpu() - fr.detach()).abs().mean()) < 1e-4 * float(fr.detach().abs().mean())
    loss = sequence_loss(flows, gt.to(dev))
    assert abs(float(loss) - float(sequence_loss([f.detach() for f in flows_ref], gt))) < 1e-4 * abs(float(loss))
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters()}
    assert len(got) == 95 and all(v is not None for v in got.values())
    compare_grads(got, want, 2e-2, 5e-2)        # measured: 6.6e-3 max-abs, cosine 0.99999999


def test_rsf_refine_gradients_match_oracle(dev):
    """Stage 2 (tools/engine_refine.py): the RAFT loop runs under no_grad on the fused kernels, only refine_block trains."""
    from pvraft_b200 import RSF_refine
    b, n, k, iters = 2, 512, 64, 4
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    W = default_weights(refine=True, args=args, seed=4)
    pc1, pc2 = O.synthetic_clouds(b, n, seed=21)
    pc1, pc2 = pc1 * 0.4, pc2 * 0.4
    gt = pc2 - pc1
    Wr = {kk: (leaf(v) if kk.startswith('refine_block.') else v.clone()) for kk, v in W.items()}
    with torch.no_grad():
        li = O.prepare(Wr, pc1, pc2, k)
        flow_ref = O.raft_loop(Wr, li, pc1, iters, 3, 0.25)[-1]
    refined_ref = O.flot_refine(Wr, 'refine_block', flow_ref, li.feat_graph)
    (refined_ref - gt).abs().sum(-1).mean().backward()
    want = {kk: v.grad for kk, v in Wr.items() if kk.startswith('refine_block.')}
    m = RSF_refine(args)
    m.load_state_dict(W)
    m = m.to(dev).train()
    with oracle_adjacency():
        refined = m([pc1.to(dev), pc2.to(dev)], iters)
    assert float((refined.detach().cpu() - refined_ref.detach()).abs().mean()) < 2e-3 * float(refined_ref.detach().abs().mean())
    (refined - gt.to(dev)).abs().sum(-1).mean().backward()
    got = {kk: p.grad for kk, p in m.named_parameters() if p.grad is not None}
    assert set(got) == set(want) and len(got) == 29            # only refine_block.* (SURVEY 8b)
    compare_grads(got, want, 2e-2, 5e-2)        # measured: 2.6e-2 max-abs (one GroupNorm bias), cosine 0.9999998


def test_training_steps_like_the_engine(dev):
    """tools/engine.py:131-147 in miniature: Adam(lr=1e-3), sequence loss, backward, step -- twice; then evaluation with the
    updated weights through the fused inference path (derived weight copies must follow the optimizer's in-place updates)."""
    from pvraft_b200 import RSF
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=64)
    torch.manual_seed(0)
    m = RSF(args).to(dev).train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(2, 512, seed=31)]
    gt = pc2 - pc1
    losses = []
    for _ in range(3):
        opt.zero_grad()
        flows = m([pc1, pc2], num_iters=2)
        loss = sequence_loss(flows, gt)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(torch.isfinite(torch.tensor(losses))) and losses[-1] < losses[0], losses
    m.eval()
    with torch.no_grad():
        ev = m([pc1, pc2], 2)
        Wn = {kk: v.detach().cpu() for kk, v in m.state_dict().items()}
        want = O.rsf_forward(Wn, pc1.cpu(), pc2.cpu(), 2, 3, 0.25, 64)
    assert float((ev[-1].cpu() - want[-1]).abs().mean()) < 1e-2 * float(want[-1].abs().mean())


def test_whole_model_gradients_with_tensor_core_layers(dev):
    """The same training step with the per-point layers on the wgmma kernel (what a captured step runs) and on the CUDA-core
    kernels: all 95 gradients agree (both are fp32-accurate; N = 1024 so that the tensor-core shapes apply)."""
    from pvraft_b200 import RSF, train as T
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=128)
    torch.manual_seed(0)
    m = RSF(args).to(dev).train()
    pc1, pc2 = [t.to(dev) * 0.4 for t in O.synthetic_clouds(2, 1024, seed=9)]
    gt = pc2 - pc1
    grads = {}
    was = T._TC_TRAIN
    try:
        for mode in ('0', '1'):
            T._TC_TRAIN = mode
            m.zero_grad(set_to_none=True)
            sequence_loss(m([pc1, pc2], num_iters=3), gt).backward()
            grads[mode] = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    finally:
        T._TC_TRAIN = was
    assert len(grads['1']) == 95
    compare_grads(grads['1'], {k: v.cpu() for k, v in grads['0'].items()}, 2e-2, 5e-2)


def test_device_side_loss_and_metrics(dev):
    """pvraft_b200.loss (and the tools/loss.py, tools/metric.py drop-ins) against the reference formulas restated in torch / numpy
    (tools/loss.py:4-40, tools/metric.py:6-79), forward and backward, with a partial mask."""
    import numpy as np
    from tools.loss import sequence_loss as seq_loss
    from tools.metric import compute_epe, compute_epe_train
    g = torch.Generator().manual_seed(0)
    b, n = 2, 700
    mask = (torch.rand(b, n, 1, generator=g) > 0.3).float()
    gt = torch.randn(b, n, 3, generator=g) * 0.5
    ests = [gt + torch.randn(b, n, 3, generator=g) * s for s in (0.4, 0.2, 0.05)]
    batch = {'ground_truth': [mask.to(dev), gt.to(dev)]}
    xs = [leaf(e, dev) for e in ests]
    loss = seq_loss(xs, batch, gamma=0.8)
    loss.backward()
    xr = [leaf(e) for e in ests]
    want = 0
    for i, e in enumerate(xr):
        err = (e - gt)[mask[..., 0] > 0]
        want = want + 0.8 ** (2 - i) * torch.mean(torch.abs(err))
    want.backward()
    assert abs(float(loss) - float(want)) < 1e-6 * abs(float(want))
    for a, r in zip(xs, xr):
        assert rel_err(a.grad.cpu(), r.grad) < 1e-6
    epe = compute_epe_train(xs[-1].detach(), batch)
    assert epe.is_cuda and epe.dim() == 0
    m = mask.numpy()[..., 0]
    sf_gt, sf_pred = gt.numpy()[m > 0], ests[-1].numpy()[m > 0]
    l2 = np.linalg.norm(sf_gt - sf_pred, axis=-1)
    rel = l2 / (np.linalg.norm(sf_gt, axis=-1) + 1e-4)
    ref = (l2.mean(), np.logical_or(l2 < 0.05, rel < 0.05).mean(), np.logical_or(l2 < 0.1, rel < 0.1).mean(),
           np.logical_or(l2 > 0.3, rel > 0.1).mean())
    assert abs(float(epe) - ref[0]) < 1e-6
    got = compute_epe(xs[-1].detach(), batch)
    assert all(abs(a - float(r)) < 2e-3 for a, r in zip(got, ref)), (got, ref)       # threshold counts may differ by a point at the edge


def test_batch_pins_once_and_moves_with_one_copy(dev):
    from pvraft_b200.data import Batch
    g = torch.Generator().manual_seed(2)
    items = [{'sequence': [torch.rand(1, 64, 3, generator=g), torch.rand(1, 64, 3, generator=g)],
              'ground_truth': [torch.ones(1, 64, 1), torch.randn(1, 64, 3, generator=g)]} for _ in range(2)]
    want = [torch.cat([it['sequence'][0] for it in items], 0), torch.cat([it['ground_truth'][1] for it in items], 0)]
    bt = Batch(items).pin_memory()
    assert bt['sequence'][0].is_pinned()
    bt = bt.to(dev)
    assert bt['sequence'][0].is_cuda and torch.equal(bt['sequence'][0].cpu(), want[0]) and torch.equal(bt['ground_truth'][1].cpu(), want[1])
