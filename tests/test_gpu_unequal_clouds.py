"""Pairs of clouds of different sizes, p = [xyz1 [B,N1,3], xyz2 [B,N2,3]], on the device.

  * the truncated state [B,N1,K] of corr_build against a float64 reference (dense and windowed builds, N2 > 49152 too), and
    the windowed build bit-identical to the dense one on forced small windows
  * the lookup with a gather table of N2 rows, on both sides of the shared-memory table limit: cell ids bit-exact, kNN slot
    sets, voxel means with the count clamped by N1 (N1 < K), fp32 and bf16 state; its backward against float64 autograd
  * the bf16 state's limit applies to N2
  * RSF / RSF_refine against the reference's own modules (unequal_rsf.npz), teacher-forced and free-running
  * CUDA-graph replay against eager, and pairs that share N1 but differ in N2
  * training: whole-model gradients against autograd through the oracle, corr_init_bwd against the sparse formula, and
    bitwise-repeatable steps under torch.use_deterministic_algorithms(True)
"""
import math
import types

import pytest
import torch

from conftest import load_golden, rel_err
import unequal_oracle as U
from oracle import pvraft_oracle as O
from test_gpu_large_clouds import same_bits
from test_gpu_train import leaf
from train_helpers import compare_grads, oracle_adjacency, sequence_loss

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def feature_maps(b, n, m, c, seed, dev):
    g = torch.Generator().manual_seed(seed)
    s = torch.linspace(0.5, 2.0, b).view(b, 1, 1)
    f1 = torch.randn(b, n, c, generator=g) * s + 0.1 * s
    f2 = torch.randn(b, m, c, generator=g) * s - 0.05 * s
    return f1.to(dev).contiguous(), f2.to(dev).contiguous()


def reference_check(f1, f2, val, idx, k, rows=4096, bound=2e-6):
    """-> (value error relative to max |corr|, rows whose candidate set differs from float64 topk, entries that differ).
    Every value is within `bound` (relative to max |corr|, the 3xTF32 GEMM's bound) of float64, so two entries closer than
    twice that may be ordered either way: every entry in one set and not the other lies that close to the row's K-th value.
    (With K a large share of N2 the K-th value sits where the values are dense, so such near-ties are common.)"""
    c = f1.shape[1]
    f2d = f2.double()
    big = max(float((f1[r0:r0 + rows].double() @ f2d.t()).abs().max()) for r0 in range(0, f1.shape[0], rows)) / math.sqrt(c)
    err = 0.0
    diff_rows = diff_entries = 0
    for r0 in range(0, f1.shape[0], rows):
        ref = f1[r0:r0 + rows].double() @ f2d.t() / math.sqrt(c)
        top = torch.topk(ref, k, dim=1)
        kth = top.values[:, -1:]
        got = idx[r0:r0 + rows].long()
        err = max(err, float((val[r0:r0 + rows].double() - torch.gather(ref, 1, got)).abs().max()))
        mine = torch.zeros_like(ref, dtype=torch.bool).scatter_(1, got, True)
        theirs = torch.zeros_like(mine).scatter_(1, top.indices, True)
        xor = mine ^ theirs
        assert int(mine.sum()) == got.numel()                      # K distinct columns per row
        near = (ref - kth).abs() <= 2 * bound * big
        assert not bool((xor & ~near).any()), 'a candidate differs from the reference away from the K-th value'
        diff_rows += int(xor.any(1).sum())
        diff_entries += int(xor.sum()) // 2
        del ref, mine, theirs, xor, near
    return err / big, diff_rows, diff_entries


def args(k, levels=3, scale=0.25):
    return types.SimpleNamespace(corr_levels=levels, base_scales=scale, truncate_k=k)


# ----------------------------------------------------------------------------------------------------------------------
# 1. the truncated state
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n, m', [(8192, 12000), (12000, 8192), (300, 1000)])
@pytest.mark.parametrize('k', [64, 512])
def test_corr_build_against_float64(dev, n, m, k):
    from pvraft_b200 import ops
    b, c = 2, 128
    f1, f2 = feature_maps(b, n, m, c, n + m + k, dev)
    val, idx = ops.corr_build(f1, f2, k)
    assert val.shape == (b, n, k) and idx.shape == (b, n, k)
    assert bool((idx >= 0).all()) and bool((idx < m).all()) and bool((idx[..., 1:] > idx[..., :-1]).all())
    for s in range(b):
        err, rows, entries = reference_check(f1[s], f2[s], val[s], idx[s], k)
        print(f'N1={n} N2={m} K={k} sample {s}: value err {err:.2e}, {rows} rows / {entries} candidates at near-ties')
        assert err < 2e-6, err


@pytest.mark.parametrize('n, m, k, window', [(8192, 12000, 512, 3072), (12000, 8192, 64, 1024), (300, 1000, 64, 256),
                                             (1000, 300, 32, 128)])
def test_windowed_build_is_bit_identical_for_unequal_sizes(dev, n, m, k, window):
    from pvraft_b200 import ops
    b, c = 2, 128
    f1, f2 = feature_maps(b, n, m, c, 7 * n + m, dev)
    plan = ops.corr_plan(b, n, m, c, k, window=window, cap=max(1, n // 300) << 20)
    assert not plan.dense and len(plan.windows) >= 3
    val, idx = ops.corr_build(f1, f2, k, plan=plan)
    want_val, want_idx = ops.corr_topk(ops.corr_dense(f1, f2), k)
    assert same_bits(val, want_val) and torch.equal(idx, want_idx)
    print(f'N1={n} N2={m} K={k}: {len(plan.windows)} windows, {len(plan.row_blocks)} row blocks: bit-identical')


def test_windowed_build_beyond_49152_columns(dev):
    from pvraft_b200 import ops
    n, m, c, k = 20000, 60000, 128, 512
    f1, f2 = feature_maps(1, n, m, c, 3, dev)
    plan = ops.corr_plan(1, n, m, c, k)
    assert not plan.dense and len(plan.windows) == 2
    val, idx = ops.corr_build(f1, f2, k)
    assert int(idx.max()) >= 49152
    err, rows, entries = reference_check(f1[0], f2[0], val[0], idx[0], k)
    print(f'N1={n} N2={m}: value err {err:.2e}; {rows} rows / {entries} candidates differ, all at the K-th value')
    assert err < 2e-6, err
    # and the first cloud beyond 49152 points against a second one below it: the dense plan (no windows)
    f1b, f2b = feature_maps(1, 60000, 4096, c, 4, dev)
    assert ops.corr_plan(1, 60000, 4096, c, k).dense
    val, idx = ops.corr_build(f1b, f2b, k)
    err, _, _ = reference_check(f1b[0], f2b[0], val[0], idx[0], k)
    assert err < 2e-6, err


# ----------------------------------------------------------------------------------------------------------------------
# 2. the lookup
# ----------------------------------------------------------------------------------------------------------------------
def unequal_state(b, n, m, k, seed, box, dev):
    """N query rows whose K distinct candidate ids (start + j * step mod M, step coprime to M) are rows of an M-point xyz2."""
    g = torch.Generator().manual_seed(seed)
    jitter = min(0.2, box / 4)   # a compact cloud (box 0.4) keeps every candidate within 0.5 of the query on each axis
    xyz2 = box * torch.rand(b, m, 3, generator=g)
    primes = torch.tensor([p for p in (7, 11, 13, 17, 19, 23, 29, 31, 37, 41, 43, 47, 53, 59, 61, 67, 71, 73, 79, 83, 89, 97)
                           if m % p])
    step = primes[torch.randint(0, len(primes), (b, n, 1), generator=g)]
    idx = (torch.randint(0, m, (b, n, 1), generator=g) + torch.arange(k).view(1, 1, k) * step) % m
    pick = torch.randint(0, m, (b, n), generator=g)
    coords = torch.gather(xyz2, 1, pick.unsqueeze(-1).expand(b, n, 3)) + (torch.rand(b, n, 3, generator=g) * 2 - 1) * jitter
    corr = torch.sort(torch.randn(b, n, k, generator=g) * 5 + 20, dim=2, descending=True).values
    return corr.to(dev), idx.to(dev), coords.to(dev).contiguous(), xyz2.to(dev).contiguous()


LOOKUP_CASES = [(8192, 4096, 32, 3.0), (8192, 4096, 512, 3.0), (4096, 20000, 32, 3.0), (4096, 20000, 512, 10.0),
                (100, 4096, 512, 0.4), (100, 20000, 128, 0.4)]   # the last two: N1 < K, compact cells (the count clamp)


@pytest.mark.parametrize('n, m, k, box', LOOKUP_CASES)
@pytest.mark.parametrize('state_dtype', [torch.float32, torch.bfloat16])
def test_lookup_with_unequal_sizes(dev, n, m, k, box, state_dtype):
    from pvraft_b200 import CorrBlock, ops
    if state_dtype == torch.bfloat16 and k < 128:
        pytest.skip('the bf16 state kernels are built for truncate_k >= 128')
    b, levels, scale = 2, 3, 0.25
    assert ops.lookup_table_in_smem(m, k) == (m == 4096)   # both sides of the shared-memory table limit
    corr, idx, coords, xyz2 = unequal_state(b, n, m, k, n + m + k, box, dev)
    cb = CorrBlock(num_levels=levels, base_scale=scale, truncate_k=k).to(dev)
    cb.state_dtype = state_dtype
    cb.set_state(corr, idx, xyz2)
    out = cb.lookup(coords, want_slots=True, want_cube=True)
    # the oracle on the CPU: its scatter_add then adds in ascending slot order, as the kernel does
    ids = cb.candidate_ids().cpu()
    xyz2, coords = xyz2.cpu(), coords.cpu()
    st = O.CorrState(cb.corr_val.float().cpu(), ids, torch.gather(xyz2, 1, ids.reshape(b, -1, 1).expand(b, n * k, 3)).reshape(b, n, k, 3))
    out = {key: v.cpu() for key, v in out.items() if v is not None}
    clamped = 0
    for lvl in range(levels):
        cube, valid = O.voxel_cube_index(st, coords, scale * 2 ** lvl)
        got = out['cube'][..., lvl]
        assert torch.equal(got >= 0, valid), f'level {lvl}: validity differs'
        assert torch.equal(torch.where(got >= 0, got, torch.zeros_like(got)).long(), cube), f'level {lvl}: cell differs'
        clamped += int((torch.zeros(b, n, 27).scatter_add_(2, cube, valid.float()) > n).sum())
    if n < k:
        assert clamped > 0, 'the case was meant to reach clamp(count, 1, N1)'
    want = O.voxel_means(st, coords, levels, scale).transpose(1, 2)
    got = out['vox'][..., :levels * 27]
    assert rel_err(got, want) < 1e-6
    assert (got != want).float().mean() < 1e-3
    dist = O.knn_sqdist(st, coords)
    want_slots = O.knn_select(st, coords).sort(-1).values
    got_slots = out['knn_slot'].long().sort(-1).values
    bad = (want_slots != got_slots).any(-1)
    if bad.any():   # only exact-distance ties at the 32nd neighbour may differ
        d = dist[bad]
        kth = torch.gather(d, 1, want_slots[bad]).max(-1, keepdim=True).values
        assert torch.equal(torch.gather(d, 1, got_slots[bad]).max(-1, keepdim=True).values, kth)
        assert torch.equal((d < kth).sum(-1), (torch.gather(d, 1, got_slots[bad]) < kth).sum(-1))


@pytest.mark.parametrize('n, m, k, box', [(256, 1000, 64, 3.0), (1000, 300, 128, 10.0), (100, 300, 128, 0.4)])
def test_lookup_backward_against_float64(dev, n, m, k, box):
    from pvraft_b200 import CorrBlock, ops, train as T
    b, levels, scale = 2, 3, 0.25
    corr, idx, coords, xyz2 = unequal_state(b, n, m, k, 5 * n + m, box, dev)
    cb = CorrBlock(num_levels=levels, base_scale=scale, truncate_k=k).to(dev)
    cb.set_state(corr, idx, xyz2)
    ids = cb.candidate_ids()
    cand = torch.gather(xyz2, 1, ids.reshape(b, -1, 1).expand(b, n * k, 3)).reshape(b, n, k, 3)
    stored = O.CorrState(leaf(cb.corr_val.double().cpu()), ids.cpu(), cand.double().cpu())
    g = torch.Generator().manual_seed(1)
    g_vox, g_sel = torch.randn(b, n, levels * 27, generator=g), torch.randn(b, n * 32, 4, generator=g)
    cv = leaf(cb.corr_val)
    vox, sel = T.CorrLookupFn.apply(cv, cb.corr_idx, cb._xyz2p, coords, levels, scale)
    (vox * g_vox.to(dev)).sum().add((sel * g_sel.to(dev)).sum()).backward()
    slots = ops.corr_lookup(cb.corr_val, cb.corr_idx, cb._xyz2p, coords, levels, scale, want_slots=True)['knn_slot'].long().cpu()
    want_vox = U.voxel_means(stored, coords.double().cpu(), levels, scale).transpose(1, 2)
    want_sel = O.knn_gather(stored, coords.double().cpu(), slots).permute(0, 2, 3, 1).reshape(b, n * 32, 4)
    ((want_vox * g_vox.double()).sum() + (want_sel * g_sel.double()).sum()).backward()
    assert rel_err(vox.detach().cpu(), want_vox.detach()) < 1e-6
    assert rel_err(cv.grad.cpu(), stored.truncated_corr.grad) < 1e-5


# ----------------------------------------------------------------------------------------------------------------------
# 3. the bf16 state's limit is on N2
# ----------------------------------------------------------------------------------------------------------------------
def test_bf16_state_limit_is_on_the_second_cloud(dev):
    from pvraft_b200 import RSF
    torch.manual_seed(0)
    m = RSF(args(128)).to(dev).eval().set_precision('bf16')
    m.use_cuda_graph = False
    big, small = O.synthetic_clouds(1, 70000, seed=3)[0], O.synthetic_clouds(1, 8192, seed=4)[0]
    with torch.no_grad():
        flows = m([big.to(dev), small.to(dev)], 2)
        assert flows[-1].shape == (1, 70000, 3) and torch.isfinite(flows[-1]).all()
        assert m.corr_block.corr_idx.dtype == torch.int16
        with pytest.raises(ValueError, match='65536'):
            m([small.to(dev), big.to(dev)], 2)


# ----------------------------------------------------------------------------------------------------------------------
# 4. the model against the reference's modules
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def golden():
    arr, W1 = load_golden('unequal_rsf.npz')
    return arr, U.golden_weights(arr, W1)


def golden_model(golden, c, dev, refine=True):
    from pvraft_b200 import RSF, RSF_refine
    arr, W = golden
    b, n1, n2, k, levels, iters, s = [int(v) for v in arr[f'{c}/meta']]
    m = (RSF_refine if refine else RSF)(args(k, levels, float(arr['base_scale'])))
    m.load_state_dict(W if refine else {kk: v for kk, v in W.items() if not kk.startswith('refine_block.')}, strict=True)
    return m.to(dev).eval(), (lambda key: arr[f'{c}/{key}']), iters, s


def test_lookup_teacher_forced_vs_reference(dev, golden):
    """Case c (N1 = 100 < K = 128 <= N2 = 300, the CUDA-core path, the count clamp reached): the correlation and voxel
    features from the reference's own state, at the reference's query coordinates of both iterations."""
    m, g, iters, s = golden_model(golden, 'c', dev)
    st = U.golden_state(g)
    m.corr_block.set_state(st.truncated_corr.to(dev), st.indices.to(dev), g('pc2').to(dev))
    with torch.no_grad():
        for it, coords in enumerate((g('pc1'), g('it1/coords'))):
            coords = coords.to(dev)
            assert rel_err(m.corr_block(coords)[..., :s].cpu(), g(f'it{it}/corr')) < 1e-5
            assert rel_err(m.corr_block.get_voxel_feature(coords)[..., :s].cpu(), g(f'it{it}/voxel_feature')) < 1e-5


def close(got, want):
    """The free-running tolerance of test_gpu_parity.py: mean |difference| below 2e-3 of mean |reference|."""
    return float((got.cpu() - want).abs().mean()) < 2e-3 * float(want.abs().mean())


@pytest.mark.parametrize('c', ['a', 'b', 'c'])
def test_free_running_vs_reference(dev, golden, c):
    """Every stored it*/ entry and the flows.  The model's forward gives the flows; the per-iteration features come from
    the same modules called as RSF.forward's statements (model/RAFTSceneFlow.py:22-50) through the reference's API."""
    p_refine, g, iters, s = golden_model(golden, c, dev, refine=True)
    rsf, _, _, _ = golden_model(golden, c, dev, refine=False)
    pc1, pc2 = g('pc1').to(dev), g('pc2').to(dev)
    with torch.no_grad():
        flows = rsf([pc1, pc2], iters)
        refined = p_refine([pc1, pc2], iters)
        fmap1, _ = rsf.feature_extractor(pc1)
        fmap2, _ = rsf.feature_extractor(pc2)
        rsf.corr_block.init_module(fmap1, fmap2, pc2)
        fct1, gctx = rsf.context_extractor(pc1)
        net, inp = torch.tanh(fct1[:, :64]).contiguous(), torch.relu(fct1[:, 64:]).contiguous()
        coords2 = pc1
        for it in range(iters):
            corr = rsf.corr_block(coords2)
            assert close(corr[..., :s], g(f'it{it}/corr'))
            assert close(rsf.corr_block.get_voxel_feature(coords2)[..., :s], g(f'it{it}/voxel_feature'))
            net, delta = rsf.update_block(net, inp, corr, coords2 - pc1, gctx)
            assert close(net[..., :s], g(f'it{it}/net'))
            coords2 = coords2 + delta
            assert close(coords2 - pc1, g(f'it{it}/flow'))
    for it in range(iters):
        assert flows[it].shape == g(f'it{it}/flow').shape and close(flows[it], g(f'it{it}/flow'))
    if c == 'a':
        assert refined.shape == g('refined').shape and close(refined, g('refined'))


# ----------------------------------------------------------------------------------------------------------------------
# 5. CUDA-graph replay
# ----------------------------------------------------------------------------------------------------------------------
def pair(n1, n2, seed, dev, b=1):
    g = torch.Generator().manual_seed(seed)
    pc1 = 10.0 * torch.rand(b, n1, 3, generator=g)
    pc2 = 10.0 * torch.rand(b, n2, 3, generator=g)
    return pc1.to(dev), pc2.to(dev)


@pytest.mark.parametrize('n1, n2', [(8192, 12288), (12288, 8192), (1000, 3000)])
def test_graph_replay_matches_eager(dev, n1, n2):
    from pvraft_b200 import RSF
    torch.manual_seed(0)
    m = RSF(args(512 if n2 >= 512 else 128)).to(dev).eval()
    p = list(pair(n1, n2, n1 + n2, dev))
    with torch.no_grad():
        m.use_cuda_graph = False
        eager = m(p, 4)
        m.use_cuda_graph = True
        graphed = m(p, 4)
        again = m(p, 4)
    assert len(m._graphs) == 1
    for e, g1, g2 in zip(eager, graphed, again):
        assert e.shape == (1, n1, 3) and torch.isfinite(e).all()
        assert rel_err(g1.cpu(), e.cpu()) < 1e-6 and rel_err(g2.cpu(), e.cpu()) < 1e-6


def test_pairs_sharing_n1_keep_their_own_graphs(dev):
    from pvraft_b200 import RSF
    torch.manual_seed(0)
    m = RSF(args(512)).to(dev).eval()
    a, b = list(pair(8192, 12288, 1, dev)), list(pair(8192, 16384, 2, dev))
    with torch.no_grad():
        m.use_cuda_graph = False
        want_a, want_b = m(a, 3), m(b, 3)
        m.use_cuda_graph = True
        for _ in range(2):
            got_a, got_b = m(a, 3), m(b, 3)
            for g, w in zip(got_a, want_a):
                assert rel_err(g.cpu(), w.cpu()) < 1e-6
            for g, w in zip(got_b, want_b):
                assert rel_err(g.cpu(), w.cpu()) < 1e-6
    assert len(m._graphs) == 2
    assert rel_err(want_a[-1].cpu(), want_b[-1].cpu()) > 1e-3   # the two pairs really differ


# ----------------------------------------------------------------------------------------------------------------------
# 6. training
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n1, n2', [(1024, 1536), (1536, 1024)])
def test_rsf_gradients_match_oracle(dev, n1, n2):
    from conftest import default_weights
    from pvraft_b200 import RSF
    b, k, iters = 2, 128, 3
    a = args(k)
    W = default_weights(args=a, seed=2)
    g = torch.Generator().manual_seed(n1 + n2)
    pc1, pc2 = 4.0 * torch.rand(b, n1, 3, generator=g), 4.0 * torch.rand(b, n2, 3, generator=g)
    gt = 0.1 * torch.randn(b, n1, 3, generator=g)
    Wr = {kk: leaf(v) for kk, v in W.items()}
    flows_ref = U.rsf_forward(Wr, pc1, pc2, iters, 3, 0.25, k)
    sequence_loss(flows_ref, gt).backward()
    want = {kk: v.grad for kk, v in Wr.items()}
    assert all(v is not None and float(v.abs().max()) > 0 for v in want.values())
    m = RSF(a)
    m.load_state_dict(W)
    m = m.to(dev).train()
    with oracle_adjacency():
        flows = m([pc1.to(dev), pc2.to(dev)], num_iters=iters)
    assert len(flows) == iters and flows[-1].shape == (b, n1, 3) and flows[-1].requires_grad
    for f, fr in zip(flows, flows_ref):
        assert float((f.detach().cpu() - fr.detach()).abs().mean()) < 1e-4 * float(fr.detach().abs().mean())
    loss = sequence_loss(flows, gt.to(dev))
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters()}
    assert len(got) == 95 and all(v is not None for v in got.values())
    compare_grads(got, want, 2e-2, 5e-2)


@pytest.mark.parametrize('n, m, det', [(1000, 3000, False), (3000, 1000, False), (1000, 3000, True)])
def test_corr_init_bwd_against_the_sparse_formula(dev, n, m, det):
    from pvraft_b200 import CorrBlock, train as T
    b, c, k = 2, 128, 256
    f1, f2 = feature_maps(b, n, m, c, n + m, dev)
    a, d = leaf(f1), leaf(f2)
    torch.use_deterministic_algorithms(det)
    try:
        val, idx = T.CorrInitFn.apply(a, d, k, CorrBlock(truncate_k=k).to(dev))
        gv = torch.randn(b, n, k, generator=torch.Generator().manual_seed(6)).to(dev)
        (val * gv).sum().backward()
    finally:
        torch.use_deterministic_algorithms(False)
    assert d.grad.shape == (b, m, c)
    s = math.sqrt(c)
    a64, d64, ids = f1.double(), f2.double(), idx.long()
    picked = torch.gather(d64.unsqueeze(1).expand(b, n, m, c), 2, ids.unsqueeze(-1).expand(b, n, k, c))   # [B,N,K,C]
    assert rel_err(val.detach(), torch.einsum('bnc,bnkc->bnk', a64, picked) / s) < 2e-6
    want_da = torch.einsum('bnk,bnkc->bnc', gv.double(), picked) / s
    want_dd = torch.zeros_like(d64)
    for s_ in range(b):
        want_dd[s_].index_add_(0, ids[s_].reshape(-1), (gv[s_].double().unsqueeze(-1) * a64[s_].unsqueeze(1)).reshape(-1, c) / s)
    assert rel_err(a.grad, want_da) < 2e-5 and rel_err(d.grad, want_dd) < 2e-5


def test_deterministic_training_steps_repeat_bitwise(dev):
    from pvraft_b200 import RSF
    pc1, pc2 = pair(1024, 1536, 9, dev, b=2)
    gt = 0.1 * torch.randn(2, 1024, 3, generator=torch.Generator().manual_seed(1)).to(dev)
    results = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            torch.manual_seed(0)
            m = RSF(args(128)).to(dev).train()
            opt = torch.optim.Adam(m.parameters(), lr=1e-3)
            for _ in range(2):
                opt.zero_grad()
                sequence_loss(m([pc1, pc2], num_iters=3), gt).backward()
                opt.step()
            results.append([p.detach().clone() for p in m.parameters()])
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(x, y) for x, y in zip(*results))
