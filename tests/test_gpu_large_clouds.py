"""Clouds beyond 49152 points: the truncated correlation built in column windows (ops.corr_build, ops.CorrPlan).

  * bit-identity with the dense build (corr_matmul + corr_topk [+ corr_reorder]) where both run, on plans forced to small
    windows and row blocks: several windows, several row blocks, a ragged last window, both top-K kernels in both steps
  * value ties across windows: the lowest columns win, as in the dense kernel
  * N = 65536 .. 131072 against a float64 reference on the device (matmul in row blocks, / sqrt(C), torch.topk): candidate
    sets equal up to entries within 1e-6 relative of the K-th value, values within the GEMM bound (2e-6 at C = 128), and a
    peak of allocated memory that leaves no room for an N x N matrix
  * the model at N = 65536: graph replay against eager, the loop on a reference state, the bf16 state limit, RSF_refine
  * training at N = 65536: CorrInitFn against the sparse formula, and one stage-1 step
"""
import math
import types

import pytest
import torch

from conftest import rel_err
from oracle import pvraft_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


def feature_maps(b, n, c, seed, dev):
    """[B,N,C] pairs whose scale and offset differ from sample to sample."""
    g = torch.Generator().manual_seed(seed)
    s = torch.linspace(0.5, 2.0, b).view(b, 1, 1)
    f1 = torch.randn(b, n, c, generator=g) * s + 0.1 * s
    f2 = torch.randn(b, n, c, generator=g) * s - 0.05 * s
    return f1.to(dev).contiguous(), f2.to(dev).contiguous()


def dense_build(f1, f2, k):
    from pvraft_b200 import ops
    return ops.corr_topk(ops.corr_dense(f1, f2), k)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ----------------------------------------------------------------------------------------------------------------------
# bit-identity with the dense build
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n, k, window', [(8192, 512, 3072),      # 3 windows, vectorised top-K in both steps
                                          (20000, 512, 8192),     # ragged N and last window
                                          (20001, 64, 1024),      # 20 windows, last one 545 columns: general kernel per window
                                          (49152, 512, 16384),    # 16384-column windows: general kernel per window
                                          (49152, 512, 2048)])    # 24 x 512 candidates: general kernel with the id map
def test_windowed_build_is_bit_identical_to_the_dense_build(dev, n, k, window):
    from pvraft_b200 import ops
    b, c = 2, 128
    f1, f2 = feature_maps(b, n, c, n + k, dev)
    plan = ops.corr_plan(b, n, n, c, k, window=window, cap=64 << 20)
    assert not plan.dense and len(plan.windows) >= 3 and len(plan.row_blocks) >= 2
    val, idx = ops.corr_build(f1, f2, k, plan=plan)
    want_val, want_idx = dense_build(f1, f2, k)
    assert same_bits(val, want_val) and torch.equal(idx, want_idx)
    got_r, want_r = ops.corr_reorder(val, idx), ops.corr_reorder(want_val, want_idx)
    assert same_bits(got_r[0], want_r[0]) and torch.equal(got_r[1], want_r[1])
    default = ops.corr_build(f1, f2, k)          # the default plan of N <= 49152 is the dense build itself
    assert same_bits(default[0], want_val) and torch.equal(default[1], want_idx)
    print(f'N={n} K={k}: {len(plan.windows)} windows (last {plan.windows[-1][1]} columns), {len(plan.row_blocks)} row blocks: '
          'bit-identical')


def f2key(v):
    """The kernels' order-preserving uint32 key of a float, as int64 (larger float, larger key; -0 < +0)."""
    u = v.contiguous().view(torch.int32).long() & 0xFFFFFFFF
    return torch.where(u >= 0x80000000, 0xFFFFFFFF - u, u | 0x80000000)


def test_ties_across_windows_keep_the_lowest_columns(dev):
    from pvraft_b200 import ops
    n, c, k = 8192, 128, 64
    g = torch.Generator().manual_seed(3)
    f1 = torch.randn(4, n, c, generator=g).abs() * 0.1
    f2 = torch.randn(4, n, c, generator=g).abs() * 0.1
    v = torch.full((c,), 4.0)
    tied = torch.arange(11, n, 37)                # 221 equal maxima spread over all 8 windows
    f2[:, tied] = v
    f1[:, :300] = v                               # rows whose maxima (221 > K of them) tie across windows
    f1[:, 300:310] = 0.0                          # constant rows: every column is +0
    f1, f2 = f1.to(dev), f2.to(dev)
    plan = ops.corr_plan(4, n, n, c, k, window=1024, cap=16 << 20)
    assert len(plan.windows) == 8 and len(plan.row_blocks) >= 2
    val, idx = ops.corr_build(f1, f2, k, plan=plan)
    want_val, want_idx = dense_build(f1, f2, k)
    assert same_bits(val, want_val) and torch.equal(idx, want_idx)
    assert torch.equal(idx[:, :300].long().cpu(), tied[:k].expand(4, 300, k))
    assert torch.equal(idx[:, 300:310].long().cpu(), torch.arange(k).expand(4, 10, k))
    # every row against the selection rule itself: key descending, then column ascending
    corr = ops.corr_dense(f1, f2)
    key = f2key(corr[:, :320])
    cols = torch.arange(n, device=dev)
    order = torch.argsort(key * (2 * n) + (n - 1 - cols), dim=-1, descending=True)[..., :k]
    assert torch.equal(order.sort(-1).values.to(torch.int32), idx[:, :320])


# ----------------------------------------------------------------------------------------------------------------------
# beyond the old limit, against a float64 reference on the device
# ----------------------------------------------------------------------------------------------------------------------
def reference_check(f1, f2, val, idx, k, rows=4096):
    """-> (value error relative to max |corr|, rows whose candidate set differs, entries that differ): every entry in one set
    and not the other lies within 1e-6 relative of the row's K-th value."""
    n, c = f1.shape
    f2d = f2.double()
    err = big = 0.0
    diff_rows = diff_entries = 0
    for r0 in range(0, n, rows):
        ref = f1[r0:r0 + rows].double() @ f2d.t() / math.sqrt(c)
        top = torch.topk(ref, k, dim=1)
        kth = top.values[:, -1:]
        got = idx[r0:r0 + rows].long()
        err = max(err, float((val[r0:r0 + rows].double() - torch.gather(ref, 1, got)).abs().max()))
        big = max(big, float(ref.abs().max()))
        mine = torch.zeros_like(ref, dtype=torch.bool).scatter_(1, got, True)
        theirs = torch.zeros_like(mine).scatter_(1, top.indices, True)
        xor = mine ^ theirs
        assert int(mine.sum()) == got.numel()                      # K distinct columns per row
        near = (ref - kth).abs() <= 1e-6 * kth.abs()
        assert not bool((xor & ~near).any()), 'a candidate differs from the reference away from the K-th value'
        diff_rows += int(xor.any(1).sum())
        diff_entries += int(xor.sum()) // 2
        del ref, mine, theirs, xor, near
    return err / big, diff_rows, diff_entries


@pytest.mark.parametrize('n', [65536, 100000, 131072])
def test_beyond_the_dense_limit_against_float64(dev, n):
    from pvraft_b200 import ops
    c, k = 128, 512
    f1, f2 = feature_maps(1, n, c, n, dev)
    plan = ops.corr_plan(1, n, n, c, k)
    assert not plan.dense and len(plan.windows) >= 2
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)                         # the two feature maps
    val, idx = ops.corr_build(f1, f2, k)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev) - base
    npad = (n + 127) // 128 * 128
    split = 4 * npad * c * 4                                        # tf32 hi/lo of both maps
    state = n * k * 8
    bound = split + state + plan.slab_bytes + (4 << 20)
    print(f'N={n}: {len(plan.windows)} windows, {len(plan.row_blocks)} row blocks, peak {peak / 2**20:.0f} MiB above the '
          f'feature maps (bound {bound / 2**20:.0f} MiB; the N x N matrix alone is {4 * n * n / 2**30:.1f} GiB)')
    assert peak <= bound and peak < 4 * n * n
    assert (idx[0, :, 1:] > idx[0, :, :-1]).all()                    # ascending columns
    err, rows, entries = reference_check(f1[0], f2[0], val[0], idx[0], k)
    print(f'N={n}: value err {err:.2e}; {rows} rows / {entries} candidates differ from float64 topk, all at the K-th value')
    assert err < 2e-6, err


# ----------------------------------------------------------------------------------------------------------------------
# the model at N = 65536
# ----------------------------------------------------------------------------------------------------------------------
N_MODEL = 65536


@pytest.fixture(scope='module')
def clouds():
    return O.synthetic_clouds(1, N_MODEL, seed=11)


def model_args(k=512):
    return types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)


def test_model_graph_replay_matches_eager(dev, clouds):
    from pvraft_b200 import RSF
    torch.manual_seed(0)
    m = RSF(model_args()).to(dev).eval()
    pc1, pc2 = clouds[0].to(dev), clouds[1].to(dev)
    with torch.no_grad():
        m.use_cuda_graph = False
        eager = m([pc1, pc2], 4)
        m.use_cuda_graph = True
        graphed = m([pc1, pc2], 4)
        again = m([pc1, pc2], 4)
    assert len(m._graphs) == 1
    for e, g, a in zip(eager, graphed, again):
        assert torch.isfinite(e).all()
        assert rel_err(g.cpu(), e.cpu()) < 1e-6 and rel_err(a.cpu(), e.cpu()) < 1e-6


def per_sample_err(got, want):
    return float((got.double() - want.double()).abs().max() / want.double().abs().max())


def test_model_loop_on_a_reference_state(dev, clouds):
    """The loop's correlation feature and motion, iteration by iteration at the model's own coordinates, from the state the
    model builds and from a float64 state installed with set_state.  The model's candidate sets are first checked against
    float64 topk (equal up to near-ties at the K-th value); the float64 state then keeps those candidates with float64 values,
    because a single swapped candidate moves every point through the GroupNorm statistics of the sample."""
    from pvraft_b200 import RSF
    k = 512
    torch.manual_seed(0)
    m = RSF(model_args(k)).to(dev).eval()
    m.use_cuda_graph = False
    pc1, pc2 = clouds[0].to(dev), clouds[1].to(dev)
    with torch.no_grad():
        flows = m([pc1, pc2], 4)
        fmap, _ = m.feature_extractor(torch.cat([pc1, pc2], 0), point_major=True)
        f1, f2 = fmap[0], fmap[1]
        cb = m.corr_block
        cb.init_module_pm(fmap[:1], fmap[1:], pc2)
        own = (cb.corr_val.clone(), cb.corr_idx.clone())
        err, rows, _ = reference_check(f1, f2, own[0][0], own[1][0], k)
        assert err < 2e-6 and rows <= N_MODEL // 100, (err, rows)
        ids = own[1][0].long()
        ref_val = torch.empty(N_MODEL, k, dtype=torch.float32, device=dev)
        for r0 in range(0, N_MODEL, 4096):
            ref = f1[r0:r0 + 4096].double() @ f2.double().t() / math.sqrt(f1.shape[-1])
            ref_val[r0:r0 + 4096] = torch.gather(ref, 1, ids[r0:r0 + 4096]).float()
        me = m.update_block.motion_encoder
        worst = dict(corr=0.0, motion=0.0)
        for it in range(4):
            coords = (pc1 + flows[it]).contiguous()
            flow = flows[it].contiguous()
            cb.corr_val, cb.corr_idx = own
            corr_a, motion_a = cb.feature_motion_tc(coords, flow, me, need_corr=True)
            cb.set_state(ref_val[None], ids[None], pc2)
            corr_b, motion_b = cb.feature_motion_tc(coords, flow, me, need_corr=True)
            worst['corr'] = max(worst['corr'], per_sample_err(corr_a, corr_b))
            worst['motion'] = max(worst['motion'], per_sample_err(motion_a, motion_b))
    print(f'N={N_MODEL}: state err {err:.2e}, {rows} rows with a near-tie at the K-th value; loop worst err', worst)
    assert worst['corr'] < 1e-5 and worst['motion'] < 2e-5, worst


def test_bf16_state_up_to_65536_points(dev, clouds):
    from pvraft_b200 import RSF
    torch.manual_seed(0)
    m = RSF(model_args(128)).to(dev).eval().set_precision('bf16')
    m.use_cuda_graph = False
    with torch.no_grad():
        flows = m([clouds[0].to(dev), clouds[1].to(dev)], 2)
        assert m.corr_block.corr_idx.dtype == torch.int16 and torch.isfinite(flows[-1]).all()
        ids = m.corr_block.candidate_ids()
        assert int(ids.max()) >= 65000 and int(ids.min()) >= 0
        one_more = [torch.cat([p, p[:, :1] + 0.01], 1).to(dev) for p in clouds]
        with pytest.raises(ValueError, match='65536'):
            m(one_more, 2)


def test_refine_model_runs_at_65536_points(dev, clouds):
    from pvraft_b200 import RSF_refine
    torch.manual_seed(0)
    m = RSF_refine(model_args()).to(dev).eval()
    with torch.no_grad():
        out = m([clouds[0].to(dev), clouds[1].to(dev)], 4)
    assert out.shape == (1, N_MODEL, 3) and torch.isfinite(out).all()


# ----------------------------------------------------------------------------------------------------------------------
# training at N = 65536
# ----------------------------------------------------------------------------------------------------------------------
def test_corr_init_fn_against_the_sparse_formula(dev):
    from pvraft_b200 import CorrBlock
    from pvraft_b200 import train as T
    n, c, k = N_MODEL, 128, 512
    a, d = feature_maps(1, n, c, 5, dev)
    a.requires_grad_(True)
    d.requires_grad_(True)
    cb = CorrBlock(truncate_k=k).to(dev)
    val, idx = T.CorrInitFn.apply(a, d, k, cb)
    g = torch.Generator().manual_seed(6)
    gv = torch.randn(1, n, k, generator=g).to(dev)
    (val * gv).sum().backward()
    s = math.sqrt(c)
    a64, d64 = a.detach()[0].double(), d.detach()[0].double()
    want_da = torch.zeros_like(a64)
    want_dd = torch.zeros_like(d64)
    e_val = 0.0
    for r0 in range(0, n, 2048):
        ids = idx[0, r0:r0 + 2048].long()
        picked = d64[ids]                                             # [rows, K, C]
        corr = torch.einsum('rc,rkc->rk', a64[r0:r0 + 2048], picked) / s
        e_val = max(e_val, float((val.detach()[0, r0:r0 + 2048].double() - corr).abs().max()))
        gr = gv[0, r0:r0 + 2048].double()
        want_da[r0:r0 + 2048] = torch.einsum('rk,rkc->rc', gr, picked) / s
        want_dd.index_add_(0, ids.reshape(-1), (gr.unsqueeze(-1) * a64[r0:r0 + 2048].unsqueeze(1)).reshape(-1, c) / s)
        del picked
    e_da, e_dd = rel_err(a.grad[0], want_da), rel_err(d.grad[0], want_dd)
    e_val /= float(val.detach().abs().max())
    print(f'CorrInitFn N={n}: value err {e_val:.2e}, d fmap1 err {e_da:.2e}, d fmap2 err {e_dd:.2e}')
    assert e_val < 2e-6
    assert e_da < 2e-5 and e_dd < 2e-5


def test_stage1_training_step_at_65536_points(dev, clouds):
    from pvraft_b200 import RSF
    torch.manual_seed(0)
    m = RSF(model_args()).to(dev).train()
    pc1, pc2 = clouds[0].to(dev), clouds[1].to(dev)
    flows = m([pc1, pc2], num_iters=2)
    gt = pc2 - pc1
    loss = sum(0.8 ** (1 - i) * (flows[i] - gt).abs().sum(-1).mean() for i in range(2))
    loss.backward()
    grads = {name: p.grad for name, p in m.named_parameters()}
    assert len(grads) == 95 and all(v is not None for v in grads.values())
    bad = [name for name, v in grads.items() if not torch.isfinite(v).all()]
    assert not bad, bad
    print(f'stage-1 step N={N_MODEL}: loss {float(loss.detach()):.4f}, all 95 gradients finite')
