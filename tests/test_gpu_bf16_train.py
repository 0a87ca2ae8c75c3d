"""The 'bf16-mixed' training mode (RSF.set_precision): the RAFT loop's per-point layers on bf16 wgmma in the forward, in dx
and in dW, over the fp32 correlation state and fp32 master weights.

  1. pvraft_tc_wgrad_bf16 against float64 products of the bf16-rounded operands, for every (cin, cout) of the loop and ragged
     row counts; db against the float64 sum of the unrounded dy; += into a non-zero dW
  2. its DET form: equal to the default within the same bound, bitwise reproducible
  3. LinearFn in the mode: forward, dx and dW for a layer of each path (bf16 dW; fp32 fallback at cout 61 and 3)
  4. a whole stage-1 step: the 95 parameter gradients and the input gradients against the 'fp32' mode
  5. bitwise: eager == captured step, two deterministic steps, switching back to 'fp32', N % 128 != 0 == 'fp32'
  6. inference in the mode: the pre-loop state is bitwise 'fp32', accuracy against the oracle, fused == unfused chain,
     RSF_refine training
  7. a 20-step Adam loop ends near the 'fp32' loop's loss
Bounds were measured on an H100 first; each assert states the measured value next to its bound.
"""
import types

import pytest
import torch

from conftest import default_weights
from oracle import pvraft_oracle as O
from train_helpers import sequence_loss

pytestmark = pytest.mark.gpu

LEVELS, SCALE = 3, 0.25
# (cin, cout) of the loop layers whose weight gradient runs on the new kernel: out_conv[3] and the head's out_conv[0]
# (128 -> 64); knn_out, conv_corr, conv1, the SetConv's fc1 point term, fc2, fc3 (64 -> 64); the GRU's [z|r] and q
LOOP_SHAPES = [(128, 64), (64, 64), (192, 128), (192, 64)]
ROWS = [2 * 8192, 5 * 4096, 1000, 77]


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture
def deterministic():
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(old)


def bf(x):
    """bf16 rounding (nearest even), widened to float64."""
    return x.to(torch.bfloat16).double()


def make_model(dev, k=128, refine=False, seed=0, mode='bf16-mixed'):
    from pvraft_b200 import RSF, RSF_refine
    args = types.SimpleNamespace(corr_levels=LEVELS, base_scales=SCALE, truncate_k=k)
    m = (RSF_refine if refine else RSF)(args)
    m.load_state_dict(default_weights(refine=refine, seed=seed, args=args), strict=True)
    return m.to(dev).set_precision(mode)


def clouds(b, n, seed, dev, scale=0.4):
    pc1, pc2 = O.synthetic_clouds(b, n, seed=seed)
    return (pc1 * scale).to(dev), (pc2 * scale).to(dev)


def step(m, pc1, pc2, iters, inputs=False):
    """One stage-1 forward + backward -> (flows, {name: grad}, input grads or None)."""
    m.train()
    m.zero_grad(set_to_none=True)
    x1, x2 = (pc1.clone().requires_grad_(True), pc2.clone().requires_grad_(True)) if inputs else (pc1, pc2)
    flows = m([x1, x2], num_iters=iters)
    sequence_loss(flows, pc2 - pc1).backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    return [f.detach() for f in flows], grads, ((x1.grad, x2.grad) if inputs else None)


def check_wgrad(dw, db, x, dy, dw0=None, db0=None):
    """dw [cout,cin] against dw0 + bf16(dy)^T bf16(x) in float64: |err| <= 1e-5 sum|dy||x| per entry; db against db0 + the
    float64 column sums of the unrounded dy: |err| <= 1e-6 sum|dy|.  -> the worst ratios."""
    x2, dy2 = x.reshape(-1, x.shape[-1]), dy.reshape(-1, dy.shape[-1])
    want = bf(dy2).t() @ bf(x2) + (0 if dw0 is None else dw0.double())
    s = dy2.double().abs().t() @ x2.double().abs()
    err = (dw.double() - want).abs()
    assert torch.isfinite(dw).all()
    w_ratio = float((err / s.clamp_min(1e-30)).max())
    assert not (err > 1e-5 * s).any(), f'{int((err > 1e-5 * s).sum())} entries off, worst {w_ratio:.3e}'   # measured <= 1.3e-7
    b_ratio = 0.0
    if db is not None:
        want_b = dy2.double().sum(0) + (0 if db0 is None else db0.double())
        sb = dy2.double().abs().sum(0)
        eb = (db.double() - want_b).abs()
        b_ratio = float((eb / sb).max())
        assert not (eb > 1e-6 * sb).any(), f'db: worst |err| / sum|dy| = {b_ratio:.3e}'   # measured <= 5e-8
    return w_ratio, b_ratio


def operands(rows, cin, cout, seed, dev):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, rows, cin, generator=g).to(dev)
    dy = (torch.randn(1, rows, cout, generator=g) * 1e-3).to(dev)
    return x, dy


# ---- 1. the kernel against float64 ----------------------------------------------------------------------------------
@pytest.mark.parametrize('cin,cout', LOOP_SHAPES)
@pytest.mark.parametrize('rows', ROWS)
def test_wgrad_kernel_against_float64(dev, cin, cout, rows):
    from pvraft_b200 import ops
    x, dy = operands(rows, cin, cout, cin * 7 + cout + rows, dev)
    dw = torch.zeros(cout, cin, device=dev)
    db = torch.zeros(cout, device=dev)
    ops.tc_wgrad_bf16(x, dy, dw, db)
    torch.cuda.synchronize()
    w_ratio, b_ratio = check_wgrad(dw, db, x, dy)
    # += into non-zero gradients, and without a bias
    dw0, db0 = torch.randn(cout, cin, device=dev) * 1e-2, torch.randn(cout, device=dev) * 1e-2
    dw2, db2 = dw0.clone(), db0.clone()
    ops.tc_wgrad_bf16(x, dy, dw2, db2)
    dw3 = dw0.clone()
    ops.tc_wgrad_bf16(x, dy, dw3)
    torch.cuda.synchronize()
    check_wgrad(dw2, db2, x, dy, dw0, db0)
    check_wgrad(dw3, None, x, dy, dw0)
    print(f'tc_wgrad_bf16 cin={cin} cout={cout} rows={rows}: worst |err| / sum|dy||x| = {w_ratio:.2e}, db {b_ratio:.2e}')


def test_wgrad_kernel_every_width_and_a_strided_destination(dev):
    """cin 32..192 and cout 32..128 in steps of 32 (the kernel's whole domain), with dw_ld > cin."""
    from pvraft_b200 import ops
    for cin in range(32, 193, 32):
        for cout in range(32, 129, 32):
            x, dy = operands(3000, cin, cout, cin + 1000 * cout, dev)
            full = torch.zeros(cout, cin + 32, device=dev)
            db = torch.zeros(cout, device=dev)
            ops.check(ops.lib().pvraft_tc_wgrad_bf16(x.data_ptr(), dy.data_ptr(), 3000, cin, cout, full.data_ptr(), cin + 32,
                                                     db.data_ptr(), None, ops._stream()), 'tc_wgrad_bf16')
            torch.cuda.synchronize()
            check_wgrad(full[:, :cin], db, x, dy)
            assert not full[:, cin:].any()


# ---- 2. DET ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('cin,cout', LOOP_SHAPES)
def test_wgrad_kernel_deterministic(dev, cin, cout, deterministic):
    from pvraft_b200 import ops
    x, dy = operands(2 * 8192, cin, cout, cin + cout, dev)
    runs = []
    for _ in range(2):
        dw, db = torch.zeros(cout, cin, device=dev), torch.zeros(cout, device=dev)
        ops.tc_wgrad_bf16(x, dy, dw, db)
        runs.append((dw, db))
    torch.use_deterministic_algorithms(False)
    dwd, dbd = torch.zeros(cout, cin, device=dev), torch.zeros(cout, device=dev)
    ops.tc_wgrad_bf16(x, dy, dwd, dbd)
    torch.cuda.synchronize()
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    check_wgrad(runs[0][0], runs[0][1], x, dy)
    s = dy.reshape(-1, cout).abs().t() @ x.reshape(-1, cin).abs()
    assert ((runs[0][0] - dwd).abs() <= 1e-5 * s).all()
    assert ((runs[0][1] - dbd).abs() <= 1e-6 * dy.reshape(-1, cout).abs().sum(0)).all()


# ---- 3. LinearFn in the mode ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('cin,cout,stats', [(192, 128, False), (64, 64, True), (128, 61, False), (64, 3, False)])
def test_linear_fn_in_the_mode(dev, cin, cout, stats):
    """Inside the loop's scope: y = bf16(x) bf16(W)^T + b; dx = bf16(dy) bf16(W) when cout % 32 == 0, else fp32; dW on the
    new kernel when cout % 32 == 0, else fp32 -- the float64 reference follows the same plan."""
    from pvraft_b200 import ops, train as T
    fwd, dx_tc, dw_tc = T.bf16_layer_plan(1024, cin, cout, stats)
    assert fwd and dx_tc == (cout % 32 == 0) and dw_tc == (cout % 32 == 0)
    g = torch.Generator().manual_seed(cin + cout)
    x = torch.randn(2, 1024, cin, generator=g).to(dev).requires_grad_(True)
    w = (torch.randn(cout, cin, 1, generator=g) / cin ** 0.5).to(dev).requires_grad_(True)
    b = torch.randn(cout, generator=g).to(dev).requires_grad_(True)
    gy = (torch.randn(2, 1024, cout, generator=g) * 1e-2).to(dev)
    with ops.bf16_compute():
        out = T.linear(x, w, b, stats)
    y = out[0] if stats else out
    y.backward(gy)
    torch.cuda.synchronize()
    x2, w2, gy2 = x.detach().reshape(-1, cin), w.detach().reshape(cout, cin), gy.reshape(-1, cout)
    want_y = bf(x2) @ bf(w2).t() + b.detach().double()
    ey = (y.detach().reshape(-1, cout).double() - want_y).abs()
    assert (ey <= 1e-5 * (x2.double().abs() @ w2.double().abs().t()) + 1e-6).all(), float(ey.max())
    rnd = bf if dx_tc else (lambda t: t.double())
    want_dx = rnd(gy2) @ rnd(w2)
    edx = (x.grad.reshape(-1, cin).double() - want_dx).abs()
    assert (edx <= 1e-5 * (gy2.double().abs() @ w2.double().abs()) + 1e-12).all(), float(edx.max())
    rnd = bf if dw_tc else (lambda t: t.double())
    want_dw = rnd(gy2).t() @ rnd(x2)
    edw = (w.grad.reshape(cout, cin).double() - want_dw).abs()
    assert (edw <= 1e-5 * (gy2.double().abs().t() @ x2.double().abs())).all(), float(edw.max())
    assert torch.allclose(b.grad.double(), gy2.double().sum(0), rtol=0, atol=1e-6 * float(gy2.abs().sum()))


# ---- 4. a whole stage-1 step ----------------------------------------------------------------------------------------
def compare(got, want, tol_l2, tol_cos, what):
    worst, dot, na, nb = ('', 0.0), 0.0, 0.0, 0.0
    errs = {}
    for k in want:
        a, w = got[k].double(), want[k].double()
        e = errs[k] = float((a - w).norm() / w.norm().clamp_min(1e-30))
        worst = (k, e) if e > worst[1] else worst
        dot += float((a * w).sum()); na += float((a * a).sum()); nb += float((w * w).sum())
    cos = dot / (na * nb) ** 0.5
    print(f'{what}: {len(want)} tensors, worst relative L2 {worst[0]} {worst[1]:.2e}, cosine {cos:.6f}; largest: ' +
          ', '.join(f'{k} {e:.1e}' for k, e in sorted(errs.items(), key=lambda kv: -kv[1])[:12]))
    assert worst[1] < tol_l2, worst
    assert cos > tol_cos, cos
    return worst[1], cos


def test_stage1_step_against_fp32(dev):
    """N = 1024, B = 2, K = 128, 3 iterations: every parameter gradient and both input gradients against the 'fp32' mode."""
    pc1, pc2 = clouds(2, 1024, 11, dev)
    m = make_model(dev, seed=2, mode='fp32')
    flows32, g32, in32 = step(m, pc1, pc2, 3, inputs=True)
    flows16, g16, in16 = step(m.set_precision('bf16-mixed'), pc1, pc2, 3, inputs=True)
    assert len(g16) == 95 and all(v is not None and torch.isfinite(v).all() for v in g16.values())
    e_flow = float((flows16[-1] - flows32[-1]).abs().mean() / flows32[-1].abs().mean())
    print(f'bf16-mixed step: flow mean-abs / mean|flow| vs fp32 {e_flow:.2e}')
    assert not torch.equal(flows16[-1], flows32[-1]) and e_flow < 2e-2   # measured 6.7e-3
    # The full gradient: cosine > 0.999 (measured 0.99997).  Per tensor, a relative L2 of 5e-2 holds for the update block
    # only (measured 4.3e-2).  Further upstream every gradient has passed through the bf16 dx of three iterations of loop
    # layers, and the feature encoder's gradient arrives only through the sparse correlation backward (the K kept entries
    # of a row, behind the lookup's voxel means and kNN max): smaller, cancellation-heavy tensors whose relative error the
    # bf16 noise of the loop (6.7e-3 in the flows) dominates.  The bounds below are about twice the measured values:
    for prefix, tol_l2, tol_cos in (('update_block.', 1e-1, 0.9999),       # measured 4.3e-2, cosine 0.99999
                                    ('corr_block.', 2e-1, 0.995),          # 8.5e-2, 0.9988
                                    ('context_extractor.', 2e-1, 0.998),   # 8.5e-2, 0.99945
                                    ('feature_extractor.', 4e-1, 0.98)):   # 1.8e-1, 0.9932
        sub = [k for k in g32 if k.startswith(prefix)]
        compare({k: g16[k] for k in sub}, {k: g32[k] for k in sub}, tol_l2, tol_cos, prefix)
    compare(g16, g32, 4e-1, 0.999, 'parameter gradients')
    # the input gradients collect the same upstream noise (measured 1.3e-1 for xyz2, 8.3e-2 for xyz1; cosine 0.9965)
    compare({'xyz1': in16[0], 'xyz2': in16[1]}, {'xyz1': in32[0], 'xyz2': in32[1]}, 3e-1, 0.99, 'input gradients')


# ---- 5. bitwise ---------------------------------------------------------------------------------------------------------
def captured_step(m, pc1, pc2, iters):
    """The same step as step(), captured into one CUDA graph and replayed once."""
    m.train()
    cur = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        for _ in range(2):
            step(m, pc1, pc2, iters)
    cur.wait_stream(side)
    m.zero_grad(set_to_none=True)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        flows = m([pc1, pc2], num_iters=iters)
        sequence_loss(flows, pc2 - pc1).backward()
    g.replay()
    torch.cuda.synchronize()
    return [f.clone() for f in flows], {k: p.grad.detach().clone() for k, p in m.named_parameters()}


def test_eager_step_equals_captured_step(dev, deterministic, monkeypatch):
    """The loop's layers follow the mode's rule in eager steps too; the fp32 layers outside the loop follow
    PVRAFT_TC_TRAIN, pinned here so that eager and captured steps take the same kernels there."""
    from pvraft_b200 import train as T
    monkeypatch.setattr(T, '_TC_TRAIN', '1')
    pc1, pc2 = clouds(2, 1024, 12, dev)
    m = make_model(dev, seed=3)
    flows_e, g_e, _ = step(m, pc1, pc2, 3)
    flows_c, g_c = captured_step(m, pc1, pc2, 3)
    for a, b in zip(flows_e, flows_c):
        assert torch.equal(a, b)
    for k in g_e:
        assert torch.equal(g_e[k], g_c[k]), k


def test_deterministic_steps_are_bitwise_and_fp32_comes_back(dev, deterministic):
    pc1, pc2 = clouds(2, 1024, 13, dev)
    m = make_model(dev, seed=4)
    f1, g1, i1 = step(m, pc1, pc2, 3, inputs=True)
    f2, g2, i2 = step(m, pc1, pc2, 3, inputs=True)
    assert all(torch.equal(a, b) for a, b in zip(f1, f2))
    assert all(torch.equal(g1[k], g2[k]) for k in g1)
    assert torch.equal(i1[0], i2[0]) and torch.equal(i1[1], i2[1])
    # back to 'fp32': a fresh fp32 model's gradients, bit for bit
    _, g_back, _ = step(m.set_precision('fp32'), pc1, pc2, 3)
    _, g_fresh, _ = step(make_model(dev, seed=4, mode='fp32'), pc1, pc2, 3)
    assert not all(torch.equal(g1[k], g_fresh[k]) for k in g1)
    assert all(torch.equal(g_back[k], g_fresh[k]) for k in g_back)


def test_cuda_core_shapes_equal_fp32_training(dev, deterministic):
    """N % 128 != 0: nothing runs on the tensor cores, so the mode is 'fp32' bit for bit."""
    pc1, pc2 = clouds(2, 1000, 14, dev)
    f16, g16, i16 = step(make_model(dev, seed=5), pc1, pc2, 3, inputs=True)
    f32, g32, i32 = step(make_model(dev, seed=5, mode='fp32'), pc1, pc2, 3, inputs=True)
    assert all(torch.equal(a, b) for a, b in zip(f16, f32))
    assert all(torch.equal(g16[k], g32[k]) for k in g16)
    assert torch.equal(i16[0], i32[0]) and torch.equal(i16[1], i32[1])


# ---- 6. inference in the mode -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('refine', [False, True], ids=['RSF', 'RSF_refine'])
def test_pre_loop_state_equals_fp32(dev, refine, deterministic):
    m = make_model(dev, refine=refine, seed=6, mode='fp32').eval()
    pc1, pc2 = clouds(2, 2048, 8, dev, scale=1.0)
    runs = []
    for mode in ('fp32', 'bf16-mixed'):
        m.set_precision(mode)
        with torch.no_grad():
            _, _, graph, graph_context, net, inp = m._encode([pc1, pc2])
        cb = m.corr_block
        runs.append((cb.corr_val.clone(), cb.corr_idx.clone(), graph.nbr.clone(), graph._rel.clone(), graph_context.nbr.clone(),
                     graph_context._rel.clone(), net, inp))
    assert runs[1][0].dtype == torch.float32 and runs[1][1].dtype == torch.int32
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize('refine', [False, True], ids=['RSF', 'RSF_refine'])
def test_inference_accuracy_against_the_oracle(dev, refine):
    """Free-running, 8 iterations, N = 1024, K = 128: mean-abs / mean|flow| < 1e-2."""
    from pvraft_b200 import RSF, RSF_refine
    args = types.SimpleNamespace(corr_levels=LEVELS, base_scales=SCALE, truncate_k=128)
    torch.manual_seed(0)
    m = (RSF_refine if refine else RSF)(args).to(dev).eval()
    pc1, pc2 = O.synthetic_clouds(2, 1024, seed=13)
    W = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    with torch.no_grad():
        want = (O.rsf_refine_forward if refine else O.rsf_forward)(W, pc1, pc2, 8, LEVELS, SCALE, 128)
        got = m.set_precision('bf16-mixed')([pc1.to(dev), pc2.to(dev)], 8)
    pick = (lambda x: x) if refine else (lambda x: x[-1])
    err = float((pick(got).cpu() - pick(want)).abs().mean() / pick(want).abs().mean())
    print(f'bf16-mixed inference (refine={refine}): mean-abs / mean|flow| vs oracle {err:.2e}')
    assert err < 1e-2   # measured 3.0e-3 (RSF), 5.1e-3 (RSF_refine)


def test_inference_fused_chain_equals_unfused(dev):
    from pvraft_b200 import ops
    m = make_model(dev, seed=1).eval()
    m.use_cuda_graph = False
    pc1, pc2 = clouds(2, 4096, 5, dev, scale=1.0)
    with torch.no_grad():
        got = m([pc1, pc2], 4)
        ops.fuse_update_chain = False
        try:
            want = m([pc1, pc2], 4)
        finally:
            ops.fuse_update_chain = True
        fp32 = m.set_precision('fp32')([pc1, pc2], 4)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert not torch.equal(got[-1], fp32[-1])


def test_refine_training_in_the_mode(dev):
    """RSF_refine trains its fp32 refiner behind the no-grad loop, which runs in the mode; input gradients work too."""
    m = make_model(dev, refine=True, seed=0)
    m.train()
    pc1, pc2 = clouds(1, 1024, 3, dev)
    x1 = pc1.clone().requires_grad_(True)
    out = m([x1, pc2], 2)
    out.abs().mean().backward()
    grads = [p.grad for p in m.refine_block.parameters()]
    assert all(g is not None and torch.isfinite(g).all() for g in grads)
    assert x1.grad is not None and torch.isfinite(x1.grad).all()


# ---- 7. a short training run ---------------------------------------------------------------------------------------------
def test_short_training_run_follows_fp32(dev):
    """20 Adam steps (lr 1e-3) on one fixed pair, N = 1024, B = 2, K = 128, 3 iterations: the final loss of the mode within
    10 % of the 'fp32' loop's, and both well below the first step's."""
    pc1, pc2 = clouds(2, 1024, 15, dev)
    losses = {}
    for mode in ('fp32', 'bf16-mixed'):
        m = make_model(dev, seed=7, mode=mode).train()
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        hist = []
        for _ in range(20):
            opt.zero_grad(set_to_none=True)
            loss = sequence_loss(m([pc1, pc2], num_iters=3), pc2 - pc1)
            loss.backward()
            opt.step()
            hist.append(float(loss))
        losses[mode] = hist
    ratio = losses['bf16-mixed'][-1] / losses['fp32'][-1]
    print(f"20 Adam steps: fp32 {losses['fp32'][0]:.4f} -> {losses['fp32'][-1]:.4f}, "
          f"bf16-mixed {losses['bf16-mixed'][0]:.4f} -> {losses['bf16-mixed'][-1]:.4f}, ratio {ratio:.4f}")
    assert all(l[-1] < 0.9 * l[0] for l in losses.values())
    assert 0.9 < ratio < 1.1   # measured 0.2561 / 0.2543 = 1.007 (from 1.61)
