"""GroupNorm statistics where a group's mean is large next to its spread.

Every GroupNorm of the library reads its statistics from raw sums (sum x, sum x^2) in [B,8,2] doubles, and its consumer
takes var = sum x^2 / n - mean^2 (csrc/common.cuh gn_affine; the backward's gn_mean_rstd).  When a group's mean is r
times its standard deviation that subtraction cancels: the variance keeps only a relative 1 / (1 + r^2) of what the sums
carry, so the sums must be accurate far beyond fp32.  These tests sweep r over R_SWEEP by adding a per-group offset where a
layer carries one (a bias, a residual, the edge features, the incoming edge tensor, the correlation values and the kNN
conv bias) and check:

  statistics   every producer of the sums (k_linear, k_tc_linear in 3xTF32 and bf16, resident and streamed weights,
               k_setconv_edge_pairs on the row table and on the global gather, k_edge_fwd, the lookup's moments), in the
               default and the deterministic form: mean and variance taken from the kernel's sums the way gn_affine
               takes them, against a float64 two-pass over the values the kernel summed -- its own fp32 output where it
               writes one, else (SetConv edge kernel) y recomputed from the fp32 inputs in the kernel's fp32 operation
               order, so that neither the GEMM's error nor the fp32 rounding of y enters.
                 variance within VAR_TOL relative, mean within MEAN_TOL (|mean| + std) (SetConv edge kernel:
                 MEAN_TOL_EDGE), at every r.
  consumers    gn_act, the tc_linear GroupNorm prologue (with and without the min array), gn_act_maxk, gn_act_bwd's dx and
               the kNN branch, fed sums of the same values, against float64 GroupNorm(+activation).  A fused fp32 affine
               fmaf(x, scale, shift) with scale and shift rounded to fp32 cannot do better than a few roundings of
               |x scale| + |shift|:
                 |error| <= C_AFFINE 2^-24 (|x scale| + |shift|)   (dx: times what multiplies the normalised value)
  the model    GroupNorm is exactly invariant to one constant added to every channel of a group, so shifting the bias of
               a layer that feeds a GroupNorm (corr_block.out_conv.0 and knn_conv.0: the SetConv fc layers have no bias)
               by r std per group must leave RSF's flow and its training gradients unchanged up to the fp32 rounding of
               y + c, ~2^-24 r relative to the group's spread.  The first RAFT iteration looks up at the unmoved
               coordinates, so its flow is a continuous function of the statistics: there the error is bounded by
               C_ITER1 r 2^-24 and must grow linearly (a factor < 30 per factor 10 of r, from r = 100; r = 10 sits at an
               r-independent rounding floor).  Free-running, the drifting coordinates can flip a voxel cell or a kNN
               near-tie, a jump of fixed size (~4e-5 here) whatever r: bounded by C_SHIFT r 2^-24 + FLIP_TOL.

Every uninitialised allocation is NaN-filled for these tests.  Measured errors per r are printed with -s.
"""
import contextlib
import math
import types

import pytest
import torch

from conftest import default_weights
from oracle import pvraft_oracle as O
from train_helpers import sequence_loss

pytestmark = pytest.mark.gpu

R_SWEEP = (0, 3, 30, 300, 3000)
VAR_TOL, MEAN_TOL = 1e-6, 1e-9
# k_setconv_edge_pairs sums a point's 32 edges in plain fp32 (a compensated sum spills in its one-pair form): its mean of a
# zero-mean group measures up to 1.2e-9 of the spread (r = 0, C = 32, global gather)
MEAN_TOL_EDGE = 2e-9
U = 2.0 ** -24
C_AFFINE = 8      # fmaf (1) + fp32 scale (1) + fp32 shift (1) + tf32 hi/lo split of the prologue output (3) + slack
C_ITER1 = 1        # first-iteration flow, r >= 100 (measured <= 0.22; sums with a 2^-24 r^2 error: 4.2 at r = 1000)
C_SHIFT = 8        # free-running flow, on top of FLIP_TOL (measured <= 4.9 at r = 10000; old sums: 51 at 1000, 1270 at 10000)
FLIP_TOL = 1e-4    # one discrete decision (a voxel cell or kNN near-tie) flipped by the coordinates' drift: measured 4.3e-5
C_SHIFT_GRAD = 5   # one-iteration training step, relative L2 (measured <= 2.3; old sums: 10.2 at r = 1000)


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def sm_count():
    from pvraft_b200 import ops
    return ops.device_info()[0]


@pytest.fixture(autouse=True)
def _poison_uninitialised(monkeypatch):
    """Always on here: every torch.empty / empty_like / new_empty allocation is NaN-filled (integers: max // 2)."""
    real_empty, real_like, real_new = torch.empty, torch.empty_like, torch.Tensor.new_empty

    def fill(t):
        if t.is_floating_point():
            t.fill_(float('nan'))
        elif t.dtype != torch.bool:
            t.fill_(torch.iinfo(t.dtype).max // 2)
        return t

    monkeypatch.setattr(torch, 'empty', lambda *a, **k: fill(real_empty(*a, **k)))
    monkeypatch.setattr(torch, 'empty_like', lambda *a, **k: fill(real_like(*a, **k)))
    monkeypatch.setattr(torch.Tensor, 'new_empty', lambda self, *a, **k: fill(real_new(self, *a, **k)))
    yield


@contextlib.contextmanager
def det_mode(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


# ----------------------------------------------------------------------------------------------------------------------
# helpers
# ----------------------------------------------------------------------------------------------------------------------
def groups(y):
    """[B, rows, C] -> [B, 8, rows * C / 8] (GroupNorm's 8 groups of C / 8 consecutive channels)."""
    b, c = y.shape[0], y.shape[-1]
    return y.reshape(b, -1, 8, c // 8).transpose(1, 2).reshape(b, 8, -1)


def two_pass(y64):
    """float64 two-pass mean and (biased) variance per sample and group."""
    g = groups(y64)
    mean = g.mean(-1)
    return mean, ((g - mean.unsqueeze(-1)) ** 2).mean(-1)


def group_std(y64):
    """Per-group standard deviation pooled over the samples -> [8]."""
    return y64.reshape(-1, 8, y64.shape[-1] // 8).transpose(0, 1).reshape(8, -1).std(1)


def group_offset(std8, r, c):
    """A per-channel offset that is r std_g for every channel of group g, with alternating signs across groups -> [C]."""
    sign = torch.tensor([1.0 if g % 2 == 0 else -1.0 for g in range(8)], dtype=torch.float64, device=std8.device)
    return (r * std8 * sign).repeat_interleave(c // 8)


def raw_sums(x64):
    """[B, rows, C] -> the [B,8,2] sums the library passes between layers."""
    g = groups(x64)
    return torch.stack([g.sum(-1), (g * g).sum(-1)], -1).contiguous()


def stats_errors(stats, y64):
    """(variance error / variance, mean error / (|mean| + std), largest |mean| / std) of the kernel's sums `stats` against a
    float64 two-pass over the values y64 [B, rows, C] they summarise; mean and variance taken the way gn_affine takes them."""
    n = y64[0].numel() // 8
    mean_k = stats[..., 0] / n
    var_k = stats[..., 1] / n - mean_k * mean_k
    mean, var = two_pass(y64)
    std = var.sqrt()
    ev = float(((var_k - var).abs() / var).max())
    em = float(((mean_k - mean).abs() / (mean.abs() + std)).max())
    return ev, em, float((mean.abs() / std).max())


def report_and_check(label, rows, mean_tol=MEAN_TOL):
    """rows: [(r, (variance error, mean error, measured r))] -> one printed line; every r within the bounds."""
    print(f'{label}: ' + '  '.join(f'r={r} (measured {m:.3g}): var {ev:.1e} mean {em:.1e}' for r, (ev, em, m) in rows))
    for r, (ev, em, _) in rows:
        assert ev <= VAR_TOL and em <= mean_tol, (label, r, ev, em)


def affine64(mean, var, gamma, beta, c):
    """float64 GroupNorm scale / shift per sample and channel ([B, C]) from per-group mean / variance ([B, 8])."""
    rstd = (var + 1e-5).rsqrt()
    sc = rstd.repeat_interleave(c // 8, 1) * gamma.double()
    return sc, beta.double() - mean.repeat_interleave(c // 8, 1) * sc


def lrelu(t, slope=0.1):
    return torch.where(t >= 0, t, slope * t)


def fma32(a, b, c):
    """fmaf on float32 tensors: the product is exact in float64, so one rounding to float32 of the float64 sum (a double
    rounding can differ from fmaf in the last bit only at exact ties)."""
    return (a.double() * b.double() + c.double()).float()


# ----------------------------------------------------------------------------------------------------------------------
# producers
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('det', [False, True], ids=['default', 'det'])
@pytest.mark.parametrize('residual', [False, True], ids=['bias', 'residual'])
@pytest.mark.parametrize('k', [32, 512], ids=['resident', 'streamed'])
@pytest.mark.parametrize('cout', [32, 64, 128])
@pytest.mark.parametrize('operands', ['3xtf32', 'bf16'])
def test_tc_linear_statistics(dev, sm_count, operands, cout, k, residual, det):
    """k_tc_linear's plain epilogue: out = x W^T + bias (+ residual) with the group offset in the bias or in the residual.
    B = 3, N = 6144: 144 tiles, more than the SMs, so CTAs carry tiles of two samples.  K = 32 keeps every width's
    weights resident, K = 512 streams them with every k-block (test_gpu_kernel_coverage.py: test_tc_matrix_takes_both_weight_paths)."""
    from pvraft_b200 import ops
    b, n = 3, 6144
    assert b * n // 128 > sm_count
    g = torch.Generator().manual_seed(cout * 7 + k + residual)
    x = torch.randn(b, n, k, generator=g).to(dev)
    w = (torch.randn(cout, k, generator=g) / k ** 0.5).to(dev)
    std8 = group_std(x.double() @ w.double().t())
    noise = torch.randn(cout, generator=g).double().to(dev) * 0.1
    res0 = (torch.randn(b, n, cout, generator=g) * 0.5).double().to(dev)
    tw = ops.tc_weights(w, bf16=operands == 'bf16')
    rows = []
    for r in R_SWEEP:
        off = group_offset(std8, r, cout)
        bias, res = (noise.float(), (res0 + off).float()) if residual else ((off + noise).float(), None)
        stats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
        with det_mode(det):
            y = ops.tc_linear([x], tw, bias, residual=res, out_stats=stats)
        rows.append((r, stats_errors(stats, y.double())))
    report_and_check(f'tc_linear {operands} cout={cout} K={k} {"residual" if residual else "bias"} '
                     f'{"det" if det else "default"}', rows)


@pytest.mark.parametrize('det', [False, True], ids=['default', 'det'])
@pytest.mark.parametrize('residual', [False, True], ids=['bias', 'residual'])
@pytest.mark.parametrize('cout', [32, 64, 128])
def test_linear_statistics(dev, cout, residual, det):
    """k_linear (the CUDA-core layer, double per element): the control.  N = 1000 is ragged for 128-point tiles."""
    from pvraft_b200 import ops
    b, n, k = 3, 1000, 64
    g = torch.Generator().manual_seed(cout + 3 * residual)
    x = torch.randn(b, n, k, generator=g).to(dev)
    w = (torch.randn(cout, k, generator=g) / k ** 0.5).to(dev)
    std8 = group_std(x.double() @ w.double().t())
    res0 = (torch.randn(b, n, cout, generator=g) * 0.5).double().to(dev)
    rows = []
    for r in R_SWEEP:
        off = group_offset(std8, r, cout)
        bias, res = (torch.zeros(cout, device=dev), (res0 + off).float()) if residual else (off.float(), None)
        stats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
        with det_mode(det):
            y = ops.linear(x, w, bias, residual=res, out_stats=stats)
        rows.append((r, stats_errors(stats, y.double())))
    report_and_check(f'linear cout={cout} {"residual" if residual else "bias"} {"det" if det else "default"}', rows)


def edge_y32(P, nbr, ef, w, cin):
    """y = (P_j - P_i) + fma(w_z, e_z, fma(w_y, e_y, w_x e_x)) in float32, in the edge kernel's operation order, one sample:
    P [N,C], nbr [N,32], ef [N,32,3] -> [N*32, C]."""
    wx, wy, wz = w[:, cin], w[:, cin + 1], w[:, cin + 2]
    ex, ey, ez = ef[..., 0:1], ef[..., 1:2], ef[..., 2:3]
    t = fma32(wz, ez, fma32(wy, ey, wx * ex))
    return ((P[nbr.long()] - P.unsqueeze(1)) + t).reshape(-1, P.shape[-1])


def overflow_fraction(nbr, order, c):
    """Share of 32-point tiles (in processing order) whose distinct rows exceed the edge kernel's row table."""
    b, n, _ = nbr.shape
    rows = min(22528 // c, 32 * 33)
    o = order.long() if order is not None else torch.arange(n, device=nbr.device).expand(b, n)
    over = total = 0
    for s in range(b):
        for t0 in range(0, n, 32):
            pts = o[s, t0:t0 + 32]
            refs = torch.cat([nbr[s, pts].reshape(-1).long(), pts])
            over += int(len(torch.unique(refs)) > rows)
            total += 1
    return over / total


@pytest.mark.parametrize('det', [False, True], ids=['default', 'det'])
@pytest.mark.parametrize('case', ['knn-morton', 'knn-index', 'random-index'])
@pytest.mark.parametrize('c', [32, 64, 128])
def test_setconv_edge_statistics(dev, c, case, det):
    """k_setconv_edge_pairs: the group offset rides on the edge features (rel + (d, 0, 0), with fc1's x column w_x = r std_g / d
    common to a group).  B = 3, N = 4100 (a ragged last tile).  knn-morton gathers from the shared-memory row table (most tiles
    fit), random-index from global memory (most tiles overflow it)."""
    from pvraft_b200 import ops
    b, n, cin, d = 3, 4100, 64, 1e5
    g = torch.Generator().manual_seed(c * 3 + len(case))
    pc, _ = O.synthetic_clouds(b, n, seed=c)
    pcd = pc.to(dev)
    nbr, rel = ops.knn(pcd, pcd, 32, mode=0, want_rel=True)
    if case == 'random-index':
        nbr = torch.randint(0, n, (b, n, 32), generator=g).to(torch.int32).to(dev)
        rel = (torch.randn(b, n, 32, 3, generator=g) * 0.3).to(dev)
    order = ops.point_order(pcd) if case == 'knn-morton' else None
    frac = overflow_fraction(nbr, order, c)
    if case == 'knn-morton' and c <= 64:   # (C = 128: a 176-row table, which a Morton tile of this cloud often overflows)
        assert frac < 0.1, frac
    if case == 'random-index':
        assert frac > 0.9, frac
    P = torch.randn(b, n, c, generator=g).to(dev)
    w = torch.randn(c, cin + 3, generator=g).to(dev)
    w[:, cin] = 0
    ef = rel.clone()
    ef[..., 0] += d
    base = torch.cat([edge_y32(P[s], nbr[s], rel[s], w, cin) for s in range(b)]).double()
    std8 = group_std(base.view(b, -1, c))
    rows = []
    for r in R_SWEEP:
        w[:, cin] = (group_offset(std8, r, c) / d).float()
        stats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
        with det_mode(det):
            ymax, ymin = ops.setconv_edge(P, nbr, ef, w, cin, stats, order=order)
        y = torch.stack([edge_y32(P[s], nbr[s], ef[s], w, cin) for s in range(b)])
        # the kernel's max / min of its own y are these values' max / min (up to an fmaf tie)
        yv = y.view(b, n, 32, c)
        assert float((ymax - yv.amax(2)).abs().max()) <= 2 * U * float(yv.abs().max())
        assert float((ymin - yv.amin(2)).abs().max()) <= 2 * U * float(yv.abs().max())
        rows.append((r, stats_errors(stats, y.double())))
        del y, yv
    report_and_check(f'setconv_edge C={c} {case} (overflowing tiles {frac:.0%}) {"det" if det else "default"}', rows, MEAN_TOL_EDGE)


@pytest.mark.parametrize('det', [False, True], ids=['default', 'det'])
@pytest.mark.parametrize('c', [32, 64, 128])
def test_edge_fwd_statistics(dev, c, det):
    """k_edge_fwd (the training path's SetConv edge stage): T = P[nbr] - P + E in place, the group offset in the incoming E.
    B = 3, N = 1001: CTAs of 8 points straddle samples."""
    from pvraft_b200 import ops
    b, n = 3, 1001
    g = torch.Generator().manual_seed(c + 11)
    P = torch.randn(b, n, c, generator=g).to(dev)
    nbr = torch.randint(0, n, (b, n, 32), generator=g).to(torch.int32).to(dev)
    E0 = torch.randn(b, n * 32, c, generator=g).double().to(dev)
    idx = nbr.long().view(b, n * 32, 1).expand(b, n * 32, c)
    base = torch.gather(P.double(), 1, idx) - P.double().repeat_interleave(32, 1) + E0
    std8 = group_std(base)
    rows = []
    for r in R_SWEEP:
        E = (E0 + group_offset(std8, r, c)).float().contiguous()
        stats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
        with det_mode(det):
            T = ops.edge_fwd(P, nbr, E, stats)
        rows.append((r, stats_errors(stats, T.double())))
    report_and_check(f'edge_fwd C={c} {"det" if det else "default"}', rows)


def knn_args(dev, sel, mom, w, bk, gamma, beta, slope):
    from pvraft_b200 import _lib, ops
    b, n = sel.shape[:2]
    kfeat, cflow = torch.empty(b, n, 64, device=dev), torch.empty(b, n, 64, device=dev)
    flow = torch.zeros(b, n, 3, device=dev)
    w_cf, b_cf = torch.zeros(64, 3, device=dev), torch.zeros(64, device=dev)
    preluk = torch.tensor([slope], dtype=torch.float32, device=dev)
    a = _lib.KnnBranchArgs()
    a.knn_sel, a.moments = ops._p(sel), ops._p(mom, torch.float64)
    a.w_knn, a.b_knn, a.gnk_gamma, a.gnk_beta, a.preluk = ops._p(w), ops._p(bk), ops._p(gamma), ops._p(beta), ops._p(preluk)
    a.preluk_host = slope
    a.kfeat, a.flow, a.w_cf, a.b_cf, a.cflow = ops._p(kfeat), ops._p(flow), ops._p(w_cf), ops._p(b_cf), ops._p(cflow)
    a.B, a.N = b, n
    ops.knn_branch(a)
    return kfeat


@pytest.mark.parametrize('det', [False, True], ids=['default', 'det'])
@pytest.mark.parametrize('corr_offset', [0.0, 300.0])
def test_lookup_moments_and_knn_branch(dev, corr_offset, det):
    """The moment path: k_corr_lookup's moments of the gathered kNN vectors f = (corr, dx, dy, dz) (correlations ~ N(20, 5),
    shifted by corr_offset), from which knn_conv.0's GroupNorm statistics follow in closed form, t = W f + b with the group
    offset in b.  Statistics: the closed form (float64, from the kernel's moments) against a float64 two-pass over t
    computed from the kernel's own knn_sel.  Consumer: k_knn_branch's kfeat = max over the 32 candidates of
    PReLU(GN(t)) against float64, with the bound taken over |W f| + |b|, the magnitude t is rounded at."""
    from pvraft_b200 import CorrBlock
    b, n, k, slope = 3, 1000, 64, 0.25
    state, coords, xyz2 = O.synthetic_state(b, n, k, seed=5, box=3.0)
    cb = CorrBlock(num_levels=3, base_scale=0.25, truncate_k=k).to(dev)
    cb.set_state((state.truncated_corr + corr_offset).to(dev), state.indices.to(torch.int32).to(dev), xyz2.to(dev))
    g = torch.Generator().manual_seed(int(corr_offset) + 1)
    w = (torch.randn(64, 4, generator=g) * 0.5).to(dev)
    gamma = (torch.randn(64, generator=g) * 0.5 + 0.3).to(dev)
    beta = (torch.randn(64, generator=g) * 0.2).to(dev)
    with det_mode(det):
        lk = cb.lookup(coords.to(dev))
    sel64 = lk['knn_sel'].double().reshape(b, n * 32, 4)
    mom = lk['moments'].double()
    w64 = w.double()
    std8 = group_std(sel64 @ w64.t())
    iu = torch.triu_indices(4, 4)
    M = torch.zeros(b, 4, 4, dtype=torch.float64, device=dev)
    M[:, iu[0], iu[1]] = mom[:, 4:14]
    M = M + M.transpose(1, 2) - torch.diag_embed(torch.diagonal(M, dim1=1, dim2=2))
    cnt = mom[:, 14:15]
    rows, cons = [], []
    for r in R_SWEEP:
        bk64 = group_offset(std8, r, 64)
        bk = bk64.float()
        t64 = sel64 @ w64.t() + bk.double()
        # closed form of the GroupNorm statistics of t from the moments (as the consumers derive them)
        m1 = mom[:, :4] @ w64.t() / cnt                                      # [B,64] E[W f]
        m2 = torch.einsum('ci,bij,cj->bc', w64, M, w64) / cnt                # [B,64] E[(W f)^2]
        bd = bk.double()
        mean_c, sq_c = m1 + bd, m2 + 2 * bd * m1 + bd * bd
        mean_k = mean_c.view(b, 8, 8).mean(-1)
        var_k = sq_c.view(b, 8, 8).mean(-1) - mean_k ** 2
        mean, var = two_pass(t64)
        std = var.sqrt()
        rows.append((r, (float(((var_k - var).abs() / var).max()), float(((mean_k - mean).abs() / (mean.abs() + std)).max()),
                         float((mean.abs() / std).max()))))
        kfeat = knn_args(dev, lk['knn_sel'], lk['moments'], w, bk, gamma, beta, slope)
        sc, sh = affine64(mean, var, gamma, beta, 64)
        tn = t64 * sc.unsqueeze(1) + sh.unsqueeze(1)
        want = torch.where(tn >= 0, tn, slope * tn).view(b, n, 32, 64).amax(2)
        mag = ((sel64.unsqueeze(-1) * w64.t()).abs().sum(-2) + bd.abs()) * sc.abs().unsqueeze(1) + sh.abs().unsqueeze(1)
        bound = C_AFFINE * U * mag.view(b, n, 32, 64).amax(2)
        err = (kfeat.double() - want).abs()
        cons.append(float((err / bound).max()))
        assert bool((err <= bound).all()), (r, float((err / bound).max()))
    report_and_check(f'lookup moments (corr offset {corr_offset}) {"det" if det else "default"}', rows)
    print(f'  knn_branch kfeat error / bound per r: ' + ' '.join(f'{e:.2f}' for e in cons))


@pytest.mark.parametrize('det', [False, True], ids=['default', 'det'])
def test_corr_feature_gn_affines(dev, det):
    """k_corrfeat (the CUDA-core correlation feature, N % 128 != 0): corr = out_conv.3(PReLU(GN(y1))) + knn_out(max over the 32
    candidates of PReLU(GN(knn_conv.0 f))), where it derives the first GroupNorm from k_linear's sums of y1 and the second
    in closed form from the lookup's moments.  The group offsets ride on out_conv.0's and knn_conv.0's biases.  Against
    float64 from the kernels' own y1 and knn_sel; the bound carries the affine rounding (C_AFFINE 2^-24 (|x scale| +
    |shift|)) through the output layers' |W|, plus the fp32 rounding of their 192-term dot products."""
    from pvraft_b200 import CorrBlock
    b, n, k = 3, 1000, 64
    state, coords, xyz2 = O.synthetic_state(b, n, k, seed=9, box=3.0)
    torch.manual_seed(9)
    cb = CorrBlock(num_levels=3, base_scale=0.25, truncate_k=k).to(dev)
    cb.set_state(state.truncated_corr.to(dev), state.indices.to(torch.int32).to(dev), xyz2.to(dev))
    oc, kc = cb.out_conv, cb.knn_conv
    with torch.no_grad():
        for gn in (oc[1], kc[1]):
            gn.weight.copy_(torch.randn(gn.weight.shape, generator=torch.Generator().manual_seed(gn.weight.numel())))
        oc[2].weight.fill_(0.25)
        kc[2].weight.fill_(-0.3)
    b_oc, b_kc = oc[0].bias.detach().clone(), kc[0].bias.detach().clone()
    std_oc = std_kc = None
    worst = []
    for r in R_SWEEP:
        with torch.no_grad():
            if std_oc is not None:
                oc[0].bias.copy_(b_oc + group_offset(std_oc, r, 128).float())
                kc[0].bias.copy_(b_kc + group_offset(std_kc, r, 64).float())
            with det_mode(det):
                corr, (lk, y1, _, _) = cb.feature_point_major(coords.to(dev))
        y64 = y1.double()
        sel64 = lk['knn_sel'].double().reshape(b, n * 32, 4)
        wk = kc[0].weight.detach().double().reshape(64, 4)
        t64 = sel64 @ wk.t() + kc[0].bias.detach().double()
        if std_oc is None:   # r = 0 comes first: the groups' spreads
            std_oc, std_kc = group_std(y64 - oc[0].bias.detach().double()), group_std(t64)
        m1, v1 = two_pass(y64)
        sc1, sh1 = affine64(m1, v1, oc[1].weight.detach(), oc[1].bias.detach(), 128)
        u1 = y64 * sc1.unsqueeze(1) + sh1.unsqueeze(1)
        a1 = torch.where(u1 >= 0, u1, 0.25 * u1)
        mag1 = (y64 * sc1.unsqueeze(1)).abs() + sh1.abs().unsqueeze(1)
        m2, v2 = two_pass(t64)
        sc2, sh2 = affine64(m2, v2, kc[1].weight.detach(), kc[1].bias.detach(), 64)
        u2 = t64 * sc2.unsqueeze(1) + sh2.unsqueeze(1)
        kf = torch.where(u2 >= 0, u2, -0.3 * u2).view(b, n, 32, 64).amax(2)
        mag2 = (((sel64.unsqueeze(-1) * wk.t()).abs().sum(-2) + kc[0].bias.detach().double().abs()) * sc2.abs().unsqueeze(1)
                + sh2.abs().unsqueeze(1)).view(b, n, 32, 64).amax(2)
        w3, b3 = oc[3].weight.detach().double().reshape(64, 128), oc[3].bias.detach().double()
        wo, bo = cb.knn_out.weight.detach().double().reshape(64, 64), cb.knn_out.bias.detach().double()
        want = a1 @ w3.t() + b3 + kf @ wo.t() + bo
        bound = (C_AFFINE * U * (mag1 @ w3.abs().t() + mag2 @ wo.abs().t())
                 + 192 * U * (a1.abs() @ w3.abs().t() + kf.abs() @ wo.abs().t() + b3.abs() + bo.abs()))
        err = (corr.double() - want).abs()
        worst.append((r, float((err / bound).max())))
    print(f'corr_feature {"det" if det else "default"} error / bound per r: ' + ' '.join(f'r={r}: {e:.3f}' for r, e in worst))
    assert all(e <= 1 for _, e in worst), worst


# ----------------------------------------------------------------------------------------------------------------------
# consumers
# ----------------------------------------------------------------------------------------------------------------------
def consumer_input(dev, b, rows, c, r, seed):
    """x [B, rows, C] = N(0, 1) + r per group (alternating signs), gamma with negative entries, beta, and the float64 sums."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(b, rows, c, generator=g).double() + group_offset(torch.ones(8, dtype=torch.float64), r, c)).float().to(dev)
    gamma = torch.randn(c, generator=g).to(dev)
    beta = (torch.randn(c, generator=g) * 0.2).to(dev)
    assert (gamma < 0).any() and (gamma > 0).any()
    return x, gamma, beta, raw_sums(x.double())


@pytest.mark.parametrize('c', [32, 64, 128])
def test_gn_act_consumers(dev, c):
    """gn_act and gn_act_maxk (y = max over a point's 32 rows of LReLU(GN(x))) against float64, B = 3, 1000 points."""
    from pvraft_b200 import ops
    b, pts = 3, 1000
    worst = []
    for r in R_SWEEP:
        x, gamma, beta, st = consumer_input(dev, b, pts * 32, c, r, seed=c + r)
        mean, var = two_pass(x.double())
        sc, sh = affine64(mean, var, gamma, beta, c)
        x64 = x.double()
        want = lrelu(x64 * sc.unsqueeze(1) + sh.unsqueeze(1))
        mag = (x64 * sc.unsqueeze(1)).abs() + sh.abs().unsqueeze(1)
        bound = C_AFFINE * U * mag
        cnt = float(pts * 32 * c // 8)
        got = ops.gn_act(x, st, gamma, beta, cnt, ops.ACT_LRELU, 0.1)
        e1 = float(((got.double() - want).abs() / bound).max())
        ym, _ = ops.gn_act_maxk(x, st, gamma, beta, cnt, ops.ACT_LRELU, 0.1)
        e2 = float(((ym.double() - want.view(b, pts, 32, c).amax(2)).abs() / bound.view(b, pts, 32, c).amax(2)).max())
        worst.append((r, e1, e2))
    print(f'gn_act C={c} error / bound per r: ' + '  '.join(f'r={r}: gn_act {e1:.2f} maxk {e2:.2f}' for r, e1, e2 in worst))
    assert all(e1 <= 1 and e2 <= 1 for _, e1, e2 in worst), worst


@pytest.mark.parametrize('minmax', [False, True], ids=['gn', 'gn-minmax'])
@pytest.mark.parametrize('c', [32, 64, 128])
def test_tc_linear_prologue_consumer(dev, c, minmax):
    """The tc_linear GroupNorm prologue (fp32 operands) through identity weights: out = LReLU(GN(raw)) with raw the max or,
    where the folded scale is negative, the min array (GN_MINMAX).  The identity's 3xTF32 product returns its operand to
    within the hi / lo split (counted in C_AFFINE)."""
    from pvraft_b200 import ops
    b, n = 3, 1024
    tw = ops.tc_weights(torch.eye(c, device=dev))
    worst = []
    for r in R_SWEEP:
        x, gamma, beta, st = consumer_input(dev, b, n, c, r, seed=3 * c + r + minmax)
        xmin = (x - torch.rand(b, n, c, generator=torch.Generator().manual_seed(r)).to(dev)) if minmax else None
        mean, var = two_pass(x.double())
        sc, sh = affine64(mean, var, gamma, beta, c)
        raw = x.double() if xmin is None else torch.where(sc.unsqueeze(1) < 0, xmin.double(), x.double())
        want = lrelu(raw * sc.unsqueeze(1) + sh.unsqueeze(1))
        bound = C_AFFINE * U * ((raw * sc.unsqueeze(1)).abs() + sh.abs().unsqueeze(1))
        got = ops.tc_linear([x], tw, None, in_min=xmin, in_stats=st, in_gamma=gamma, in_beta=beta, in_count=float(n * c // 8),
                            in_act=ops.ACT_LRELU, in_slope=0.1)
        worst.append((r, float(((got.double() - want).abs() / bound).max())))
    print(f'tc_linear prologue C={c} {"minmax" if minmax else "gn"} error / bound per r: ' +
          ' '.join(f'r={r}: {e:.2f}' for r, e in worst))
    assert all(e <= 1 for _, e in worst), worst


@pytest.mark.parametrize('c', [32, 64, 128])
def test_gn_act_bwd_consumer(dev, c):
    """gn_act_bwd's dx (no activation: its kink would turn a rounding of the normalised value into an O(dy) difference)
    against float64 autograd of GroupNorm.  dx = rstd (dxh - mean(dxh) - xh mean(dxh xh)): an error d of xh reaches dx
    times rstd max|dxh| (1 + max|xh|), so the bound is C_AFFINE 2^-24 max_g(|x scale| + |shift|) / |gamma| times that."""
    from pvraft_b200 import ops
    b, rows = 3, 4000
    worst = []
    for r in R_SWEEP:
        x, gamma, beta, st = consumer_input(dev, b, rows, c, r, seed=5 * c + r)
        dy = torch.randn(b, rows, c, generator=torch.Generator().manual_seed(r + 1)).to(dev)
        x64 = x.double().requires_grad_(True)
        mean, var = two_pass(x64)
        g = groups(x64)
        xh = ((g - mean.unsqueeze(-1)) * (var.unsqueeze(-1) + 1e-5).rsqrt())
        xh = xh.view(b, 8, rows, c // 8).transpose(1, 2).reshape(b, rows, c)
        (((xh * gamma.double() + beta.double()) * dy.double()).sum()).backward()
        want = x64.grad
        dx, _, _, _ = ops.gn_act_bwd(x, dy, st, gamma, beta, float(rows * c // 8), ops.ACT_NONE, 0.0)
        with torch.no_grad():
            rstd = (var + 1e-5).rsqrt()                                                  # [B,8]
            a_g = groups((x.double() - mean.repeat_interleave(c // 8, 1).unsqueeze(1)).abs() * rstd.repeat_interleave(c // 8, 1).unsqueeze(1)
                         + (mean * rstd).abs().repeat_interleave(c // 8, 1).unsqueeze(1)).amax(-1)
            dxh_g = groups((dy.double() * gamma.double()).abs()).amax(-1)
            xh_g = groups(xh.abs()).amax(-1)
            bound = C_AFFINE * U * a_g * rstd * dxh_g * (1 + xh_g)                       # [B,8]
            err = groups((dx.double() - want).abs()).amax(-1)
        worst.append((r, float((err / bound).max())))
    print(f'gn_act_bwd dx C={c} error / bound per r: ' + ' '.join(f'r={r}: {e:.2f}' for r, e in worst))
    assert all(e <= 1 for _, e in worst), worst


# ----------------------------------------------------------------------------------------------------------------------
# the model: a per-group shift of the biases that feed a GroupNorm changes nothing
# ----------------------------------------------------------------------------------------------------------------------
SHIFTED = {'corr_block.out_conv.0.bias': 'corr_block.out_conv.1.weight', 'corr_block.knn_conv.0.bias': 'corr_block.knn_conv.1.weight'}


def oracle_group_std(W, pc1, pc2, iters, k):
    """Per-group standard deviation of the input of each GroupNorm in SHIFTED, over the oracle's forward (float32 values,
    pooled over samples and iterations) -> {gamma name: [8] float64}."""
    gammas = {id(W[name]): name for name in SHIFTED.values()}
    acc = {}
    real = O.group_norm

    def rec(x, gamma, beta, groups=O.GN_GROUPS):
        name = gammas.get(id(gamma))
        if name is not None:
            xg = x.detach().double().reshape(x.shape[0], groups, -1).transpose(0, 1).reshape(groups, -1)
            acc.setdefault(name, []).append(xg)
        return real(x, gamma, beta, groups)

    O.group_norm = rec
    try:
        with torch.no_grad():
            O.rsf_forward(W, pc1, pc2, iters, 3, 0.25, k)
    finally:
        O.group_norm = real
    return {name: torch.cat(v, 1).std(1) for name, v in acc.items()}


def shifted_weights(W, std, r):
    W2 = dict(W)
    for bias, gamma in SHIFTED.items():
        c = W[bias].shape[0]
        W2[bias] = (W[bias].double() + group_offset(std[gamma].to(W[bias].device), r, c).to(W[bias].device)).float()
    return W2


@pytest.fixture(scope='module')
def shift_setup(dev):
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=128)
    W = default_weights(args=args, seed=3)
    out = {}
    for n in (1024, 1000):
        pc1, pc2 = O.synthetic_clouds(2, n, seed=n)
        pc1, pc2 = pc1 * 0.4, pc2 * 0.4
        Wd = {k: v.to(dev) for k, v in W.items()}
        out[n] = (pc1, pc2, oracle_group_std(Wd, pc1.to(dev), pc2.to(dev), 8, args.truncate_k))
    return args, W, out


def rsf_flows(args, W, pc1, pc2, dev, iters=8):
    """-> the flow after every iteration."""
    from pvraft_b200 import RSF
    m = RSF(args)
    m.load_state_dict(W)
    m = m.to(dev).eval()
    with torch.no_grad():
        return m([pc1.to(dev), pc2.to(dev)], num_iters=iters)


@pytest.mark.parametrize('n', [1024, 1000], ids=['tensor-core', 'cuda-core'])
def test_bias_shift_leaves_the_flow_unchanged(dev, shift_setup, n):
    """RSF free-running 8 iterations (deterministic mode, so that the shift is the only difference) with corr_block.out_conv.0 /
    knn_conv.0 biases shifted by r std_g per group against itself unshifted; error = max |flow difference| / max |flow| per
    iteration.  First iteration: <= C_ITER1 r 2^-24 for r >= 100 and linear in r.  Every iteration: <= C_SHIFT r 2^-24 +
    FLIP_TOL.  (r = 10000 goes past the issue's sweep so that two factors of 10 lie above the rounding floor.)"""
    args, W, data = shift_setup
    pc1, pc2, std = data[n]
    print(f'N={n}: group std of the shifted GroupNorm inputs ' + ', '.join(f'{k}: {float(v.mean()):.3g}' for k, v in std.items()))
    rs = (10, 100, 1000, 10000)
    with det_mode(True):
        ref = rsf_flows(args, W, pc1, pc2, dev)
        errs = {}
        for r in rs:
            got = rsf_flows(args, shifted_weights(W, std, r), pc1, pc2, dev)
            errs[r] = [float((g - f).abs().max() / f.abs().max()) for g, f in zip(got, ref)]
    for r in rs:
        print(f'bias shift N={n} r={r}: flow error per iteration / (r 2^-24): ' + ' '.join(f'{e / (r * U):.3g}' for e in errs[r]))
    for r in rs:
        assert r < 100 or errs[r][0] <= C_ITER1 * r * U, (r, errs[r][0])
        assert max(errs[r]) <= C_SHIFT * r * U + FLIP_TOL, (r, errs[r])
    assert errs[1000][0] < 30 * errs[100][0] and errs[10000][0] < 30 * errs[1000][0], {r: e[0] for r, e in errs.items()}


def test_bias_shift_leaves_the_gradients_unchanged(dev, shift_setup):
    """One stage-1 training step (one RAFT iteration, whose lookups do not depend on the statistics; N = 1024, deterministic
    mode) with the shifted biases against the unshifted one: every gradient except the shifted biases' own, relative L2
    difference over all of them <= C_SHIFT_GRAD r 2^-24.  (Per tensor max-abs is not a measure here: the backward of a max over neighbours routes a
    channel's gradient to one arg-max row, and a near-tie that a rounding flips moves it.)"""
    from pvraft_b200 import RSF
    args, W, data = shift_setup
    pc1, pc2, std = data[1024]
    gt = (pc2 - pc1).to(dev)

    def grads(Wx):
        m = RSF(args)
        m.load_state_dict(Wx)
        m = m.to(dev).train()
        flows = m([pc1.to(dev), pc2.to(dev)], num_iters=1)
        sequence_loss(flows, gt).backward()
        return {k: p.grad.detach().double() for k, p in m.named_parameters() if k not in SHIFTED}

    with det_mode(True):
        ref = grads(W)
        errs = {}
        for r in (10, 100, 1000):
            got = grads(shifted_weights(W, std, r))
            num = sum(float(((got[k] - v) ** 2).sum()) for k, v in ref.items())
            errs[r] = math.sqrt(num / sum(float((v ** 2).sum()) for v in ref.values()))
    print('bias shift gradients (relative L2): ' + ' '.join(f'r={r}: {e:.2e} ({e / (r * U):.2f} r 2^-24)' for r, e in errs.items()))
    for r, e in errs.items():
        assert e <= C_SHIFT_GRAD * r * U, (r, e)
