"""Training-path parity at the batches, point counts and weights the whole-model training tests never run with.  Every
reference is float64 (plain torch on the device or on the CPU) and independent of the library, except where a test says
it compares the library with itself (per-sample against batched runs).

  (a) the configurations of the gradient entry points that one stage-1 step at the bench training shape (B = 2,
      N = 8192, K = 512, 8 iterations) launches are recorded, and every recorded (op, width, activation, form) must be one
      of the kernel cases below: a new layer fails this until its configuration is covered
  (b) every such op at B = 3, N = 1004 (N % 8 = 4: the 8-point CTAs of k_edge_fwd, k_edge_bwd, k_lookup_bwd,
      k_lookup_xyz_bwd and k_corr_init_bwd straddle two samples; the count of such CTAs is asserted and printed) and at
      B = 8 with the bench's 8192 points (8192 * 32 edge rows) per sample, which shrinks gn_act_bwd's per-sample grid cap
      (8 * SMs + B - 1) / B; in the default form and the deterministic (DET) form, whose bits must repeat across two runs
  (c) a sample's gradients do not depend on its batch: a B = 5 / B = 3 step against the same samples one at a time
  (d) whole-model gradients with trained-looking weights (negative GroupNorm scales, PReLU slopes -0.3 and 1.7)
  (e) the bench training shape against autograd through the CPU oracle

Every uninitialised allocation is NaN-filled (integers: a huge value), so an output a kernel never writes fails its
assertion.  Inputs are scaled and offset differently per sample and errors are measured per sample (max-abs / max-abs of
that sample): state taken from the wrong sample is an O(1) error.

gn_act_maxk ranks rows on fmaf(x, sc, sh) with the folded GroupNorm scale and shift, while gn_act_bwd recomputes
t = fmaf(xh, gamma, beta).  Within an ulp of t = 0 the two may take different activation branches: that is a known
discretisation of the fused forward, not a tolerance to widen, so the gradient checks keep every t at least 1e-3 away
from 0 (the value checks do not need to).

Tolerances are those of test_gpu_kernel_coverage.py / test_gpu_train.py for the same ops at smaller shapes:
  edge_fwd 1e-6 and the GroupNorm sum bound of check_out_stats; edge_bwd 1e-5
  gn_act_bwd dx, dgamma, dbeta 5e-5; dslope within 1e-6 of sum |dy * t| over t < 0 (the sum may cancel)
  gn_act_maxk values 1e-6, arg = the first row attaining the maximum
  linear_wgrad, linear_bwd_small dW, db 5e-5, dx 1e-5
  corr_lookup_bwd, corr_lookup_xyz_bwd 1e-5;  corr_init_bwd 2e-5
  whole model: per tensor relative L2 < 2e-2, max-abs / max-abs < 5e-2, cosine of the whole gradient > 0.99999
Measured worst values are printed with -s.
"""
import math
import types

import pytest
import torch

from conftest import default_weights
from oracle import pvraft_oracle as O
from train_helpers import compare_grads, oracle_adjacency, randomise_affine, sequence_loss

pytestmark = pytest.mark.gpu

SHAPES = {'straddle': (3, 1004),     # N % 8 = 4: 8-point CTAs hold rows of two samples
          'bench': (8, 8192)}        # the bench's points per sample at B = 8
BENCH_TRAIN = dict(b=2, n=8192, k=512, iters=8)   # bench.py --mode train

# (b)'s cases: the widths one stage-1 step launches (see test_recorded_configurations_are_covered)
EDGE_C = [16, 48, 64, 96]
GN_CASES = ([('plain', c, 'lrelu') for c in (32, 64, 128)] + [('plain', 128, 'prelu'), ('plain', 64, 'none')]
            + [('arg', c, 'lrelu') for c in (16, 48, 64, 96)] + [('arg', 64, 'prelu'), ('arg', 64, 'none')])
PRELU_SLOPES = (-0.3, 0.25, 1.7)
MAXK_CASES = [(c, 'lrelu') for c in (16, 48, 64, 96)] + [(64, 'prelu'), (64, 'none')]
WGRAD_CASES = [(16, 32), (32, 32), (32, 48), (48, 64), (64, 3), (64, 64), (64, 96), (81, 128), (96, 128), (128, 61), (128, 64),
               (128, 128), (192, 64), (192, 128)]
SMALL_COUT = [16, 48, 64, 96]
LOOKUP_K = [128, 512]
CORR_INIT = [(128, 512)]


def covered():
    keys = {('edge_fwd', c, None, 'stats') for c in EDGE_C} | {('edge_bwd', c, None, None) for c in EDGE_C}
    keys |= {('gn_act_bwd', c, act, form) for form, c, act in GN_CASES}
    keys |= {('gn_act_maxk', c, act, 'arg') for c, act in MAXK_CASES}
    keys |= {('linear_wgrad', cc, None, None) for cc in WGRAD_CASES}
    keys |= {('linear_bwd_small', (cin, cout), None, dx) for cin in (3, 4) for cout in SMALL_COUT for dx in ('dx', 'no dx')}
    keys |= {('corr_lookup_bwd', (k, 3), None, None) for k in LOOKUP_K} | {('corr_lookup_xyz_bwd', k, None, None) for k in LOOKUP_K}
    keys |= {('corr_init_bwd', ck, None, None) for ck in CORR_INIT}
    return keys


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module', autouse=True)
def _cpu_threads():
    old = torch.get_num_threads()
    torch.set_num_threads(min(16, old))      # torch CPU ops collapse at 100+ threads on these op sizes
    yield
    torch.set_num_threads(old)


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


# ----------------------------------------------------------------------------------------------------------------------
# helpers
# ----------------------------------------------------------------------------------------------------------------------
def sample_scaled(g, b, *shape, offset=0.3):
    """Standard normal values; sample s is scaled by (1 + s) and shifted by offset * s."""
    x = torch.randn(b, *shape, generator=g)
    s = torch.arange(b, dtype=torch.float32).view(b, *([1] * len(shape)))
    return x * (1 + s) + offset * s


def per_sample_err(got, want):
    """max over samples of max|got_b - want_b| / max|want_b|, in float64 (NaN if anything is NaN)."""
    g = got.double().reshape(got.shape[0], -1)
    w = want.double().to(g.device).reshape(want.shape[0], -1)
    return float(((g - w).abs().amax(1) / w.abs().amax(1).clamp_min(1e-30)).max())


def check_out_stats(stats, y):
    """GroupNorm sums accumulated by a kernel, per sample and group, against float64 sums of the values y [B,R,C] they
    summarise: |error| <= 1e-5 |sum| + 1e-7 sum|y| for the first moment, 1e-5 relative for the second."""
    b, r, c = y.shape
    s = y.double().reshape(b, r, 8, c // 8)
    s1, s2, sabs = s.sum((1, 3)), (s ** 2).sum((1, 3)), s.abs().sum((1, 3))
    d1, d2 = (stats[..., 0] - s1).abs(), (stats[..., 1] - s2).abs()
    assert bool((d1 <= 1e-5 * s1.abs() + 1e-7 * sabs).all()), (stats[..., 0], s1)
    assert bool((d2 <= 1e-5 * s2).all()), (stats[..., 1], s2)
    return max(float((d1 / sabs).max()), float((d2 / s2).max()))


def ctas_spanning_samples(b, n, per_cta=8):
    """CTAs of a grid that gives each CTA `per_cta` consecutive points of B*N whose points belong to two samples."""
    total = b * n
    return sum(1 for c0 in range(0, total, per_cta) if c0 // n != (min(c0 + per_cta, total) - 1) // n)


def same_bits(a, b):
    a, b = a.detach().contiguous(), b.detach().contiguous()
    if a.is_floating_point():
        a, b = a.view(torch.int64 if a.element_size() == 8 else torch.int32), b.view(torch.int64 if b.element_size() == 8 else torch.int32)
    return torch.equal(a, b)


class det_mode:
    """torch.use_deterministic_algorithms(flag) inside the scope."""

    def __init__(self, flag):
        self.flag = flag

    def __enter__(self):
        self.was, self.warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
        torch.use_deterministic_algorithms(self.flag)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.was, warn_only=self.warn)
        return False


def run_checked(det, fn):
    """fn() -> tuple of tensors, under the deterministic flag `det`; DET: a second run must give the same bits."""
    with det_mode(det):
        out = tuple(t.clone() for t in fn())
        if det:
            again = fn()
            assert all(same_bits(x, y) for x, y in zip(out, again)), 'the deterministic form is not repeatable'
    return out


def act_code(act):
    from pvraft_b200 import ops
    return ops.ACT_NONE if act == 'none' else ops.ACT_LRELU


def gn_stats(x64):
    b, r, c = x64.shape
    xs = x64.reshape(b, r, 8, c // 8)
    return torch.stack([xs.sum((1, 3)), (xs ** 2).sum((1, 3))], -1).contiguous()


def gn_t(x64, gamma, beta):
    """GroupNorm with the statistics of x itself, float64: -> t [B,R,C]."""
    b, r, c = x64.shape
    xs = x64.reshape(b, r, 8, c // 8)
    mean = xs.mean((1, 3), keepdim=True)
    var = ((xs - mean) ** 2).mean((1, 3), keepdim=True)
    return ((xs - mean) / torch.sqrt(var + 1e-5)).reshape(b, r, c) * gamma + beta


def apply_act(t, act, slope):
    return t if act == 'none' else torch.where(t >= 0, t, slope * t)


def away_from_zero(x, gamma, beta, margin=1e-3):
    """x moved so that every t = GroupNorm(x) * gamma + beta is at least `margin` away from 0 (see the module docstring)."""
    b, r, c = x.shape
    x64 = x.double()
    near = gn_t(x64, gamma.double(), beta.double()).abs() < 2 * margin   # (moving them shifts the statistics a little)
    std = x64.reshape(b, r, 8, c // 8).std((1, 3), unbiased=False).repeat_interleave(c // 8, 1).unsqueeze(1)   # [B,1,C]
    step = 10 * margin * std / gamma.double().abs()       # moves t by about 10 * margin (|gamma| >= 0.3: the statistics barely move)
    x = torch.where(near, (x64 + step).float(), x)
    t = gn_t(x.double(), gamma.double(), beta.double())
    assert float(t.abs().min()) >= margin, float(t.abs().min())
    return x


# ----------------------------------------------------------------------------------------------------------------------
# (a) the configurations one stage-1 step at the bench training shape launches
# ----------------------------------------------------------------------------------------------------------------------
def record_key(op, a, k):
    """(op, width, activation, form) of one gradient entry-point call, and (B, rows per sample)."""
    def act_of(act, slope_dev):
        from pvraft_b200 import ops
        return 'none' if act == ops.ACT_NONE else ('prelu' if slope_dev is not None else ('lrelu' if act == ops.ACT_LRELU else f'act{act}'))

    if op == 'linear_wgrad':
        x, dy = a[0], a[1]
        return (op, (x.shape[-1], dy.shape[-1]), None, None), (x.shape[0], x.shape[1])
    if op == 'linear_bwd_small':
        x, dy = a[0], a[1]
        dx = k.get('want_dx', a[5] if len(a) > 5 else False)
        return (op, (x.shape[-1], dy.shape[-1]), None, 'dx' if dx else 'no dx'), (x.shape[0], x.shape[1])
    if op == 'gn_act_bwd':
        x = a[0]
        act = a[6]
        sdev = k.get('slope_dev', a[9] if len(a) > 9 else None)
        arg = k.get('arg', a[10] if len(a) > 10 else None)
        return (op, x.shape[-1], act_of(act, sdev), 'arg' if arg is not None else 'plain'), (x.shape[0], x.shape[1])
    if op == 'gn_act_maxk':
        x = a[0]
        sdev = k.get('slope_dev', a[7] if len(a) > 7 else None)
        return (op, x.shape[-1], act_of(a[5], sdev), 'arg'), (x.shape[0], x.shape[1])
    if op == 'edge_fwd':
        p = a[0]
        st = k.get('stats', a[3] if len(a) > 3 else None)
        return (op, p.shape[-1], None, 'stats' if st is not None else 'no stats'), (p.shape[0], p.shape[1])
    if op == 'edge_bwd':
        dp = a[2]
        return (op, dp.shape[-1], None, None), (dp.shape[0], dp.shape[1])
    if op == 'corr_lookup_bwd':
        idx = a[0]
        return (op, (idx.shape[-1], a[6]), None, None), (idx.shape[0], idx.shape[1])
    if op == 'corr_lookup_xyz_bwd':
        idx = a[0]
        return (op, idx.shape[-1], None, None), (idx.shape[0], idx.shape[1])
    if op == 'corr_init_bwd':
        g, f1 = a[0], a[2]
        return (op, (f1.shape[-1], g.shape[-1]), None, None), (f1.shape[0], f1.shape[1])
    raise KeyError(op)


RECORDED_OPS = ('linear_wgrad', 'linear_bwd_small', 'gn_act_bwd', 'gn_act_maxk', 'edge_fwd', 'edge_bwd', 'corr_lookup_bwd',
                'corr_lookup_xyz_bwd', 'corr_init_bwd')


@pytest.fixture(scope='module')
def recorded(dev):
    """One stage-1 step (forward + backward) at the bench training shape, default weights, every call of the gradient entry
    points recorded: {(op, width, activation, form): {(B, rows per sample), ...}}."""
    from pvraft_b200 import RSF, ops
    seen = {}
    with pytest.MonkeyPatch.context() as mp:
        for name in RECORDED_OPS:
            real = getattr(ops, name)

            def wrap(*a, _real=real, _name=name, **k):
                key, shape = record_key(_name, a, k)
                seen.setdefault(key, set()).add(shape)
                return _real(*a, **k)
            mp.setattr(ops, name, wrap)
        c = BENCH_TRAIN
        args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=c['k'])
        torch.manual_seed(0)
        m = RSF(args).to(dev).train()
        pc1, pc2 = [t.to(dev) for t in O.synthetic_clouds(c['b'], c['n'], seed=1234)]
        flows = m([pc1, pc2], num_iters=c['iters'])
        sequence_loss(flows, pc2 - pc1).backward()
        torch.cuda.synchronize()
    return seen


def test_recorded_configurations_are_covered(recorded):
    """Every (op, width, activation, form) that a stage-1 step at the bench training shape launches has a case in (b)."""
    for key in sorted(recorded, key=str):
        print('recorded', key, sorted(recorded[key]))
    assert {k[0] for k in recorded} >= set(RECORDED_OPS) - {'corr_lookup_xyz_bwd'}, 'an entry point was never called'
    missing = set(recorded) - covered()
    assert not missing, f'configurations without a parity case: {sorted(missing, key=str)}'


# ----------------------------------------------------------------------------------------------------------------------
# (b) kernel parity against float64
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('c', EDGE_C)
def test_edge_forward_backward(dev, c, shape, det):
    """T = P[nbr] - P + E in place with the per-sample GroupNorm sums; dP[nbr] += dT, dP -= sum_j dT."""
    from pvraft_b200 import ops
    b, n = SHAPES[shape]
    span = ctas_spanning_samples(b, n)
    assert span > 0 if shape == 'straddle' else span == 0
    g = torch.Generator().manual_seed(c * 10 + b)
    p = sample_scaled(g, b, n, c).to(dev)
    e = sample_scaled(g, b, n * 32, c, offset=-0.2).to(dev)
    nbr = torch.randint(0, n, (b, n, 32), generator=g).to(torch.int32).to(dev)
    dt = sample_scaled(g, b, n * 32, c, offset=0.1).to(dev)

    def run():
        stats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
        t = ops.edge_fwd(p, nbr, e.clone(), stats)
        dp = ops.edge_bwd(dt, nbr, torch.zeros(b, n, c, device=dev))
        return t, stats, dp
    t, stats, dp = run_checked(det, run)
    e_t = e_dp = 0.0
    for s in range(b):   # float64, one sample at a time
        ps, nb = p[s].double(), nbr[s].long()
        want = ps[nb] - ps.unsqueeze(1) + e[s].double().view(n, 32, c)
        e_t = max(e_t, per_sample_err(t[s:s + 1].view(1, n, 32, c), want[None]))
        dts = dt[s].double().view(n, 32, c)
        want_dp = -dts.sum(1)
        want_dp.index_add_(0, nb.reshape(-1), dts.reshape(-1, c))
        e_dp = max(e_dp, per_sample_err(dp[s:s + 1], want_dp[None]))
    e_st = check_out_stats(stats, t)
    print(f'edge C={c} B={b} N={n} {"DET" if det else "atomic"} ({span} CTAs span two samples): forward {e_t:.2e}, stats {e_st:.2e}, '
          f'backward {e_dp:.2e}')
    assert e_t < 1e-6 and e_dp < 1e-5, (e_t, e_dp)


def gn_case_ids():
    out = []
    for form, c, act in GN_CASES:
        for s in (PRELU_SLOPES if act == 'prelu' else (None,)):
            out.append((form, c, act, s))
    return out


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('form,c,act,slope', gn_case_ids())
def test_gn_act_bwd(dev, form, c, act, slope, shape, det):
    """dx, dgamma, dbeta (and dslope for PReLU through slope_dev) against float64 autograd of GroupNorm + activation with the
    statistics of x itself; gamma of both signs.  The arg form takes its arg from gn_act_maxk on the same x, and dy reaches
    only that row of each (point, channel)."""
    from pvraft_b200 import ops
    b, n = SHAPES[shape]
    rows = n * 32 if form == 'arg' else n
    g = torch.Generator().manual_seed(c * 7 + rows + b + len(act))
    gamma = torch.randn(c, generator=g).sign() * (0.3 + torch.rand(c, generator=g))   # both signs, |gamma| >= 0.3
    gamma, beta = gamma.to(dev), (torch.randn(c, generator=g) * 0.2).to(dev)
    assert bool((gamma < 0).any()) and bool((gamma > 0).any())
    x = away_from_zero(sample_scaled(g, b, rows, c).to(dev), gamma, beta)
    stats, count = gn_stats(x.double()), float(rows * (c // 8))
    sl = 0.1 if act != 'prelu' else slope
    sdev = torch.tensor([slope], dtype=torch.float32, device=dev) if act == 'prelu' else None
    code = act_code(act)
    am = None
    if form == 'arg':
        _, am = ops.gn_act_maxk(x, stats, gamma, beta, count, code, 0.1, slope_dev=sdev)
        dy = sample_scaled(g, b, n, c, offset=0.2).to(dev)
    else:
        dy = sample_scaled(g, b, rows, c, offset=0.2).to(dev)
    cap = (8 * torch.cuda.get_device_properties(dev).multi_processor_count + b - 1) // b

    def run():
        dx, dg, dbt, ds = ops.gn_act_bwd(x, dy, stats, gamma, beta, count, code, 0.1, want_dslope=act == 'prelu', slope_dev=sdev, arg=am)
        return (dx, dg, dbt) + ((ds,) if ds is not None else ())
    out = run_checked(det, run)
    if form == 'arg':
        dyd = torch.zeros(b, n, 32, c, dtype=torch.float64, device=dev)
        dyd.scatter_(2, am.long().unsqueeze(2), dy.double().unsqueeze(2))
        dyd = dyd.reshape(b, rows, c)
    else:
        dyd = dy.double()
    xr = x.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    sr = torch.tensor(sl, dtype=torch.float64, device=dev, requires_grad=True)
    t = gn_t(xr, gr, br)
    (apply_act(t, act, sr) * dyd).sum().backward()
    e_dx = per_sample_err(out[0], xr.grad)
    e_g = per_sample_err(out[1][None], gr.grad[None])
    e_b = per_sample_err(out[2][None], br.grad[None])
    msg = f'gn_act_bwd {form} C={c} {act}{"" if slope is None else f" slope={slope}"} B={b} rows={rows} (grid cap {cap} CTAs per sample) ' \
          f'{"DET" if det else "atomic"}: dx {e_dx:.2e}, dgamma {e_g:.2e}, dbeta {e_b:.2e}'
    if act == 'prelu':
        td = t.detach()
        scale = float((dyd * td).abs()[td < 0].sum())    # 0 when no maximum with gradient lies below 0: then dslope must be 0
        e_s = abs(float(out[3]) - float(sr.grad)) / scale if scale > 0 else abs(float(out[3]))
        msg += f', dslope {e_s:.2e} of sum|dy t|'
        assert e_s <= 1e-6 if scale > 0 else e_s == 0.0, (float(out[3]), float(sr.grad), scale)
    print(msg)
    assert e_dx < 5e-5 and e_g < 5e-5 and e_b < 5e-5, (e_dx, e_g, e_b)
    del xr, t


@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('c,act,slope', [(c, act, s) for c, act in MAXK_CASES for s in (PRELU_SLOPES if act == 'prelu' else (None,))])
def test_gn_act_maxk(dev, c, act, slope, shape):
    """max over each point's 32 rows of act(GroupNorm(x)) within 1e-6 of float64; arg = the first row attaining the maximum.
    Rows 9 and 20 of every point are exact copies of row 5, pushed to an extreme for every other channel, so exact ties
    decide many maxima: the arg must then be 5."""
    from pvraft_b200 import ops
    b, n = SHAPES[shape]
    g = torch.Generator().manual_seed(c + n + b)
    x = sample_scaled(g, b, n, 32, c)
    hi = torch.arange(c) % 2 == 0
    top = torch.where(hi, x.amax(2) + 1.0, x.amin(2) - 1.0)
    for j in (5, 9, 20):
        x[:, :, j] = top
    x = x.reshape(b, n * 32, c).to(dev)
    gamma, beta = torch.randn(c, generator=g).to(dev), (torch.randn(c, generator=g) * 0.2).to(dev)
    stats, count = gn_stats(x.double()), float(n * 32 * (c // 8))
    sl = 0.1 if act != 'prelu' else slope
    sdev = torch.tensor([slope], dtype=torch.float32, device=dev) if act == 'prelu' else None
    y, arg = ops.gn_act_maxk(x, stats, gamma, beta, count, act_code(act), 0.1, slope_dev=sdev)
    t = apply_act(gn_t(x.double(), gamma.double(), beta.double()), act, sl).view(b, n, 32, c)
    want = t.amax(2)
    err = per_sample_err(y, want)
    a = arg.long()
    assert bool((a < 32).all())
    at = torch.gather(t, 2, a.unsqueeze(2)).squeeze(2)
    scale = want.abs().reshape(b, -1).amax(1).view(b, 1, 1)
    assert bool(((want - at) <= 1e-6 * scale).all()), 'arg does not attain the maximum'
    xv = x.view(b, n, 32, c)
    xa = torch.gather(xv, 2, a.unsqueeze(2))
    rowid = torch.arange(32, device=dev).view(1, 1, 32, 1)
    earlier = rowid < a.unsqueeze(2)
    assert not bool((earlier & (xv == xa)).any()), 'an earlier row with the same value attains the maximum'
    assert not bool((earlier & (t > at.unsqueeze(2) + 1e-6 * scale.unsqueeze(-1))).any()), 'an earlier row is larger'
    ties = int((a == 5).sum())
    assert ties > 0 and not bool(((a == 9) | (a == 20)).any())
    print(f'gn_act_maxk C={c} {act}{"" if slope is None else f" slope={slope}"} B={b} N={n}: values {err:.2e}, '
          f'{ties} maxima decided by an exact tie')
    assert err < 1e-6, err


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('cin,cout', WGRAD_CASES)
def test_linear_wgrad(dev, cin, cout, shape, det):
    """dW += dy^T x, db += column sums over every row, into a destination with a row stride of cin + 5 whose padding stays
    untouched."""
    from pvraft_b200 import ops
    b, n = SHAPES[shape]
    g = torch.Generator().manual_seed(cin * 131 + cout + b)
    x, dy = sample_scaled(g, b, n, cin).to(dev), sample_scaled(g, b, n, cout, offset=-0.2).to(dev)
    ld = cin + 5

    def run():
        dw = torch.full((cout, ld), 7.0, device=dev)
        dw[:, :cin] = 0
        db = torch.zeros(cout, device=dev)
        ops.linear_wgrad(x, dy, dw, db)
        return dw, db
    dw, db = run_checked(det, run)
    xd, dyd = x.double().reshape(-1, cin), dy.double().reshape(-1, cout)
    e_w = per_sample_err(dw[None, :, :cin], (dyd.t() @ xd)[None])
    e_b = per_sample_err(db[None], dyd.sum(0)[None])
    print(f'linear_wgrad {cin}->{cout} B={b} rows={n} {"DET" if det else "atomic"}: dW {e_w:.2e}, db {e_b:.2e}')
    assert bool((dw[:, cin:] == 7.0).all()), 'the padding of the strided destination was written'
    assert e_w < 5e-5 and e_b < 5e-5, (e_w, e_b)


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('want_dx', [False, True])
@pytest.mark.parametrize('cout', SMALL_COUT)
@pytest.mark.parametrize('cin', [3, 4])
def test_linear_bwd_small(dev, cin, cout, want_dx, shape, det):
    """Edge-level rows (32 per point): dW += dy^T x, db += column sums and dx = dy W in one pass."""
    from pvraft_b200 import ops
    b, n = SHAPES[shape]
    r = n * 32
    g = torch.Generator().manual_seed(cin * 17 + cout + b + want_dx)
    x, dy = sample_scaled(g, b, r, cin).to(dev), sample_scaled(g, b, r, cout, offset=-0.2).to(dev)
    w = torch.randn(cout, cin, generator=g).to(dev)

    def run():
        dw, db = torch.zeros(cout, cin, device=dev), torch.zeros(cout, device=dev)
        dx = ops.linear_bwd_small(x, dy, w, dw, db, want_dx=want_dx)
        return (dw, db) + ((dx,) if want_dx else ())
    out = run_checked(det, run)
    xd, dyd = x.double().reshape(-1, cin), dy.double().reshape(-1, cout)
    e_w = per_sample_err(out[0][None], (dyd.t() @ xd)[None])
    e_b = per_sample_err(out[1][None], dyd.sum(0)[None])
    e_x = per_sample_err(out[2], (dy.double() @ w.double())) if want_dx else 0.0
    print(f'linear_bwd_small {cin}->{cout} B={b} rows={r} dx={want_dx} {"DET" if det else "atomic"}: dW {e_w:.2e}, db {e_b:.2e}, dx {e_x:.2e}')
    assert e_w < 5e-5 and e_b < 5e-5 and e_x < 1e-5, (e_w, e_b, e_x)


def lookup_case(dev, b, n, m, k, seed, box=3.0):
    """A state of k distinct candidate rows of xyz2 [B,M,3] per query point, correlations sorted descending, queries next to
    random xyz2 points; installed in a CorrBlock (stored order)."""
    g = torch.Generator().manual_seed(seed)
    xyz2 = (box * torch.rand(b, m, 3, generator=g) + torch.arange(b).view(b, 1, 1) * 5.0).to(dev)   # per-sample offsets
    gd = torch.Generator(device=dev).manual_seed(seed)
    idx = torch.rand(b, n, m, generator=gd, device=dev).topk(k, dim=2).indices
    pick = torch.randint(0, m, (b, n), generator=g).to(dev)
    coords = torch.gather(xyz2, 1, pick.unsqueeze(-1).expand(b, n, 3)) + ((torch.rand(b, n, 3, generator=g) * 2 - 1) * 0.2).to(dev)
    corr = torch.sort(sample_scaled(g, b, n, k) * 5 + 20, dim=2, descending=True).values.to(dev)
    return corr, idx, coords.contiguous(), xyz2.contiguous()


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('scale', [0.25, 0.3])
@pytest.mark.parametrize('k', LOOKUP_K)
@pytest.mark.parametrize('shape', list(SHAPES))
def test_corr_lookup_backward(dev, shape, k, scale, det):
    """d corr and d xyz2 of (voxel means, kNN 4-vectors) against float64 autograd through O.voxel_cube_index's cells and the
    gathers of O.knn_gather, on the kernel's own slots; 3 levels; N1 != N2 at B = 3."""
    from pvraft_b200 import CorrBlock, ops
    b, n = SHAPES[shape]
    m = n + 496 if shape == 'straddle' else n
    levels = 3
    span = ctas_spanning_samples(b, n)
    corr, idx, coords, xyz2 = lookup_case(dev, b, n, m, k, seed=n + k + int(scale * 100))
    cb = CorrBlock(num_levels=levels, base_scale=scale, truncate_k=k).to(dev)
    cb.set_state(corr, idx.to(torch.int32), xyz2)
    out = ops.corr_lookup(cb.corr_val, cb.corr_idx, cb._xyz2p, coords, levels, scale, want_slots=True, vox_ld=levels * 27)
    slots = out['knn_slot']
    g = torch.Generator().manual_seed(k)
    g_vox = sample_scaled(g, b, n, levels * 27).to(dev)
    g_sel = sample_scaled(g, b, n * 32, 4, offset=-0.1).to(dev)

    def run():
        d_corr = ops.corr_lookup_bwd(cb.corr_idx, cb._xyz2p, coords, slots, g_vox, g_sel, levels, scale)
        d_xyz2 = ops.corr_lookup_xyz_bwd(cb.corr_idx, slots, g_sel, torch.zeros(b, m, 3, device=dev))
        return d_corr, d_xyz2
    d_corr, d_xyz2 = run_checked(det, run)
    # float64 reference (cells and the kNN choice are discrete: taken in fp32 as the reference computes them)
    ids = cb.corr_idx.long()
    cand32 = torch.gather(xyz2.unsqueeze(1).expand(b, n, m, 3), 2, ids.unsqueeze(-1).expand(b, n, k, 3))
    st32 = O.CorrState(cb.corr_val, ids, cand32)
    cv = cb.corr_val.double().requires_grad_(True)
    x2 = xyz2.double().requires_grad_(True)
    loss = 0
    for lvl in range(levels):
        cube, valid = O.voxel_cube_index(st32, coords, scale * 2 ** lvl)
        w = valid.double()
        s = torch.zeros(b, n, 27, dtype=torch.float64, device=dev).scatter_add(2, cube, cv * w)
        cnt = torch.zeros(b, n, 27, dtype=torch.float64, device=dev).scatter_add(2, cube, w)
        loss = loss + (s / cnt.clamp(1, n) * g_vox[..., lvl * 27:(lvl + 1) * 27].double()).sum()
    sl = slots.long()
    cand64 = torch.gather(x2.unsqueeze(1).expand(b, n, m, 3), 2, ids.unsqueeze(-1).expand(b, n, k, 3))
    sel_c = torch.gather(cv, 2, sl)
    sel_x = torch.gather(cand64, 2, sl.unsqueeze(-1).expand(b, n, 32, 3)) - coords.double().unsqueeze(2)
    gs = g_sel.double().view(b, n, 32, 4)
    loss = loss + (sel_c * gs[..., 0]).sum() + (sel_x * gs[..., 1:]).sum()
    loss.backward()
    e_c, e_x = per_sample_err(d_corr, cv.grad), per_sample_err(d_xyz2, x2.grad)
    print(f'corr_lookup backward B={b} N1={n} N2={m} K={k} scale={scale} {"DET" if det else "atomic"} ({span} CTAs span two samples): '
          f'd corr {e_c:.2e}, d xyz2 {e_x:.2e}')
    assert e_c < 1e-5 and e_x < 1e-5, (e_c, e_x)


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('c,k', CORR_INIT)
def test_corr_init_backward(dev, c, k, shape, det):
    """d fmap1 = G fmap2 / sqrt(C), d fmap2 = G^T fmap1 / sqrt(C) with G the dense float64 [N,M] gradient of the kept entries."""
    from pvraft_b200 import ops
    b, n = SHAPES[shape]
    m = n + 496 if shape == 'straddle' else n
    span = ctas_spanning_samples(b, n)
    g = torch.Generator().manual_seed(c + k + b)
    f1, f2 = sample_scaled(g, b, n, c).to(dev), sample_scaled(g, b, m, c, offset=-0.2).to(dev)
    gd = torch.Generator(device=dev).manual_seed(k)
    idx = torch.rand(b, n, m, generator=gd, device=dev).topk(k, dim=2).indices
    gv = sample_scaled(g, b, n, k).to(dev)

    def run():
        return ops.corr_init_bwd(gv, idx.to(torch.int32), f1, f2)
    d1, d2 = run_checked(det, run)
    G = torch.zeros(b, n, m, dtype=torch.float64, device=dev).scatter_(2, idx, gv.double())
    e1 = per_sample_err(d1, G @ f2.double() / math.sqrt(c))
    e2 = per_sample_err(d2, G.transpose(1, 2) @ f1.double() / math.sqrt(c))
    print(f'corr_init_bwd C={c} K={k} B={b} N={n} M={m} {"DET" if det else "atomic"} ({span} CTAs span two samples): '
          f'd fmap1 {e1:.2e}, d fmap2 {e2:.2e}')
    assert e1 < 2e-5 and e2 < 2e-5, (e1, e2)


# ----------------------------------------------------------------------------------------------------------------------
# (c) a sample's gradients do not depend on its batch
# ----------------------------------------------------------------------------------------------------------------------
def per_sample_clouds(b, n, seed):
    pc1, pc2 = O.synthetic_clouds(b, n, seed=seed)
    s = torch.arange(b, dtype=torch.float32).view(b, 1, 1)
    scale, shift = 0.4 * (1 + 0.1 * s), 3.0 * s
    return pc1 * scale + shift, pc2 * scale + shift


def step_grads(m, pc1, pc2, iters):
    """One stage-1 step with the sum over samples of each sample's sequence loss -> (flows, param grads, xyz1 / xyz2 grads)."""
    m.zero_grad(set_to_none=True)
    x1, x2 = pc1.clone().requires_grad_(True), pc2.clone().requires_grad_(True)
    flows = m([x1, x2], num_iters=iters)
    gt = pc2 - pc1
    loss = sum(sequence_loss([f[s:s + 1] for f in flows], gt[s:s + 1]) for s in range(pc1.shape[0]))
    loss.backward()
    return [f.detach() for f in flows], {k: p.grad.detach().clone() for k, p in m.named_parameters()}, x1.grad, x2.grad


@pytest.mark.parametrize('path', ['cuda_core', 'tensor_core'])
def test_sample_gradients_do_not_depend_on_the_batch(dev, path):
    """B = 5, N = 1004 (CUDA-core layers) and B = 3, N = 1024 with the tensor-core layers forced: the parameter gradients equal
    the sum of the single-sample steps' gradients and each sample's input gradients equal its own single-sample step's, up
    to summation order (the kNN graph, the top-K and the lookup are per sample, so every discrete choice is the same).
    Under deterministic algorithms each sample's flows are the bits of its single-sample run."""
    from pvraft_b200 import RSF, train as T
    b, n = (5, 1004) if path == 'cuda_core' else (3, 1024)
    k, iters = 128, 3
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    m = RSF(args)
    m.load_state_dict(default_weights(args=args, seed=3))
    randomise_affine(m, 5, (-0.3, 1.7))
    m = m.to(dev).train()
    pc1, pc2 = [t.to(dev) for t in per_sample_clouds(b, n, seed=n + b)]
    was = T._TC_TRAIN
    T._TC_TRAIN = '1' if path == 'tensor_core' else '0'
    try:
        _, gb, x1b, x2b = step_grads(m, pc1, pc2, iters)
        singles = [step_grads(m, pc1[s:s + 1], pc2[s:s + 1], iters) for s in range(b)]
        with det_mode(True):
            fb = step_grads(m, pc1, pc2, iters)[0]
            fs = [step_grads(m, pc1[s:s + 1], pc2[s:s + 1], iters)[0] for s in range(b)]
    finally:
        T._TC_TRAIN = was
    pairs = [(kk, gb[kk], sum(sg[1][kk] for sg in singles)) for kk in gb]
    pairs += [(f'xyz1[{s}]', x1b[s], singles[s][2][0]) for s in range(b)] + [(f'xyz2[{s}]', x2b[s], singles[s][3][0]) for s in range(b)]
    worst_l2, worst_cos = ('', 0.0), ('', 1.0)
    for name, a, w in pairs:
        a, w = a.double(), w.double()
        l2 = float((a - w).norm() / w.norm().clamp_min(1e-30))
        cos = float((a * w).sum() / (a.norm() * w.norm()).clamp_min(1e-300))
        worst_l2 = (name, l2) if l2 > worst_l2[1] else worst_l2
        worst_cos = (name, cos) if cos < worst_cos[1] else worst_cos
    print(f'batch independence {path} B={b} N={n}: worst relative L2 {worst_l2[0]} {worst_l2[1]:.2e}, '
          f'worst cosine {worst_cos[0]} {worst_cos[1]:.10f}')
    assert worst_l2[1] < 5e-5, worst_l2           # measured 4.5e-6 (B = 5) and 2.7e-6 (B = 3)
    assert worst_cos[1] > 1 - 1e-9, worst_cos    # measured 1 - 1e-11 or closer
    differ = [(s, i) for s in range(b) for i in range(iters) if not same_bits(fb[i][s], fs[s][i][0])]
    assert not differ, f'deterministic flows differ from the single-sample run at (sample, iteration) {differ}'


# ----------------------------------------------------------------------------------------------------------------------
# (d) whole-model gradients with trained-looking weights
# ----------------------------------------------------------------------------------------------------------------------
def oracle_step(W, pc1, pc2, iters, k):
    Wr = {kk: v.clone().requires_grad_(True) for kk, v in W.items()}
    x1r, x2r = pc1.clone().requires_grad_(True), pc2.clone().requires_grad_(True)
    flows = O.rsf_forward(Wr, x1r, x2r, iters, 3, 0.25, k)
    loss = sequence_loss(flows, pc2 - pc1)
    loss.backward()
    return [f.detach() for f in flows], float(loss), dict({kk: v.grad for kk, v in Wr.items()}, xyz1=x1r.grad, xyz2=x2r.grad)


def model_step(m, pc1, pc2, iters, dev):
    m.zero_grad(set_to_none=True)
    x1, x2 = pc1.to(dev).requires_grad_(True), pc2.to(dev).requires_grad_(True)
    with oracle_adjacency():
        flows = m([x1, x2], num_iters=iters)
    loss = sequence_loss(flows, (pc2 - pc1).to(dev))
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters()}
    assert len(got) == 95 and all(v is not None for v in got.values())
    return [f.detach().cpu() for f in flows], float(loss), dict(got, xyz1=x1.grad, xyz2=x2.grad)


def flows_close(flows, flows_ref):
    worst = 0.0
    for f, fr in zip(flows, flows_ref):
        e = float((f - fr).abs().mean() / fr.abs().mean())
        worst = max(worst, e)
    return worst


@pytest.mark.parametrize('slopes', [(-0.3, 1.7), (1.7, -0.3)])
@pytest.mark.parametrize('path', ['cuda_core', 'tensor_core'])
def test_trained_weight_gradients_match_oracle(dev, path, slopes):
    """A 3-iteration stage-1 step, B = 3, K = 128, GroupNorm affines drawn at random (negative scales) and PReLU slopes
    (out_conv, knn_conv) = `slopes`: all 95 parameter gradients and both input gradients against autograd through the
    oracle, on the oracle's kNN graph.  N = 1004 runs the CUDA-core layers, N = 1024 the tensor-core layers (forced)."""
    from pvraft_b200 import RSF, train as T
    b, k, iters = 3, 128, 3
    n = 1004 if path == 'cuda_core' else 1024
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    m = RSF(args)
    m.load_state_dict(default_weights(args=args, seed=2))
    randomise_affine(m, 7, slopes)
    W = {kk: v.detach().clone() for kk, v in m.state_dict().items()}
    assert any(bool((W[kk] < 0).any()) for kk in W if '.gn' in kk and kk.endswith('weight'))
    m = m.to(dev).train()
    pc1, pc2 = per_sample_clouds(b, n, seed=n + 7)
    flows_ref, loss_ref, want = oracle_step(W, pc1, pc2, iters, k)
    was = T._TC_TRAIN
    T._TC_TRAIN = '1' if path == 'tensor_core' else '0'
    try:
        flows, loss, got = model_step(m, pc1, pc2, iters, dev)
    finally:
        T._TC_TRAIN = was
    e_f = flows_close(flows, flows_ref)
    e_l = abs(loss - loss_ref) / abs(loss_ref)
    print(f'trained weights {path} N={n} slopes={slopes}: flows {e_f:.2e} (mean abs / mean abs), loss {e_l:.2e}')
    assert e_f < 1e-4 and e_l < 1e-4, (e_f, e_l)
    compare_grads(got, want, 2e-2, 5e-2)


# ----------------------------------------------------------------------------------------------------------------------
# (e) the bench training shape against the oracle
# ----------------------------------------------------------------------------------------------------------------------
def available_host_bytes():
    try:
        with open('/proc/meminfo') as f:
            for line in f:
                if line.startswith('MemAvailable:'):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def test_bench_training_shape_matches_oracle(dev):
    """One stage-1 step at the shape bench.py --mode train times (B = 2, N = 8192, K = 512, 8 iterations, default weights):
    loss, flows and the 95 parameter gradients against autograd through the CPU oracle on the oracle's kNN graph.  The
    oracle's forward and backward need about 19 GB of host memory at this shape."""
    from pvraft_b200 import RSF
    free = available_host_bytes()
    if free < 24 * 2 ** 30:
        pytest.skip(f'the CPU oracle at the bench training shape needs about 24 GB of free host memory, {free / 2 ** 30:.1f} GB available')
    c = BENCH_TRAIN
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=c['k'])
    W = default_weights(args=args, seed=0)
    pc1, pc2 = O.synthetic_clouds(c['b'], c['n'], seed=1234)
    Wr = {kk: v.clone().requires_grad_(True) for kk, v in W.items()}
    flows_ref = O.rsf_forward(Wr, pc1, pc2, c['iters'], 3, 0.25, c['k'])
    loss_ref = sequence_loss(flows_ref, pc2 - pc1)
    loss_ref.backward()
    want = {kk: v.grad for kk, v in Wr.items()}
    flows_ref = [f.detach() for f in flows_ref]
    del Wr
    m = RSF(args)
    m.load_state_dict(W)
    m = m.to(dev).train()
    with oracle_adjacency():
        flows = m([pc1.to(dev), pc2.to(dev)], num_iters=c['iters'])
    loss = sequence_loss(flows, (pc2 - pc1).to(dev))
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters()}
    assert len(got) == 95 and all(v is not None for v in got.values())
    e_f = flows_close([f.detach().cpu() for f in flows], flows_ref)
    e_l = abs(float(loss) - float(loss_ref)) / abs(float(loss_ref))
    print(f'bench training shape: flows {e_f:.2e} (mean abs / mean abs), loss {e_l:.2e}')
    assert e_f < 1e-4 and e_l < 1e-4, (e_f, e_l)
    compare_grads(got, want, 2e-2, 5e-2)
