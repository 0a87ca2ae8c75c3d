"""Parity of the fp32 CUDA-core forward kernels of csrc/pointmlp.cu against float64, at the shapes where a persistent CTA
carries tiles of several samples: k_linear, k_gn_act, k_transpose, k_corrfeat, k_gru and k_flowout, behind ops.linear,
ops.gn_act, ops.transpose, ops.corr_feature, ops.gru and ops.flow_out.  These kernels carry every forward at N % 128 != 0,
the encoders' first layers (SetConv(3, 32).fc1 / fc2) and the refine head at every N, and the training forward and its
dx = dy W products at shapes the tensor-core rule rejects.  Every reference is float64 plain torch on the device.

  (a) the configurations the product launches are recorded (eager forwards of RSF / RSF_refine at N = 1000 and 1024, one
      iteration at the bench shape B = 8, N = 8192, a stage-1 and a refine training step, every reference-layout module
      seam), and every recorded key must be one of the cases below: a new configuration fails until it has a case
  (b) every entry point at three shapes: `single` (1, 37), one partial tile; `tail` (3, 1004), whose last tile per sample
      holds 44 points; `multi` (8, 7999), 125 tiles per sample, where at occupancies 1 to 4 on the H100's 132 SMs some CTAs
      run tiles of two samples (the count is asserted and printed).  That is the code that carries state from one tile
      to the next: the per-sample GroupNorm affine reload (k_linear, k_corrfeat, k_flowout), k_linear's flush of its
      output sums at a sample change (default and DET form) and k_gru's register prefetch of the next tile
  (c) batch invariance, bitwise: each kernel over the `multi` batch against the same kernel once per sample, with the same
      statistics and moments as inputs (a point's arithmetic does not depend on the CTA that runs its tile, so any
      difference is state carried across a sample boundary); k_linear's DET output sums too, per sample
  (d) RSF at B = 3, N = 4999 (79 tiles per sample), K = 512, trained-looking weights, against the oracle on the oracle's
      adjacency: module seams teacher-forced per iteration, and free-running

Every uninitialised allocation is NaN-filled (integers: a huge value), so an output a kernel never writes fails.  Inputs
are scaled and offset differently per sample and errors are measured per sample (max-abs / max-abs of that sample):
state taken from the wrong sample is an O(1) error.

Bounds (per-sample max-abs / max-abs), those of the existing tests of the same ops; measured worst values on an H100
80GB HBM3 (700 W) in brackets, printed with -s:
  linear 2e-6 * max(1, cin / 128) [7.6e-7 of that scale];  output GroupNorm sums: 1e-5 relative + 1e-7 of the
  group's sum of |y| (check_out_stats) [1.3e-15 of the sum of |y|, or of the second moment]
  gn_act 1e-6 [1.7e-7];  transpose bitwise
  corr feature 1e-5 [4.9e-7];  motion 2e-5 [5.0e-7], channels 61-63 = the flow, bitwise
  gru 1e-5 [5.8e-7];  flow_out delta 5e-5 [3.9e-7], coords2_out = coords2 + delta and flow_out = coords2_out - coords1
  bitwise
  model level: teacher-forced corr 1e-5 [1.3e-6], net 1e-5 [2.3e-7], delta 5e-5 [7.9e-7]; free-running mean-abs 1e-4
  of mean |flow| [9.8e-6]
"""
import inspect
import types

import pytest
import torch

from conftest import default_weights
from oracle import pvraft_oracle as O
from train_helpers import oracle_adjacency, randomise_affine, sequence_loss

pytestmark = pytest.mark.gpu

SHAPES = {'single': (1, 37),       # one partial tile
          'tail': (3, 1004),       # 16 tiles per sample, the last holds 44 points
          'multi': (8, 7999)}      # 125 tiles per sample: CTAs straddle samples at every occupancy 1..4
TP = 64                            # points per tile of the CUDA-core kernels (csrc/tile_gemm.cuh kTP)

PLAIN, GN, MINMAX = 0, 1, 2        # pvraft_linear_args.in_mode (include/pvraft_b200.h)
NONE, RELU, LRELU = 0, 1, 2        # activation codes

WORST = {}


def note(check, err):
    WORST[check] = max(WORST.get(check, 0.0), err)
    return err


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def sm_count():
    from pvraft_b200 import ops
    return ops.device_info()[0]


@pytest.fixture(scope='module', autouse=True)
def _cpu_threads():
    old = torch.get_num_threads()
    torch.set_num_threads(min(16, old))      # torch CPU ops collapse at 100+ threads on these op sizes
    yield
    torch.set_num_threads(old)


@pytest.fixture(scope='module', autouse=True)
def _print_worst():
    yield
    print('\nworst per-sample errors:', {k: f'{v:.2e}' for k, v in sorted(WORST.items())})


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


def gn_stats(x64):
    """[B,N,C] -> the [B,8,2] (sum, sum of squares) GroupNorm sums the library passes between layers."""
    b, n, c = x64.shape
    xs = x64.reshape(b, n, 8, c // 8)
    return torch.stack([xs.sum((1, 3)), (xs ** 2).sum((1, 3))], -1).contiguous()


def gn_act_ref(x64, xmin64, stats, gamma, beta, count, slope):
    """act(GroupNorm(x)) from the sums (slope 1: no activation); with xmin64 the input is the min array where the
    GroupNorm scale is < 0."""
    c = x64.shape[-1]
    mean = stats[..., 0] / count
    rstd = (stats[..., 1] / count - mean ** 2 + 1e-5).rsqrt()
    sc = rstd.repeat_interleave(c // 8, 1).unsqueeze(1) * gamma.double()
    sh = beta.double() - mean.repeat_interleave(c // 8, 1).unsqueeze(1) * sc
    raw = x64 if xmin64 is None else torch.where(sc < 0, xmin64, x64)
    t = raw * sc + sh
    return torch.where(t >= 0, t, slope * t)


def gn_self(t64):
    """GroupNorm(8) of t [..., R, C] with the statistics of t itself over R (no affine), float64."""
    r, c = t64.shape[-2:]
    tg = t64.reshape(-1, r, 8, c // 8)
    mean = tg.mean((1, 3), keepdim=True)
    var = tg.var((1, 3), unbiased=False, keepdim=True)
    return ((tg - mean) * (var + 1e-5).rsqrt()).reshape(t64.shape)


def prelu(t, slope):
    return torch.where(t >= 0, t, slope * t)


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


def both_signs(g, c):
    """A GroupNorm gamma with both signs and |gamma| >= 0.3 (a scale's sign never depends on rounding)."""
    gamma = torch.randn(c, generator=g).sign() * (0.3 + torch.rand(c, generator=g))
    gamma[0], gamma[-1] = -abs(float(gamma[0])), abs(float(gamma[-1]))
    return gamma


def straddling_ctas(b, n, sm, occ):
    """CTAs of a CUDA-core kernel launched at `occ` CTAs per SM that run tiles of two samples: tile_grid launches
    min(tiles, SMs * occ) CTAs and split_range gives each ceil(tiles / grid) consecutive tiles (csrc/pointmlp.cu)."""
    tps = -(-n // TP)
    total = b * tps
    grid = min(total, sm * occ)
    per = -(-total // grid)
    count = 0
    for w in range(grid):
        t0, t1 = min(per * w, total), min(per * w + per, total)
        if t0 < t1 and t0 // tps != (t1 - 1) // tps:
            count += 1
    return count


def test_multi_shape_straddles_samples(sm_count):
    """At `multi` some CTAs run tiles of two samples at every occupancy the kernels can have (1-4); at `single` and `tail`
    (fewer tiles than SMs) none does."""
    for name, (b, n) in SHAPES.items():
        counts = [straddling_ctas(b, n, sm_count, occ) for occ in (1, 2, 3, 4)]
        print(f'{name} B={b} N={n} ({-(-n // TP)} tiles per sample, {sm_count} SMs): CTAs holding tiles of two samples at '
              f'occupancy 1-4: {counts}')
        if name == 'multi':
            assert all(c > 0 for c in counts), counts
        else:
            assert all(c == 0 for c in counts), counts


# ----------------------------------------------------------------------------------------------------------------------
# (b) cases: every configuration the product launches, plus the regimes where the kernels branch
# ----------------------------------------------------------------------------------------------------------------------
def L(cin, cout, mode=PLAIN, act=NONE, out=NONE, res=False, stats=False, bias=False, w=None, slope=None):
    """A k_linear case: (recorded key, input slope, weight form).  w: None (a [cout, cin] weight), 'w_ld' (rows of cin + 3
    of which the first cin are used: SetConv.fc1) or 'w_cin' (cin - 3 weight columns; the input's last 3 are ignored:
    out_conv[0] on the padded voxel rows)."""
    key = (cin, cout, mode, act, out, res, stats, bias, w is not None)
    return key, (None if act != LRELU else (0.1 if slope is None else slope)), w


LINEAR_CASES = [
    # inference: the SetConv layers at N % 128 != 0 and the first layers at every N (encoders, flow head, refiner)
    L(3, 16, w='w_ld'), L(32, 48, w='w_ld'), L(64, 96, w='w_ld'), L(64, 64, w='w_ld'),
    L(32, 48, GN, LRELU, w='w_ld'), L(64, 96, GN, LRELU, w='w_ld'),
    L(16, 32, MINMAX, LRELU, stats=True), L(48, 64, MINMAX, LRELU, stats=True), L(96, 128, MINMAX, LRELU, stats=True),
    L(64, 64, MINMAX, LRELU, stats=True),
    L(32, 32, GN, LRELU, stats=True), L(64, 64, GN, LRELU, stats=True), L(128, 128, GN, LRELU, stats=True),
    # correlation feature head (out_conv[0] on the voxel rows, CorrBlock.get_voxel_feature's out_conv[3]), refine head
    L(84, 128, stats=True, bias=True, w='w_cin'), L(128, 64, bias=True), L(128, 3, GN, LRELU, res=True, bias=True),
    # training forward (LinearFn) at shapes the tensor-core rule rejects
    L(3, 16), L(3, 48), L(3, 96), L(3, 64), L(32, 48), L(64, 96), L(64, 64),
    L(16, 32, stats=True), L(48, 64, stats=True), L(96, 128, stats=True), L(64, 64, stats=True), L(32, 32, stats=True),
    L(128, 128, stats=True), L(81, 128, stats=True, bias=True), L(4, 64, stats=True, bias=True),
    L(128, 64, bias=True), L(64, 64, bias=True), L(3, 64, bias=True), L(128, 61, bias=True), L(192, 128, bias=True),
    L(192, 64, bias=True), L(64, 3, bias=True), L(128, 3, bias=True),
    # training backward: dx = dy W, 128 output columns at a time
    L(32, 16), L(64, 48), L(128, 96), L(48, 32), L(96, 64), L(128, 81), L(64, 128), L(61, 128), L(128, 64), L(3, 128),
    L(32, 32), L(128, 128),
    # regimes: cin 61 / 256, cout 65, no input activation, slopes -0.3 and 1.7, ReLU output, residual with tail stores
    L(61, 64, bias=True), L(61, 32, out=RELU, bias=True), L(256, 128, GN, LRELU, stats=True, bias=True), L(256, 64, GN, NONE),
    L(64, 65, GN, LRELU, res=True, bias=True), L(81, 65, res=True), L(64, 64, GN, NONE, stats=True),
    L(128, 128, GN, LRELU, stats=True, slope=-0.3), L(128, 128, GN, LRELU, stats=True, slope=1.7),
    L(16, 32, MINMAX, LRELU, stats=True, slope=-0.3), L(96, 128, MINMAX, LRELU, stats=True, slope=1.7),
    L(64, 64, GN, LRELU, out=RELU, stats=True, bias=True), L(192, 16, GN, LRELU, res=True, stats=True),
    L(32, 3, MINMAX, LRELU, res=True, bias=True), L(3, 128, out=RELU, bias=True, w='w_ld'),
    L(256, 128, GN, LRELU, out=RELU, res=True, stats=True, bias=True, slope=-0.3),
]
LINEAR_CASES = list(dict.fromkeys(LINEAR_CASES))


def linear_id(case):
    (cin, cout, mode, act, out, res, stats, bias, _), slope, w = case
    s = f'{cin}x{cout}-{("plain", "gn", "minmax")[mode]}'
    s += '' if act == NONE else f'-lrelu{slope}'
    s += '-relu' if out == RELU else ''
    s += '-res' if res else ''
    s += '-stats' if stats else ''
    s += '-bias' if bias else ''
    return s + (f'-{w}' if w else '')


GN_ACT_C = [16, 32, 48, 64, 96, 128, 256]
GN_ACT_MODES = [('none', None), ('lrelu', 0.1), ('prelu', -0.3), ('prelu', 1.7)]   # prelu: the slope read on the device
TRANSPOSE_C = [3, 61, 64, 128]
PRELU_PAIRS = [(-0.3, 1.7), (0.25, -0.3), (1.7, 0.25)]                            # (prelu1, preluk)
CORR_FORMS = {'loop': (True, True, True),               # feature + motion, corr written: the RAFT loop at N % 128 != 0
              'feature': (True, False, True),           # CorrBlock.__call__
              'motion': (False, True, False)}           # MotionEncoder.forward, from corr_in
FLOW_OUT_CASES = [(True, False, False, False),            # FlowHead.forward
                  (True, True, True, True),               # the RAFT loop: coords2_out aliases coords2
                  (True, True, False, False), (True, True, True, False), (True, True, False, True),
                  (False, True, False, False), (False, True, True, False), (False, True, True, True)]


def covered():
    keys = {('linear',) + case[0] for case in LINEAR_CASES}
    for c in GN_ACT_C:
        for act, _ in GN_ACT_MODES:
            for tr in (False, True):
                keys.add(('gn_act', c, NONE if act == 'none' else LRELU, act == 'prelu', tr))
    keys |= {('corr_feature',) + f for f in CORR_FORMS.values()}
    keys |= {('flow_out',) + f for f in FLOW_OUT_CASES}
    keys |= {('gru',), ('transpose',)}
    return keys


# ----------------------------------------------------------------------------------------------------------------------
# (a) the configurations the product launches
# ----------------------------------------------------------------------------------------------------------------------
RECORDED_OPS = ('linear', 'gn_act', 'transpose', 'corr_feature', 'gru', 'flow_out')


def record_key(op, sig, a, k):
    """(op, configuration...) of one call, and its shape."""
    if op in ('linear', 'gn_act', 'transpose'):
        p = sig.bind(*a, **k)
        p.apply_defaults()
        p = p.arguments
    if op == 'linear':
        x, w = p['x'], p['weight']
        cin = x.shape[-1] if p['cin'] is None else p['cin']
        cout = w.shape[0] if p['cout'] is None else p['cout']
        key = (op, cin, cout, p['in_mode'], p['in_act'], p['out_act'], p['residual'] is not None, p['out_stats'] is not None,
               p['bias'] is not None, bool(p['w_ld'] or p['w_cin']))
        return key, tuple(x.shape[:2])
    if op == 'gn_act':
        x = p['x']
        return (op, x.shape[-1], p['act'], p['slope_dev'] is not None, bool(p['transpose_out'])), tuple(x.shape[:2])
    if op == 'transpose':
        return (op,), tuple(p['x'].shape)
    s = a[0]
    if op == 'corr_feature':
        return (op, s.y1 is not None, s.motion is not None, s.corr_feat is not None), (s.B, s.N)
    if op == 'flow_out':
        alias = s.coords2_out is not None and s.coords2_out == s.coords2
        return (op, s.delta is not None, s.coords2_out is not None, s.flow_out is not None, alias), (s.B, s.N)
    return (op,), (s.B, s.N)


@pytest.fixture(scope='module')
def recorded(dev):
    """Eager runs of the product (CUDA graphs off, default weights) with every call of the six entry points recorded:
    {(op, configuration...): {shape, ...}}."""
    from pvraft_b200 import RSF, RSF_refine, ops
    seen = {}
    with pytest.MonkeyPatch.context() as mp:
        for name in RECORDED_OPS:
            real = getattr(ops, name)
            sig = inspect.signature(real)

            def wrap(*a, _real=real, _name=name, _sig=sig, **k):
                key, shape = record_key(_name, _sig, a, k)
                seen.setdefault(key, set()).add(shape)
                return _real(*a, **k)
            mp.setattr(ops, name, wrap)

        def model(cls, k, seed=0):
            torch.manual_seed(seed)
            m = cls(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)).to(dev)
            m.use_cuda_graph = False
            return m

        b, n = 2, 1000
        pc1, pc2 = [t.to(dev) for t in O.synthetic_clouds(b, n, seed=21)]
        m, mr = model(RSF, 128).eval(), model(RSF_refine, 128).eval()
        with torch.no_grad():
            m([pc1, pc2], 2)
            mr([pc1, pc2], 2)
            q1, q2 = [t.to(dev) for t in O.synthetic_clouds(b, 1024, seed=22)]
            mr([q1, q2], 2)                                   # the refine head behind the tensor-core loop
            big = model(RSF, 512).eval()
            r1, r2 = [t.to(dev) for t in O.synthetic_clouds(8, 8192, seed=23)]
            big([r1, r2], 1)                                  # the encoders' first layers at the bench shape
            del big, r1, r2
        # training steps: stage 1 and the refiner
        m.train()
        sequence_loss(m([pc1, pc2], num_iters=2), pc2 - pc1).backward()
        mr.train()
        (mr([pc1, pc2], num_iters=2) - (pc2 - pc1)).abs().mean().backward()
        m.eval()
        # every reference-layout module seam
        with torch.no_grad():
            xyz1, _, graph, graph_context, net, inp = m._encode([pc1, pc2])
            cb, ub = m.corr_block, m.update_block
            coords = (pc1 + 0.05 * torch.randn_like(pc1)).contiguous()
            flow = (coords - pc1).contiguous()
            corr = cb(coords)
            cb.get_voxel_feature(coords)
            cb.get_knn_feature(coords)
            ub.motion_encoder(flow, corr)
            net_cm, inp_cm = net.transpose(1, 2).contiguous(), inp.transpose(1, 2).contiguous()
            ub.gru(net_cm, torch.cat([inp_cm, inp_cm], 1))
            ub.flow_head(net_cm, graph_context)
            ub(net_cm, inp_cm, corr, flow, graph_context)
            fe = m.feature_extractor
            x = fe.feat_conv1(pc1, graph)
            x = fe.feat_conv2(x, graph)
            fe.feat_conv3(x, graph)
            fe(pc1, point_major=False)
        torch.cuda.synchronize()
    return seen


def test_recorded_configurations_are_covered(recorded):
    """Every configuration of the six CUDA-core entry points that the product launches has a parity case in (b)."""
    from pvraft_b200 import ops
    assert (ops.IN_PLAIN, ops.IN_GN, ops.IN_GN_MINMAX) == (PLAIN, GN, MINMAX)
    assert (ops.ACT_NONE, ops.ACT_RELU, ops.ACT_LRELU) == (NONE, RELU, LRELU)
    for key in sorted(recorded, key=str):
        print('recorded', key, sorted(recorded[key]))
    assert {k[0] for k in recorded} == set(RECORDED_OPS), 'an entry point was never called'
    missing = set(recorded) - covered()
    assert not missing, f'configurations without a parity case: {sorted(missing, key=str)}'


# ----------------------------------------------------------------------------------------------------------------------
# (b) k_linear
# ----------------------------------------------------------------------------------------------------------------------
def linear_inputs(case, b, n, dev, seed):
    (cin, cout, mode, act, out, res, stats, bias, _), slope, wform = case
    g = torch.Generator().manual_seed(seed)
    x = sample_scaled(g, b, n, cin).to(dev)
    wcols = cin + 3 if wform == 'w_ld' else (cin - 3 if wform == 'w_cin' else cin)
    k = min(cin, wcols)
    c = dict(x=x, w=(torch.randn(cout, wcols, generator=g) / k ** 0.5).to(dev), k=k,
             bias=torch.randn(cout, generator=g).to(dev) if bias else None,
             residual=sample_scaled(g, b, n, cout, offset=-0.2).to(dev) if res else None,
             kw=dict(cin=cin, cout=cout, w_ld=cin + 3 if wform == 'w_ld' else 0, w_cin=cin - 3 if wform == 'w_cin' else 0,
                     in_mode=mode, in_act=act, in_slope=0.0 if slope is None else slope, out_act=out))
    if mode != PLAIN:
        gamma, beta = both_signs(g, cin).to(dev), (torch.randn(cin, generator=g) * 0.2).to(dev)
        xmin = (x - torch.rand(b, n, cin, generator=g).to(dev)) if mode == MINMAX else None
        st, cnt = gn_stats(x.double()), float(n * (cin // 8))
        c.update(gamma=gamma, beta=beta, xmin=xmin, stats=st, count=cnt)
        c['kw'].update(in_min=xmin, in_stats=st, in_gamma=gamma, in_beta=beta, in_count=cnt)
    return c


def linear_run(c, want_stats, sl=slice(None)):
    """ops.linear on the samples `sl` of the case -> (out, out_stats or None)."""
    from pvraft_b200 import ops
    kw = dict(c['kw'])
    for name in ('in_min', 'in_stats'):
        if kw.get(name) is not None:
            kw[name] = kw[name][sl].contiguous()
    x = c['x'][sl].contiguous()
    ostats = torch.zeros(x.shape[0], 8, 2, dtype=torch.float64, device=x.device) if want_stats else None
    res = None if c['residual'] is None else c['residual'][sl].contiguous()
    y = ops.linear(x, c['w'], c['bias'], out_stats=ostats, residual=res, **kw)
    return (y, ostats) if want_stats else (y,)


def linear_ref(case, c):
    (cin, cout, mode, act, out, res, stats, bias, _), slope, _ = case
    x64 = c['x'].double()[..., :c['k']]
    if mode != PLAIN:
        x64 = gn_act_ref(x64, None if c['xmin'] is None else c['xmin'].double(), c['stats'], c['gamma'], c['beta'], c['count'],
                         1.0 if act == NONE else slope)
    y = x64 @ c['w'].double()[:, :c['k']].t()
    if bias:
        y = y + c['bias'].double()
    if out == RELU:
        y = torch.relu(y)
    if res:
        y = y + c['residual'].double()
    return y


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('case', LINEAR_CASES, ids=[linear_id(c) for c in LINEAR_CASES])
def test_linear(dev, case, shape, det):
    """out = out_act(W in_act(GN(x)) + bias) + residual, and the output's per-sample GroupNorm sums (default and DET form,
    which must repeat its bits); IN_GN_MINMAX takes the min array in the channels whose GroupNorm scale is negative."""
    key, slope, wform = case
    cin, cout, stats = key[0], key[1], key[6]
    if det and not stats:
        pytest.skip('the deterministic form differs only in the output sums')
    b, n = SHAPES[shape]
    c = linear_inputs(case, b, n, dev, seed=cin * 1000 + cout * 7 + n + LINEAR_CASES.index(case))
    if key[2] == MINMAX:
        assert bool((c['gamma'] < 0).any()) and bool((c['gamma'] > 0).any())
    out = run_checked(det, lambda: linear_run(c, stats))
    err = note('linear', per_sample_err(out[0], linear_ref(case, c)) / max(1, cin / 128))
    es = note('linear stats', check_out_stats(out[1], out[0])) if stats else None
    print(f'linear {linear_id(case)} B={b} N={n}{" DET" if det else ""}: err {err:.2e} (of the bound\'s scale)'
          + (f', stats {es:.2e}' if es is not None else ''))
    assert err < 2e-6, err


# ----------------------------------------------------------------------------------------------------------------------
# (b) k_gn_act, k_transpose
# ----------------------------------------------------------------------------------------------------------------------
def gn_act_inputs(c, b, n, dev, seed):
    g = torch.Generator().manual_seed(seed)
    x = sample_scaled(g, b, n, c).to(dev)
    return dict(x=x, stats=gn_stats(x.double()), count=float(n * (c // 8)), gamma=both_signs(g, c).to(dev),
                beta=(torch.randn(c, generator=g) * 0.2).to(dev))


def gn_act_run(d, act, slope, transpose_out, sl=slice(None)):
    from pvraft_b200 import ops
    sdev = torch.tensor([slope], dtype=torch.float32, device=d['x'].device) if act == 'prelu' else None
    return ops.gn_act(d['x'][sl].contiguous(), d['stats'][sl].contiguous(), d['gamma'], d['beta'], d['count'],
                      NONE if act == 'none' else LRELU, 0.1 if act == 'prelu' else (slope or 0.0), transpose_out, slope_dev=sdev)


@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('transpose_out', [False, True])
@pytest.mark.parametrize('act,slope', GN_ACT_MODES)
@pytest.mark.parametrize('c', GN_ACT_C)
def test_gn_act(dev, c, act, slope, transpose_out, shape):
    """act(GroupNorm(x)) from the sums, point-major or channel-major; PReLU through the device slope (the host slope 0.1
    passed beside it must be ignored)."""
    b, n = SHAPES[shape]
    d = gn_act_inputs(c, b, n, dev, seed=c * 31 + n + int(10 * (slope or 0)) + transpose_out)
    got = gn_act_run(d, act, slope, transpose_out)
    want = gn_act_ref(d['x'].double(), None, d['stats'], d['gamma'], d['beta'], d['count'], 1.0 if act == 'none' else slope)
    if transpose_out:
        want = want.transpose(1, 2)
    assert got.shape == want.shape
    err = note('gn_act', per_sample_err(got, want))
    print(f'gn_act C={c} {act}{"" if slope is None else f" {slope}"} transpose={transpose_out} B={b} N={n}: err {err:.2e}')
    assert err < 1e-6, err


@pytest.mark.parametrize('shape', ['tail', 'multi'])
@pytest.mark.parametrize('c', TRANSPOSE_C)
def test_transpose(dev, c, shape):
    """[B,R,C] -> [B,C,R], bitwise, with neither R nor C a multiple of 32 (and C = 64, 128)."""
    from pvraft_b200 import ops
    b, r = SHAPES[shape]
    x = sample_scaled(torch.Generator().manual_seed(c + r), b, r, c).to(dev)
    assert torch.equal(ops.transpose(x), x.transpose(1, 2).contiguous())
    assert torch.equal(ops.transpose(x.transpose(1, 2).contiguous()), x)


# ----------------------------------------------------------------------------------------------------------------------
# (b) k_corrfeat
# ----------------------------------------------------------------------------------------------------------------------
def knn_moments(sel64):
    """[B,N,32,4] -> [B,16] moments as the lookup accumulates them."""
    b = sel64.shape[0]
    f = sel64.reshape(b, -1, 4)
    iu = torch.triu_indices(4, 4)
    m = torch.zeros(b, 16, dtype=torch.float64, device=sel64.device)
    m[:, :4] = f.sum(1)
    m[:, 4:14] = torch.einsum('bni,bnj->bij', f, f)[:, iu[0], iu[1]]
    m[:, 14] = f.shape[1]
    return m


def corr_inputs(b, n, slopes, dev, seed):
    g = torch.Generator().manual_seed(seed)

    def w(co, ci, s=1.0):
        return (torch.randn(co, ci, generator=g) * s / ci ** 0.5).to(dev)

    def v(c, s=1.0):
        return (torch.randn(c, generator=g) * s).to(dev)

    y1 = sample_scaled(g, b, n, 128).to(dev)
    sel = sample_scaled(g, b, n, 32, 4, offset=-0.2).to(dev)
    c = dict(y1=y1, y1_stats=gn_stats(y1.double()), gn1_gamma=both_signs(g, 128).to(dev), gn1_beta=v(128, 0.2),
             prelu1=torch.tensor([slopes[0]], device=dev), w_out=w(64, 128), b_out=v(64),
             knn_sel=sel, moments=knn_moments(sel.double()), w_knn=w(64, 4), b_knn=v(64), gnk_gamma=both_signs(g, 64).to(dev),
             gnk_beta=v(64, 0.2), preluk=torch.tensor([slopes[1]], device=dev), w_kout=w(64, 64), b_kout=v(64),
             corr_in=sample_scaled(g, b, n, 64).to(dev), flow=sample_scaled(g, b, n, 3, offset=0.5).to(dev),
             w_cc=w(64, 64), b_cc=v(64), w_cf=w(64, 3), b_cf=v(64), w_cm=w(61, 128), b_cm=v(61))
    return c


def corr_run(c, form, sl=slice(None)):
    """ops.corr_feature in one of CORR_FORMS on the samples `sl` -> (corr or None, motion or None)."""
    from pvraft_b200 import _lib, ops
    feat, motion, write_corr = CORR_FORMS[form]
    t = {k: (v[sl].contiguous() if k in ('y1', 'y1_stats', 'knn_sel', 'moments', 'corr_in', 'flow') else v) for k, v in c.items()}
    b, n = t['y1'].shape[:2]
    a = _lib.CorrFeatArgs()
    if feat:
        for k in ('y1', 'gn1_gamma', 'gn1_beta', 'prelu1', 'w_out', 'b_out', 'knn_sel', 'w_knn', 'b_knn', 'gnk_gamma', 'gnk_beta',
                  'preluk', 'w_kout', 'b_kout'):
            setattr(a, k, ops._p(t[k]))
        a.y1_stats, a.moments = ops._p(t['y1_stats'], torch.float64), ops._p(t['moments'], torch.float64)
    else:
        a.corr_in = ops._p(t['corr_in'])
    corr = torch.empty(b, n, 64, device=t['y1'].device) if write_corr else None
    mot = torch.empty(b, n, 64, device=t['y1'].device) if motion else None
    a.corr_feat, a.motion = ops._p(corr), ops._p(mot)
    if motion:
        for k in ('flow', 'w_cc', 'b_cc', 'w_cf', 'b_cf', 'w_cm', 'b_cm'):
            setattr(a, k, ops._p(t[k]))
    a.B, a.N = b, n
    ops.corr_feature(a)
    return corr, mot


def corr_ref(c):
    """Correlation feature head (model/corr.py:42-45, 71-73, 86-93), float64, one sample at a time."""
    d = {k: v.double() for k, v in c.items()}
    b, n = c['y1'].shape[:2]
    s1, sk = float(c['prelu1']), float(c['preluk'])
    a1 = gn_act_ref(d['y1'], None, d['y1_stats'], d['gn1_gamma'], d['gn1_beta'], float(n * 16), s1)
    out = a1 @ d['w_out'].t() + d['b_out']
    for s in range(b):
        t = d['knn_sel'][s].reshape(n * 32, 4) @ d['w_knn'].t() + d['b_knn']
        t = gn_self(t) * d['gnk_gamma'] + d['gnk_beta']
        kmax = prelu(t, sk).reshape(n, 32, 64).amax(1)
        out[s] += kmax @ d['w_kout'].t() + d['b_kout']
    return out


def motion_ref(c, corr64):
    """MotionEncoder (model/update.py:15-21), float64: [relu(conv(relu(conv_corr(corr)), relu(conv_flow(flow)))), flow]."""
    d = {k: v.double() for k, v in c.items()}
    cc = torch.relu(corr64 @ d['w_cc'].t() + d['b_cc'])
    cf = torch.relu(d['flow'] @ d['w_cf'].t() + d['b_cf'])
    mo = torch.relu(torch.cat([cc, cf], -1) @ d['w_cm'].t() + d['b_cm'])
    return torch.cat([mo, d['flow']], -1)


def corr_cases():
    return [(f, s) for f in ('loop', 'feature') for s in PRELU_PAIRS] + [('motion', None)]


@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('form,slopes', corr_cases())
def test_corr_feature(dev, form, slopes, shape):
    """The feature head (GroupNorm + PReLU of y1 -> out_conv[3], plus the kNN branch from the moments of knn_sel, PReLU, max,
    knn_out) and the motion encoder, in the three forms the product launches; PReLU slopes below 0, in (0, 1) and above 1,
    GroupNorm gammas of both signs.  Motion channels 61-63 carry the flow bitwise."""
    b, n = SHAPES[shape]
    c = corr_inputs(b, n, slopes or (0.25, 0.25), dev, seed=n + len(form) * 10 + int(10 * (slopes or (0, 0))[0]))
    corr, mot = corr_run(c, form)
    msg = f'corr_feature {form}{"" if slopes is None else f" slopes={slopes}"} B={b} N={n}:'
    if form == 'motion':
        want_corr = c['corr_in'].double()
    else:
        want_corr = corr_ref(c)
        e = note('corr', per_sample_err(corr, want_corr))
        msg += f' corr {e:.2e}'
        assert e < 1e-5, e
    if mot is not None:
        e = note('motion', per_sample_err(mot, motion_ref(c, want_corr)))
        msg += f' motion {e:.2e}'
        assert e < 2e-5, e
        assert torch.equal(mot[..., 61:], c['flow'])
    print(msg)


# ----------------------------------------------------------------------------------------------------------------------
# (b) k_gru
# ----------------------------------------------------------------------------------------------------------------------
def gru_inputs(b, n, saturating, dev, seed):
    g = torch.Generator().manual_seed(seed)
    h, inp, mot = [(sample_scaled(g, b, n, 64, offset=o) * 0.5).to(dev) for o in (0.3, -0.2, 0.1)]
    ws = [(torch.randn(64, 192, generator=g) / 192 ** 0.5).to(dev) for _ in range(3)]
    if saturating:   # pre-activations around +-30: sigmoid and tanh saturate
        bs = [(torch.randn(64, generator=g).sign() * 30 + torch.randn(64, generator=g)).to(dev) for _ in range(3)]
    else:
        bs = [torch.randn(64, generator=g).to(dev) for _ in range(3)]
    return dict(net=h, inp=inp, motion=mot, w_z=ws[0], w_r=ws[1], w_q=ws[2], b_z=bs[0], b_r=bs[1], b_q=bs[2])


def gru_run(c, sl=slice(None)):
    from pvraft_b200 import _lib, ops
    h, inp, mot = [c[k][sl].contiguous() for k in ('net', 'inp', 'motion')]
    out = torch.empty_like(h)
    a = _lib.GruArgs(ops._p(h), ops._p(inp), ops._p(mot), ops._p(c['w_z']), ops._p(c['b_z']), ops._p(c['w_r']), ops._p(c['b_r']),
                     ops._p(c['w_q']), ops._p(c['b_q']), ops._p(out), h.shape[0], h.shape[1])
    ops.gru(a)
    return out


def gru_ref(c):
    """ConvGRU (model/update.py:31-40), float64."""
    d = {k: v.double() for k, v in c.items()}
    hx = torch.cat([d['net'], d['inp'], d['motion']], -1)
    z = torch.sigmoid(hx @ d['w_z'].t() + d['b_z'])
    r = torch.sigmoid(hx @ d['w_r'].t() + d['b_r'])
    q = torch.tanh(torch.cat([r * d['net'], d['inp'], d['motion']], -1) @ d['w_q'].t() + d['b_q'])
    return (1 - z) * d['net'] + z * q


@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('saturating', [False, True])
def test_gru(dev, saturating, shape):
    """h' = (1 - z) h + z tanh(W_q [r h, x] + b_q) with [z, r] = sigmoid(W [h, x] + b); ordinary and saturating gates."""
    b, n = SHAPES[shape]
    c = gru_inputs(b, n, saturating, dev, seed=n + saturating)
    err = note('gru', per_sample_err(gru_run(c), gru_ref(c)))
    print(f'gru saturating={saturating} B={b} N={n}: err {err:.2e}')
    assert err < 1e-5, err


# ----------------------------------------------------------------------------------------------------------------------
# (b) k_flowout
# ----------------------------------------------------------------------------------------------------------------------
def flow_out_inputs(b, n, dev, seed):
    g = torch.Generator().manual_seed(seed)
    z3 = sample_scaled(g, b, n, 64).to(dev)
    c1 = (sample_scaled(g, b, n, 3) * 3).to(dev)
    return dict(z3=z3, z3_stats=gn_stats(z3.double()), gn3_gamma=both_signs(g, 64).to(dev), gn3_beta=(torch.randn(64, generator=g) * 0.2).to(dev),
                net=(sample_scaled(g, b, n, 64, offset=-0.2) * 0.5).to(dev),
                w_c1=(torch.randn(64, 64, generator=g) / 8).to(dev), b_c1=torch.randn(64, generator=g).to(dev),
                w_o0=(torch.randn(64, 128, generator=g) / 128 ** 0.5).to(dev), b_o0=torch.randn(64, generator=g).to(dev),
                w_o2=(torch.randn(3, 64, generator=g) / 8).to(dev), b_o2=torch.randn(3, generator=g).to(dev),
                coords1=c1, coords2=(c1 + torch.randn(b, n, 3, generator=g).to(dev) * 0.1).contiguous())


def flow_out_run(c, outs, sl=slice(None)):
    """ops.flow_out with the outputs `outs` = (delta?, coords2_out?, flow_out?, coords2_out aliases coords2?) on the samples
    `sl` -> (delta, coords2 after the call, coords2_out, flow) (None where not requested)."""
    from pvraft_b200 import _lib, ops
    want_delta, want_c2, want_flow, alias = outs
    t = {k: v[sl].contiguous() for k, v in c.items() if k in ('z3', 'z3_stats', 'net', 'coords1', 'coords2')}
    b, n = t['z3'].shape[:2]
    dev = t['z3'].device
    coords2 = t['coords2'].clone()
    delta = torch.empty(b, n, 3, device=dev) if want_delta else None
    c2o = (coords2 if alias else torch.empty(b, n, 3, device=dev)) if want_c2 else None
    flow = torch.empty(b, n, 3, device=dev) if want_flow else None
    a = _lib.FlowOutArgs(ops._p(t['z3']), ops._p(t['z3_stats'], torch.float64), ops._p(c['gn3_gamma']), ops._p(c['gn3_beta']),
                         ops._p(t['net']), ops._p(c['w_c1']), ops._p(c['b_c1']), ops._p(c['w_o0']), ops._p(c['b_o0']),
                         ops._p(c['w_o2']), ops._p(c['b_o2']), ops._p(t['coords1']), ops._p(coords2), ops._p(delta), ops._p(c2o),
                         ops._p(flow), b, n)
    ops.flow_out(a)
    return delta, coords2, c2o, flow


def flow_out_ref(c):
    """FlowHead tail (model/update.py:69-72) on LeakyReLU(GN3(z3)), float64 -> delta [B,N,3]."""
    d = {k: v.double() for k, v in c.items()}
    n = c['z3'].shape[1]
    s = gn_act_ref(d['z3'], None, d['z3_stats'], d['gn3_gamma'], d['gn3_beta'], float(n * 8), 0.1)
    a = d['net'] @ d['w_c1'].t() + d['b_c1']
    y = torch.relu(torch.cat([s, a], -1) @ d['w_o0'].t() + d['b_o0'])
    return y @ d['w_o2'].t() + d['b_o2']


@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('outs', FLOW_OUT_CASES, ids=lambda o: '-'.join(n for n, f in zip(('delta', 'c2', 'flow', 'alias'), o) if f))
def test_flow_out(dev, outs, shape):
    """delta against float64 (GN3 gammas of both signs); coords2_out = coords2 + delta in fp32 and flow_out = coords2_out -
    coords1, bitwise, from the kernel's own delta (a delta-only run where this one writes none); coords2 untouched unless
    aliased."""
    b, n = SHAPES[shape]
    c = flow_out_inputs(b, n, dev, seed=n + 5)
    own = flow_out_run(c, (True, False, False, False))[0]
    err = note('delta', per_sample_err(own, flow_out_ref(c)))
    delta, coords2, c2o, flow = flow_out_run(c, outs)
    if delta is not None:
        assert same_bits(delta, own)
    if c2o is not None:
        assert torch.equal(c2o, c['coords2'] + own)
        if flow is not None:
            assert torch.equal(flow, c2o - c['coords1'])
    if not outs[3]:
        assert torch.equal(coords2, c['coords2'])
    print(f'flow_out {outs} B={b} N={n}: delta err {err:.2e}')
    assert err < 5e-5, err


# ----------------------------------------------------------------------------------------------------------------------
# (c) batch invariance
# ----------------------------------------------------------------------------------------------------------------------
def per_sample_equal(batched, singles):
    """Sample s of each batched output has the bits of the single-sample run s; -> the samples that differ."""
    return [s for s, one in enumerate(singles) if not all(x is None or same_bits(x[s:s + 1], y) for x, y in zip(batched, one))]


BATCH_LINEAR = [L(16, 32, MINMAX, LRELU, stats=True), L(128, 3, GN, LRELU, res=True, bias=True),
                L(84, 128, stats=True, bias=True, w='w_cin'), L(256, 128, GN, LRELU, out=RELU, res=True, stats=True, bias=True, slope=-0.3)]


@pytest.mark.parametrize('det', [False, True])
@pytest.mark.parametrize('case', BATCH_LINEAR, ids=[linear_id(c) for c in BATCH_LINEAR])
def test_linear_batch_invariance(dev, case, det):
    """k_linear over the `multi` batch against one launch per sample: the same output bits; DET: the same output sums,
    bitwise; default form: sums within the GroupNorm sum bound of each other."""
    assert case in LINEAR_CASES
    key = case[0]
    stats = key[6]
    if det and not stats:
        pytest.skip('the deterministic form differs only in the output sums')
    b, n = SHAPES['multi']
    c = linear_inputs(case, b, n, dev, seed=key[0] + key[1] + 99)
    with det_mode(det):
        both = linear_run(c, stats)
        singles = [linear_run(c, stats, slice(s, s + 1)) for s in range(b)]
    assert not per_sample_equal(both[:1], [o[:1] for o in singles]), 'outputs differ from the single-sample launches'
    if stats:
        st_one = torch.cat([o[1] for o in singles])
        if det:
            assert same_bits(both[1], st_one), 'DET output sums differ from the single-sample launches'
        else:
            y = both[0].double().reshape(b, n, 8, key[1] // 8)
            s1, s2, sabs = y.sum((1, 3)), (y ** 2).sum((1, 3)), y.abs().sum((1, 3))
            d1, d2 = (both[1][..., 0] - st_one[..., 0]).abs(), (both[1][..., 1] - st_one[..., 1]).abs()
            assert bool((d1 <= 1e-5 * s1.abs() + 1e-7 * sabs).all() and (d2 <= 1e-5 * s2).all()), (both[1], st_one)
    print(f'linear {linear_id(case)}{" DET" if det else ""}: B={b} N={n} bitwise equal to one launch per sample')


def test_gn_act_transpose_batch_invariance(dev):
    from pvraft_b200 import ops
    b, n = SHAPES['multi']
    d = gn_act_inputs(128, b, n, dev, seed=3)
    for tr in (False, True):
        both = gn_act_run(d, 'prelu', -0.3, tr)
        assert not per_sample_equal((both,), [(gn_act_run(d, 'prelu', -0.3, tr, slice(s, s + 1)),) for s in range(b)])
    x = d['x'][..., :61].contiguous()
    both = ops.transpose(x)
    assert not per_sample_equal((both,), [(ops.transpose(x[s:s + 1].contiguous()),) for s in range(b)])


@pytest.mark.parametrize('form', list(CORR_FORMS))
def test_corr_feature_batch_invariance(dev, form):
    """k_corrfeat over the `multi` batch against one launch per sample, with the same y1 sums and kNN moments."""
    b, n = SHAPES['multi']
    c = corr_inputs(b, n, (-0.3, 1.7), dev, seed=len(form))
    both = corr_run(c, form)
    bad = per_sample_equal(both, [corr_run(c, form, slice(s, s + 1)) for s in range(b)])
    assert not bad, f'samples {bad} differ from their single-sample launches'


def test_gru_batch_invariance(dev):
    b, n = SHAPES['multi']
    c = gru_inputs(b, n, False, dev, seed=7)
    bad = per_sample_equal((gru_run(c),), [(gru_run(c, slice(s, s + 1)),) for s in range(b)])
    assert not bad, f'samples {bad} differ from their single-sample launches'


@pytest.mark.parametrize('outs', [(True, True, True, True), (True, False, False, False)], ids=['loop', 'delta'])
def test_flow_out_batch_invariance(dev, outs):
    b, n = SHAPES['multi']
    c = flow_out_inputs(b, n, dev, seed=11)
    bad = per_sample_equal(flow_out_run(c, outs), [flow_out_run(c, outs, slice(s, s + 1)) for s in range(b)])
    assert not bad, f'samples {bad} differ from their single-sample launches'


# ----------------------------------------------------------------------------------------------------------------------
# (d) the model at a multi-tile ragged shape
# ----------------------------------------------------------------------------------------------------------------------
def per_sample_clouds(b, n, seed):
    pc1, pc2 = O.synthetic_clouds(b, n, seed=seed)
    s = torch.arange(b, dtype=torch.float32).view(b, 1, 1)
    scale, shift = 0.4 * (1 + 0.1 * s), 3.0 * s
    return pc1 * scale + shift, pc2 * scale + shift


def knn_tie_rows(cb, coords, state, pc2):
    """Rows whose 32 lookup neighbours (the product's, on its own slots) differ from the oracle's; each must differ only at
    an exact tie of the 32nd distance (either set is valid, see check_lookup in test_gpu_kernel_coverage.py)."""
    b = coords.shape[0]
    slots = cb.lookup(coords.to(cb.corr_val.device), want_slots=True)['knn_slot'].long().cpu()
    got = torch.gather(cb.candidate_ids().cpu(), 2, slots)
    want = torch.gather(state.indices, 2, O.knn_select(state, coords))
    differ = (got.sort(-1).values != want.sort(-1).values).any(-1)

    def kth(ids):   # largest squared distance of a selection, in the oracle's fp32 form
        d = torch.gather(pc2.unsqueeze(1).expand(b, ids.shape[1], -1, 3), 2, ids.unsqueeze(-1).expand(*ids.shape, 3)) - coords.unsqueeze(2)
        return ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).amax(-1)
    assert torch.equal(kth(got)[differ], kth(want)[differ]), 'kNN sets differ beyond exact ties'
    return differ


def test_model_level_multi_tile_ragged(dev, sm_count):
    """RSF at B = 3, N = 4999 (79 tiles per sample: at one CTA per SM, CTAs hold tiles of two samples), K = 512, 3
    iterations, random GroupNorm affines and PReLU slopes (-0.3, 1.7), on the oracle's adjacency: CorrBlock.__call__ and
    UpdateBlock.forward teacher-forced with the oracle's state per iteration, and the free-running flows.  A row whose
    32nd kNN distance ties exactly may take either neighbour (one row of the 44 991 here): such rows are left out of the
    correlation comparison."""
    from pvraft_b200 import RSF, Graph
    b, n, k, iters = 3, 4999, 512, 3
    assert straddling_ctas(b, n, sm_count, 1) > 0
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    m = RSF(args)
    m.load_state_dict(default_weights(args=args, seed=4))
    randomise_affine(m, 9, (-0.3, 1.7))
    W = {key: v.detach().clone() for key, v in m.state_dict().items()}
    m = m.to(dev).eval()
    m.use_cuda_graph = False
    pc1, pc2 = per_sample_clouds(b, n, seed=4999)
    with torch.no_grad():
        li = O.prepare(W, pc1, pc2, k)
        trace = []
        want = O.raft_loop(W, li, pc1, iters, 3, 0.25, trace)
        with oracle_adjacency():
            got = m([pc1.to(dev), pc2.to(dev)], iters)
        free = [float((g.cpu() - w).abs().mean() / w.abs().mean()) for g, w in zip(got, want)]
        m.corr_block.set_state(li.state.truncated_corr.to(dev), li.state.indices.to(dev), pc2.to(dev))
        og = li.graph
        nbr = (og.edges.reshape(b, n, 32) - (torch.arange(b) * n).view(b, 1, 1)).to(torch.int32)
        graph = Graph(nbr.to(dev), og.edge_feats.reshape(b, n, 32, 3).to(dev).contiguous(), 32, [b * n, b * n])
        net, inp = li.net.to(dev), li.inp.to(dev)
        worst = dict(corr=0.0, net=0.0, delta=0.0)
        ties = 0
        for it, t in enumerate(trace):
            coords = t['coords'].to(dev).contiguous()
            tie = knn_tie_rows(m.corr_block, t['coords'], li.state, pc2)
            ties += int(tie.sum())
            corr = torch.where(tie.unsqueeze(1), t['corr'], m.corr_block(coords).cpu())
            errs = dict(corr=per_sample_err(corr, t['corr']))
            net2, delta = m.update_block(net, inp, t['corr'].to(dev), (t['coords'] - pc1).to(dev), graph)
            errs.update(net=per_sample_err(net2, t['net']), delta=per_sample_err(delta, t['delta']))
            for key, e in errs.items():
                worst[key] = max(worst[key], note(f'model {key}', e))
            assert errs['corr'] < 1e-5 and errs['net'] < 1e-5 and errs['delta'] < 5e-5, (it, errs)
            net = t['net'].to(dev)
    note('model free-running', max(free))
    print(f'model B={b} N={n} K={k}: teacher-forced worst', {key: f'{v:.2e}' for key, v in worst.items()},
          f'({ties} rows with a tied 32nd neighbour left out), free-running mean-abs / mean|flow| per iteration',
          [f'{e:.1e}' for e in free])
    assert ties <= 1e-3 * b * n * iters, ties
    assert max(free) < 1e-4, free
