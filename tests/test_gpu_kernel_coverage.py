"""Kernel parity at the shapes, template instantiations and parameter regimes where a kernel can be wrong without the rest of
the suite noticing: every reference here is float64 (torch on the device or on the CPU) and independent of the library.

  * persistent kernels with more tiles than SMs, so that a CTA carries its operand ring, mbarrier phases, accumulator
    hand-off, GroupNorm table and statistics slot across tile (and sample) boundaries: k_tc_linear, k_corr_gemm
  * every k_tc_linear<NT> width, resident and streamed weights, 1-3 sources, every epilogue, the `tail` columns
  * every k_corr_lookup<KPL, POW2, SMEM_TAB, HALF> instantiation, the dynamic and the static work split
  * trained-weight regimes (negative / > 1 PReLU slopes, negative GroupNorm scales) in the kNN branch and the RAFT loop
  * the largest rows corr_topk stages (M = 49152), the SetConv edge kernel and the remaining gradient widths at the bench batch

Every uninitialised allocation is NaN-filled (integers: a huge value) for these tests, so a tile a kernel never writes
cannot pass by holding the previous call's result.  Errors are measured per sample (max-abs / max-abs of that sample) on
inputs whose scale and offset differ from sample to sample: state taken from the wrong sample is an O(1) error.

Tolerances (those of the existing tests of the same op at the depths they cover; measured worst values are printed with -s):
  tc_linear plain 3e-6 up to K = 256, GRU / FLOW epilogues 1e-5;  corr_matmul 2e-6 up to C = 128.  Deeper contractions get
      the bound scaled by K / 256 (C / 128): the tensor cores accumulate in fp32 and the error grows with the depth
      (measured about 1e-8 x K: 2-3e-6 at K = 512, 2.6e-6 at C = 256, on an H100 80GB HBM3, 700 W)
  output GroupNorm sums, against float64 sums of what they summarise: 1e-5 relative + 1e-7 of the group's sum of |y|
  corr_lookup cells bit-exact, means 1e-6, kNN sets up to exact ties, gathered vectors exact, moments as test_gpu_parity
  kNN branch 1e-5;  teacher-forced loop corr 1e-5, motion 2e-5, net 2e-5, delta 5e-5
  setconv_edge 1e-6;  gradients 2e-5 (corr_init_bwd), 1e-5 / 1e-6 (edge_bwd / edge_fwd)
"""
import math
import types

import pytest
import torch

from conftest import default_weights, rel_err
from oracle import pvraft_oracle as O
from train_helpers import randomise_affine

pytestmark = pytest.mark.gpu

SMEM_BUDGET = 227 * 1024             # opt-in dynamic shared memory per CTA on sm_90 (csrc/common.cuh)
ROWS = {'one_tile': (1, 128),        # a single 128-point tile
        'mixed': (5, 4096),          # 160 tiles > 132 SMs: CTA 0 runs tiles 0 (sample 0) and 132 (sample 4)
        'bench': (8, 8192)}          # the timed bench batch: 512 tiles


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
    """act(GroupNorm(x)) from the sums; with xmin64 the per-channel input is the min array where the GroupNorm scale is < 0."""
    c = x64.shape[-1]
    mean = stats[..., 0] / count
    rstd = (stats[..., 1] / count - mean ** 2 + 1e-5).rsqrt()
    sc = rstd.repeat_interleave(c // 8, 1).unsqueeze(1) * gamma.double()
    sh = beta.double() - mean.repeat_interleave(c // 8, 1).unsqueeze(1) * sc
    raw = x64 if xmin64 is None else torch.where(sc < 0, xmin64, x64)
    t = raw * sc + sh
    return torch.where(t >= 0, t, slope * t)


def check_out_stats(stats, y):
    """GroupNorm sums accumulated by a kernel, per sample and group, against float64 sums of the values y [B,R,C] they
    summarise: |error| <= 1e-5 |sum| + 1e-7 sum|y| for the first moment (which may cancel to nearly zero: the absolute
    part scales with the magnitude of what was summed), 1e-5 relative for the second."""
    b, r, c = y.shape
    s = y.double().reshape(b, r, 8, c // 8)
    s1, s2, sabs = s.sum((1, 3)), (s ** 2).sum((1, 3)), s.abs().sum((1, 3))
    d1, d2 = (stats[..., 0] - s1).abs(), (stats[..., 1] - s2).abs()
    assert bool((d1 <= 1e-5 * s1.abs() + 1e-7 * sabs).all()), (stats[..., 0], s1)
    assert bool((d2 <= 1e-5 * s2).all()), (stats[..., 1], s2)
    return max(float((d1 / sabs).max()), float((d2 / s2).max()))


def tc_weights_resident(k, n_pad, gru=False):
    """The host rule of pvraft_tc_linear_fwd: the whole hi/lo weight matrix stays in shared memory when that leaves a ring of
    >= 3 activation stages (or at least as many as streaming would); otherwise the weights travel with every k-block."""
    pitch = ((n_pad + 31) & ~31) + 4
    fixed = (4 * k + 2 * n_pad + 128 * pitch + (8 * 32 * 20 if gru else 0) + 4 * 128 * 2) * 4 + 1024 + 64
    budget = SMEM_BUDGET - 2048 - fixed
    a_stage = 2 * 128 * 32 * 4
    w_all = (k // 32) * 2 * n_pad * 32 * 4
    stages_res = (budget - w_all) // a_stage if w_all < budget else 0
    stages_str = budget // (a_stage + 2 * n_pad * 32 * 4)
    return stages_res >= 3 or stages_res >= stages_str


def ctas_spanning_samples(n_tiles, grid, tiles_per_sample):
    """Number of CTAs of a persistent kernel (tiles c, c + grid, ...) whose tiles belong to more than one sample."""
    return sum(1 for c in range(grid) if len({t // tiles_per_sample for t in range(c, n_tiles, grid)}) > 1)


def tc_tiles(b, n, sm):
    n_tiles = b * n // 128
    return n_tiles, ctas_spanning_samples(n_tiles, min(n_tiles, sm), n // 128)


def assert_multi_tile(rows, b, n, sm):
    n_tiles, spanning = tc_tiles(b, n, sm)
    if rows == 'one_tile':
        assert n_tiles == 1
    else:
        assert n_tiles > sm and spanning > 0, (n_tiles, sm, spanning)
    return n_tiles, spanning


# ----------------------------------------------------------------------------------------------------------------------
# tc_linear (k_tc_linear<NT>)
# ----------------------------------------------------------------------------------------------------------------------
def test_tc_matrix_takes_both_weight_paths():
    """The width matrix below runs both weight paths: K = 32 keeps every width resident, K = 512 streams n_pad >= 32."""
    for n_pad in range(16, 129, 16):
        assert tc_weights_resident(32, n_pad)
        assert tc_weights_resident(512, n_pad) == (n_pad == 16)
    assert not tc_weights_resident(192, 128, gru=True) and not tc_weights_resident(192, 64, gru=True)   # the GRU layers stream


@pytest.mark.parametrize('rows', ['one_tile', 'mixed', 'bench'])
@pytest.mark.parametrize('k', [32, 512])
@pytest.mark.parametrize('n_pad', [16, 32, 48, 64, 80, 96, 112, 128])
def test_tc_linear_every_tile_width(dev, sm_count, n_pad, k, rows):
    """Plain epilogue at every instantiated width: GroupNorm prologue with negative gammas (K = 512: with the max/min
    selection), bias, residual, output statistics when cout is a multiple of 32; widths that are not get cout = n_pad - 3."""
    from pvraft_b200 import ops
    b, n = ROWS[rows]
    n_tiles, spanning = assert_multi_tile(rows, b, n, sm_count)
    cout = n_pad if n_pad % 32 == 0 else n_pad - 3
    minmax = k == 512
    g = torch.Generator().manual_seed(n_pad * 1000 + k + b)
    x = sample_scaled(g, b, n, k).to(dev)
    xmin = (x - torch.rand(b, n, k, generator=g).to(dev)) if minmax else None
    w = (torch.randn(cout, k, generator=g) / k ** 0.5).to(dev)
    bias = torch.randn(cout, generator=g).to(dev)
    res = sample_scaled(g, b, n, cout, offset=-0.2).to(dev)
    gamma, beta = torch.randn(k, generator=g).to(dev), (torch.randn(k, generator=g) * 0.2).to(dev)
    assert (gamma < 0).any() and (gamma > 0).any()
    stats, cnt = gn_stats(x.double()), float(n * k // 8)
    a_in = gn_act_ref(x.double(), None if xmin is None else xmin.double(), stats, gamma, beta, cnt, 0.1)
    want = (a_in.reshape(-1, k) @ w.double().t()).reshape(b, n, cout) + bias.double() + res.double()
    ostats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev) if cout % 32 == 0 else None
    tw = ops.tc_weights(w)
    assert tw[2] == n_pad
    got = ops.tc_linear([x], tw, bias, in_min=xmin, in_stats=stats, in_gamma=gamma, in_beta=beta, in_count=cnt,
                        in_act=ops.ACT_LRELU, in_slope=0.1, residual=res, out_stats=ostats)
    err = per_sample_err(got, want)
    es = check_out_stats(ostats, got) if ostats is not None else None
    print(f'tc_linear n_pad={n_pad} K={k} {rows} ({n_tiles} tiles, {spanning} CTAs span samples): weights '
          f'{"resident" if tc_weights_resident(k, n_pad) else "streamed"}, err {err:.2e}' + (f', stats {es:.2e}' if es is not None else ''))
    assert err < 3e-6 * max(1, k / 256), err


@pytest.mark.parametrize('prologue', ['none', 'gn', 'minmax'])
@pytest.mark.parametrize('channels', [(64,), (64, 32), (96, 64, 32)])
def test_tc_linear_concatenated_sources(dev, sm_count, channels, prologue):
    """1-3 sources concatenated along K, the GroupNorm prologue (plain / with the min array, negative gammas) on source 0 only."""
    from pvraft_b200 import ops
    b, n = ROWS['mixed']
    assert_multi_tile('mixed', b, n, sm_count)
    cout, k = 64, sum(channels)
    g = torch.Generator().manual_seed(k * 10 + len(prologue))
    srcs = [sample_scaled(g, b, n, c, offset=0.3 - 0.2 * i).to(dev) for i, c in enumerate(channels)]
    c0 = channels[0]
    xmin = (srcs[0] - torch.rand(b, n, c0, generator=g).to(dev)) if prologue == 'minmax' else None
    gamma, beta = torch.randn(c0, generator=g).to(dev), (torch.randn(c0, generator=g) * 0.2).to(dev)
    w = (torch.randn(cout, k, generator=g) / k ** 0.5).to(dev)
    bias = torch.randn(cout, generator=g).to(dev)
    kw, first = {}, srcs[0].double()
    if prologue != 'none':
        stats, cnt = gn_stats(srcs[0].double()), float(n * c0 // 8)
        first = gn_act_ref(first, None if xmin is None else xmin.double(), stats, gamma, beta, cnt, 0.1)
        kw = dict(in_min=xmin, in_stats=stats, in_gamma=gamma, in_beta=beta, in_count=cnt, in_act=ops.ACT_LRELU, in_slope=0.1)
    a_in = torch.cat([first] + [s.double() for s in srcs[1:]], -1)
    want = torch.relu((a_in.reshape(-1, k) @ w.double().t()).reshape(b, n, cout) + bias.double())
    ostats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
    got = ops.tc_linear(srcs, ops.tc_weights(w), bias, out_act=ops.ACT_RELU, out_stats=ostats, **kw)
    err = per_sample_err(got, want)
    es = check_out_stats(ostats, got)
    print(f'tc_linear sources {channels} prologue={prologue}: err {err:.2e}, stats {es:.2e}')
    assert err < 3e-6, err


@pytest.mark.parametrize('rows', ['mixed', 'bench'])
@pytest.mark.parametrize('n_pad', [32, 64, 96, 128])
def test_tc_linear_tail_columns(dev, sm_count, n_pad, rows):
    """cat([relu(W [a | b] + bias), tail]) with cout = n_pad - 3: the MotionEncoder's output layout (model/update.py:20)."""
    from pvraft_b200 import ops
    b, n = ROWS[rows]
    assert_multi_tile(rows, b, n, sm_count)
    cout = n_pad - 3
    g = torch.Generator().manual_seed(n_pad + b)
    srcs = [sample_scaled(g, b, n, 64).to(dev), sample_scaled(g, b, n, 64, offset=-0.1).to(dev)]
    tail = sample_scaled(g, b, n, 3).to(dev)
    w = (torch.randn(cout, 128, generator=g) / 128 ** 0.5).to(dev)
    bias = torch.randn(cout, generator=g).to(dev)
    want = torch.relu((torch.cat([s.double() for s in srcs], -1).reshape(-1, 128) @ w.double().t()).reshape(b, n, cout) + bias.double())
    got = ops.tc_linear(srcs, ops.tc_weights(w), bias, out_act=ops.ACT_RELU, tail=tail)
    assert got.shape == (b, n, n_pad)
    err = per_sample_err(got[..., :cout], want)
    print(f'tc_linear tail n_pad={n_pad} {rows}: err {err:.2e}')
    assert err < 3e-6, err
    assert torch.equal(got[..., cout:], tail)


@pytest.mark.parametrize('rows', ['mixed', 'bench'])
@pytest.mark.parametrize('pre', ['bias', 'bias+residual'])
def test_tc_linear_gru_epilogues(dev, sm_count, pre, rows):
    """ConvGRU gates (model/update.py:31-39) as the two fused layers run them: [z | r] = sigmoid(W_zr [h, inp, motion] + b
    (+ per-point pre-activation term)), out = z, out2 = r h; then h' = (1 - z) h + z tanh(W_q [r h, inp, motion] + b_q (+ term))."""
    from pvraft_b200 import ops
    b, n = ROWS[rows]
    assert_multi_tile(rows, b, n, sm_count)
    m = b * n
    g = torch.Generator().manual_seed(b * 3 + len(pre))
    h = (sample_scaled(g, b, n, 64) * 0.5).to(dev)
    inp, mot = (sample_scaled(g, b, n, 64) * 0.5).to(dev), (sample_scaled(g, b, n, 64, offset=-0.3) * 0.5).to(dev)
    wz, wr, wq = [(torch.randn(64, 192, generator=g) / 192 ** 0.5).to(dev) for _ in range(3)]
    bz, br, bq = [torch.randn(64, generator=g).to(dev) for _ in range(3)]
    res_zr = sample_scaled(g, b, n, 128).to(dev) if pre == 'bias+residual' else None
    res_q = sample_scaled(g, b, n, 64).to(dev) if pre == 'bias+residual' else None
    assert not tc_weights_resident(192, 128, gru=True)
    z, rh = torch.empty_like(h), torch.empty_like(h)
    ops.tc_linear([h, inp, mot], ops.tc_weights((wz, wr)), bz, bias2=br, epilogue=ops.TC_GRU_ZR, out=z, out2=rh, h=h, cout=64,
                  residual=res_zr)
    a = torch.cat([h, inp, mot], -1).double().reshape(m, 192)
    zr = a @ torch.cat([wz, wr]).double().t() + torch.cat([bz, br]).double()
    if res_zr is not None:
        zr = zr + res_zr.double().reshape(m, 128)
    z_ref = torch.sigmoid(zr[:, :64]).reshape(b, n, 64)
    rh_ref = torch.sigmoid(zr[:, 64:]).reshape(b, n, 64) * h.double()
    e_z, e_rh = per_sample_err(z, z_ref), per_sample_err(rh, rh_ref)
    out = torch.empty_like(h)
    ops.tc_linear([rh, inp, mot], ops.tc_weights(wq), bq, epilogue=ops.TC_GRU_Q, out=out, h=h, z=z, cout=64, residual=res_q)
    q = torch.cat([rh, inp, mot], -1).double().reshape(m, 192) @ wq.double().t() + bq.double()   # on the kernel's own r h and z
    if res_q is not None:
        q = q + res_q.double().reshape(m, 64)
    zd = z.double()
    h_ref = (1 - zd) * h.double() + zd * torch.tanh(q).reshape(b, n, 64)
    e_h = per_sample_err(out, h_ref)
    print(f'tc_linear GRU {pre} {rows}: z {e_z:.2e}, r*h {e_rh:.2e}, h\' {e_h:.2e}')
    assert e_z < 1e-5 and e_rh < 1e-5 and e_h < 1e-5, (e_z, e_rh, e_h)


@pytest.mark.parametrize('rows', ['mixed', 'bench'])
def test_tc_linear_flow_epilogue(dev, sm_count, rows):
    """FlowHead tail + RAFT update (model/update.py:71-72, RAFTSceneFlow.py:45-46): delta = w3 relu(W [lrelu(GN(z3)), net] + b)
    + b3, coords2 += delta in place (coords2_out aliases coords2), flow = coords2 - coords1."""
    from pvraft_b200 import ops
    b, n = ROWS[rows]
    assert_multi_tile(rows, b, n, sm_count)
    g = torch.Generator().manual_seed(17 + b)
    z3, net = sample_scaled(g, b, n, 64).to(dev), (sample_scaled(g, b, n, 64, offset=-0.2) * 0.5).to(dev)
    gamma, beta = torch.randn(64, generator=g).to(dev), (torch.randn(64, generator=g) * 0.2).to(dev)
    w = (torch.randn(64, 128, generator=g) / 128 ** 0.5).to(dev)
    bias = torch.randn(64, generator=g).to(dev)
    w3, b3 = (torch.randn(3, 64, generator=g) / 8).to(dev), torch.randn(3, generator=g).to(dev)
    c1 = (sample_scaled(g, b, n, 3) * 3).to(dev)
    c2_in = (c1 + torch.randn(b, n, 3, generator=g).to(dev) * 0.1).contiguous()
    stats, cnt = gn_stats(z3.double()), float(n * 8)
    a_in = torch.cat([gn_act_ref(z3.double(), None, stats, gamma, beta, cnt, 0.1), net.double()], -1).reshape(-1, 128)
    y = torch.relu(a_in @ w.double().t() + bias.double())
    delta_ref = (y @ w3.double().t() + b3.double()).reshape(b, n, 3)
    delta, coords2, flow = torch.empty_like(c1), c2_in.clone(), torch.empty_like(c1)
    ops.tc_linear([z3, net], ops.tc_weights(w), bias, in_stats=stats, in_gamma=gamma, in_beta=beta, in_count=cnt,
                  in_act=ops.ACT_LRELU, in_slope=0.1, epilogue=ops.TC_FLOW, out=delta, cout=64, w3=w3, b3=b3, coords1=c1,
                  coords2=coords2, coords2_out=coords2, flow_out=flow)
    err = per_sample_err(delta, delta_ref)
    print(f'tc_linear FLOW {rows}: delta err {err:.2e}')
    assert err < 1e-5, err
    assert torch.equal(coords2, c2_in + delta)              # fp32 coords2 + delta, in place
    assert torch.equal(flow, coords2 - c1)


@pytest.mark.parametrize('case', ['resident', 'streamed', 'flow'])
def test_tc_linear_settled_parameters_give_identical_bits(dev, case):
    """The first launch after a weight split (parameters read after griddepcontrol.wait) and the fourth (read before it)
    produce the same bits."""
    from pvraft_b200 import ops
    b, n = ROWS['mixed']
    g = torch.Generator().manual_seed(len(case))
    k = {'resident': 32, 'streamed': 512, 'flow': 128}[case]
    cout = 64 if case == 'flow' else 128
    x = sample_scaled(g, b, n, k).to(dev)
    gamma, beta = torch.randn(k, generator=g).to(dev), (torch.randn(k, generator=g) * 0.2).to(dev)
    bias = torch.randn(cout, generator=g).to(dev)
    w = (torch.randn(cout, k, generator=g) / k ** 0.5).to(dev)     # a fresh parameter: tc_weights splits it
    w3, b3 = (torch.randn(3, 64, generator=g) / 8).to(dev), torch.randn(3, generator=g).to(dev)
    c1 = sample_scaled(g, b, n, 3).to(dev)
    stats = gn_stats(x.double())
    assert tc_weights_resident(k, cout) == (case != 'streamed')
    tw = ops.tc_weights(w)
    outs, flags = [], []
    for _ in range(4):
        flags.append(0 if getattr(ops._TLS, 'unsettled', 0) else 1)
        if case == 'flow':
            out, c2o, fl = torch.empty_like(c1), torch.empty_like(c1), torch.empty_like(c1)
            ops.tc_linear([x[..., :64].contiguous(), x[..., 64:].contiguous()], tw, bias, in_stats=gn_stats(x[..., :64].double()),
                          in_gamma=gamma[:64], in_beta=beta[:64], in_count=float(n * 8), in_act=ops.ACT_LRELU, in_slope=0.1,
                          epilogue=ops.TC_FLOW, out=out, cout=64, w3=w3, b3=b3, coords1=c1, coords2=c1, coords2_out=c2o, flow_out=fl)
            outs.append(torch.cat([out, c2o, fl], -1))
        else:
            outs.append(ops.tc_linear([x], tw, bias, in_stats=stats, in_gamma=gamma, in_beta=beta, in_count=float(n * k // 8),
                                      in_act=ops.ACT_LRELU, in_slope=0.1))
    assert flags == [0, 0, 0, 1], flags
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0].view(torch.int32), outs[3].view(torch.int32))


# ----------------------------------------------------------------------------------------------------------------------
# corr_matmul (k_corr_gemm)
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('b,n', [(1, 1536), (3, 1024)])
@pytest.mark.parametrize('c', [32, 64, 96, 128, 256])
def test_corr_matmul_multi_tile_ctas(dev, sm_count, b, n, c):
    """1, 2, 3, 4 and 8 k-blocks through the 3-stage ring, with CTAs that run two tiles (B = 3: of two samples)."""
    from pvraft_b200 import ops
    tpb = (n // 128) ** 2
    n_tiles = b * tpb
    spanning = ctas_spanning_samples(n_tiles, min(n_tiles, sm_count), tpb)
    assert n_tiles > sm_count and (b == 1 or spanning > 0)
    g = torch.Generator().manual_seed(n + c)
    f1 = sample_scaled(g, b, n, c).to(dev)
    f2 = sample_scaled(g, b, n, c, offset=-0.2).to(dev)
    got = ops.corr_matmul(f1, f2)
    want = torch.matmul(f1.double(), f2.double().transpose(1, 2)) / math.sqrt(c)
    err = per_sample_err(got, want)
    print(f'corr_matmul B={b} N={n} C={c} ({n_tiles} tiles, {spanning} CTAs span samples): err {err:.2e}')
    assert err < 2e-6 * max(1, c / 128), err


def test_corr_matmul_bench_shape(dev, sm_count):
    """B=8, N=8192, C=128 (8192 tiles, 62-63 per CTA): every output element is written, and two rows of every 128-row band
    (one per consumer warpgroup) match float64 over all columns, i.e. every output tile is checked."""
    from pvraft_b200 import ops
    b, n, c = 8, 8192, 128
    assert b * (n // 128) ** 2 > sm_count
    g = torch.Generator().manual_seed(8192)
    f1 = sample_scaled(g, b, n, c).to(dev)
    f2 = sample_scaled(g, b, n, c, offset=-0.2).to(dev)
    got = ops.corr_matmul(f1, f2)
    assert bool(torch.isfinite(got).all()), 'an output tile was never written'
    band = torch.arange(0, n, 128)
    rows = torch.cat([band + torch.randint(0, 64, (n // 128,), generator=g), band + 64 + torch.randint(0, 64, (n // 128,), generator=g)])
    rows = rows.to(dev)
    want = torch.matmul(f1.double()[:, rows], f2.double().transpose(1, 2)) / math.sqrt(c)
    err = per_sample_err(got[:, rows], want)
    print(f'corr_matmul bench shape: err {err:.2e} over {rows.numel()} rows per sample')
    assert err < 2e-6, err
    del got


# ----------------------------------------------------------------------------------------------------------------------
# corr_lookup (k_corr_lookup<KPL, POW2, SMEM_TAB, HALF>)
# ----------------------------------------------------------------------------------------------------------------------
def lookup_warp_bytes(k):
    return ((max(k, 512) * 2 + k * 4 + 256 + 128 + 2 * 128 * 4 + 16) + 127) & ~127


def lookup_smem_table(n, k):
    """The host rule of launch_lookup: the sample's xyz table is staged in shared memory when it fits next to 8 warps."""
    return ((n * 16 + 127) & ~127) + 8 * lookup_warp_bytes(k) + (k + 1) * 8 + 8 <= SMEM_BUDGET


def lookup_grid(b, n, k, sm):
    avail = SMEM_BUDGET - (((n * 16 + 127) & ~127) if lookup_smem_table(n, k) else 0) - ((k + 1) * 8 + 8)
    warps = min(20, avail // lookup_warp_bytes(k))
    return min(sm, -(-(b * n) // warps)), warps


def make_block(state, xyz2, dev, levels, scale, state_dtype):
    from pvraft_b200 import CorrBlock
    cb = CorrBlock(num_levels=levels, base_scale=scale, truncate_k=state.truncated_corr.shape[-1]).to(dev)
    cb.state_dtype = state_dtype
    cb.set_state(state.truncated_corr.to(dev), state.indices.to(torch.int32).to(dev), xyz2.to(dev))
    return cb


def check_lookup(cb, out, coords, rows, levels, scale, moments=True):
    """The assertions of test_lookup_against_oracle on the rows `rows` of every sample (on the block's stored candidate
    order), plus whole-tensor invariants: every output row written, slots distinct and in range, moments of all rows."""
    b, n, k = cb.corr_val.shape
    r = rows.numel()
    assert r >= k or r == n   # (the oracle clamps cell counts at its number of rows)
    ids = cb.candidate_ids()[:, rows.to(cb.corr_val.device)]
    xyz = torch.gather(cb._xyz2, 1, ids.reshape(b, -1, 1).expand(b, r * k, 3)).reshape(b, r, k, 3)
    sub = O.CorrState(cb.corr_val.float()[:, rows.to(cb.corr_val.device)].cpu(), ids.cpu(), xyz.cpu())
    csub = coords[:, rows]
    vox_all = out['vox']
    assert bool(torch.isfinite(vox_all).all()) and bool((vox_all[..., levels * 27:] == 0).all())
    slots_all = out['knn_slot'].long()
    assert bool(((slots_all >= 0) & (slots_all < k)).all())
    s = slots_all.sort(-1).values
    assert bool((s[..., 1:] > s[..., :-1]).all()), 'duplicate neighbour slots'
    for lvl in range(levels):
        cube, valid = O.voxel_cube_index(sub, csub, scale * 2 ** lvl)
        got = out['cube'][:, rows.to(vox_all.device), :, lvl].cpu()
        assert torch.equal(got >= 0, valid), f'level {lvl}: validity differs'
        assert torch.equal(torch.where(got >= 0, got, torch.zeros_like(got)).long(), cube), f'level {lvl}: cell differs'
    want = O.voxel_means(sub, csub, levels, scale).transpose(1, 2)
    got = vox_all[:, rows.to(vox_all.device), :levels * 27].cpu()
    e_vox = rel_err(got, want)
    assert e_vox < 1e-6, e_vox
    assert (got != want).float().mean() < 1e-3, 'voxel means are expected to be (almost always) bit-identical'
    dist = O.knn_sqdist(sub, csub)
    want_slots = O.knn_select(sub, csub).sort(-1).values
    got_slots = slots_all[:, rows.to(vox_all.device)].cpu().sort(-1).values
    bad = (want_slots != got_slots).any(-1)
    if bad.any():
        assert torch.equal(torch.gather(dist, 2, want_slots).max(-1).values[bad], torch.gather(dist, 2, got_slots).max(-1).values[bad]), \
            'kNN sets differ beyond exact ties'
    sel = slots_all[:, rows.to(vox_all.device)].cpu()
    assert torch.equal(out['knn_sel'][:, rows.to(vox_all.device)].cpu(), O.knn_gather(sub, csub, sel).permute(0, 2, 3, 1))
    if moments:
        f = out['knn_sel'].double().reshape(b, -1, 4)
        m = out['moments']
        assert torch.allclose(m[:, :4], f.sum(1), rtol=1e-12, atol=1e-9)
        iu = torch.triu_indices(4, 4)
        second = torch.einsum('bni,bnj->bij', f, f)[:, iu[0], iu[1]]
        assert torch.allclose(m[:, 4:14], second, rtol=1e-12, atol=1e-9)
        assert torch.equal(m[:, 14].cpu(), torch.full((b,), float(n * 32), dtype=torch.float64))
    return e_vox


def lookup_rows(n, k, g):
    r = min(n, max(256, k))
    return torch.randperm(n, generator=g)[:r].sort().values


LOOKUP_CASES = [(k, scale, table, dtype) for k in (32, 64, 128, 256, 512, 1024) for scale in (0.25, 0.3) for table in ('smem', 'global')
                for dtype in ('fp32', 'bf16') if dtype == 'fp32' or k >= 128]


@pytest.mark.parametrize('k,scale,table,dtype', LOOKUP_CASES)
def test_lookup_every_instantiation(dev, sm_count, k, scale, table, dtype):
    """Every K x {power-of-two, other} base scale x {shared-memory, global} xyz table x {fp32, bf16 state}."""
    b, n, box = (2, max(512, k), 3.0) if table == 'smem' else (1, 16384, 12.0)
    assert lookup_smem_table(n, k) == (table == 'smem')
    state_dtype = torch.float32 if dtype == 'fp32' else torch.bfloat16
    state, coords, xyz2 = O.synthetic_state(b, n, k, seed=k + n + int(scale * 100), box=box)
    cb = make_block(state, xyz2, dev, 3, scale, state_dtype)
    out = cb.lookup(coords.to(dev), want_slots=True, want_cube=True)
    e = check_lookup(cb, out, coords, lookup_rows(n, k, torch.Generator().manual_seed(k)), 3, scale)
    print(f'lookup K={k} scale={scale} {table} table {dtype} (B={b}, N={n}): voxel means err {e:.2e}')


def test_lookup_static_split_without_moments(dev, sm_count):
    """moments = NULL: equal contiguous shares of B*N per CTA, warps claiming points from the CTA's counter (each CTA has
    more than 2 * warps points, so the counter is used); every row checked."""
    from pvraft_b200 import ops
    from pvraft_b200._lib import lib
    b, n, k, levels, scale = 2, 8192, 128, 3, 0.25
    grid, warps = lookup_grid(b, n, k, sm_count)
    assert b * n > grid * 2 * warps
    state, coords, xyz2 = O.synthetic_state(b, n, k, seed=5, box=8.0)
    cb = make_block(state, xyz2, dev, levels, scale, torch.float32)
    ld = (levels * 27 + 3) // 4 * 4
    cd = coords.to(dev).contiguous()
    vox = torch.empty(b, n, ld, dtype=torch.float32, device=dev)
    sel = torch.empty(b, n, 32, 4, dtype=torch.float32, device=dev)
    slots = torch.empty(b, n, 32, dtype=torch.int32, device=dev)
    cube = torch.empty(b, n, k, levels, dtype=torch.int8, device=dev)
    rc = lib().pvraft_corr_lookup_fwd(ops._p(cb.corr_val), ops._p(cb.corr_idx, torch.int32), ops._p(cb._xyz2p), ops._p(cd), b, n, n, k,
                                      levels, scale, ops._p(vox), ld, ops._p(sel), ops._p(slots, torch.int32), None,
                                      ops._p(cube, torch.int8), None, ops._stream())
    assert rc == 0
    out = dict(vox=vox, knn_sel=sel, knn_slot=slots, cube=cube)
    e = check_lookup(cb, out, coords, torch.arange(n), levels, scale, moments=False)
    print(f'lookup static split without moments ({grid} CTAs x {warps} warps): voxel means err {e:.2e}')


@pytest.mark.parametrize('b,n,k', [(150, 32, 32), (3, 2048, 256), (7, 1024, 128)])
def test_lookup_work_splits_with_moments(dev, sm_count, b, n, k):
    """B = 150 > CTAs: the static split with moments (CTA ranges straddle samples); B = 3, 7: per-sample dynamic claims."""
    grid, warps = lookup_grid(b, n, k, sm_count)
    static = grid < b
    assert static == (b == 150)
    state, coords, xyz2 = O.synthetic_state(b, n, k, seed=b + n, box=3.0)
    cb = make_block(state, xyz2, dev, 3, 0.25, torch.float32)
    out = cb.lookup(coords.to(dev), want_slots=True, want_cube=True)
    rows = torch.arange(n) if b * n <= 8192 else lookup_rows(n, k, torch.Generator().manual_seed(b))
    e = check_lookup(cb, out, coords, rows, 3, 0.25)
    print(f'lookup B={b} N={n} K={k} {"static" if static else "dynamic"} split ({grid} CTAs): voxel means err {e:.2e}')


def test_lookup_configs4_size(dev):
    """BASELINE configs[4]: N = 32768, K = 512 (global xyz table)."""
    b, n, k = 1, 32768, 512
    assert not lookup_smem_table(n, k)
    state, coords, xyz2 = O.synthetic_state(b, n, k, seed=32768, box=16.0)
    cb = make_block(state, xyz2, dev, 3, 0.25, torch.float32)
    out = cb.lookup(coords.to(dev), want_slots=True, want_cube=True)
    e = check_lookup(cb, out, coords, lookup_rows(n, k, torch.Generator().manual_seed(4)), 3, 0.25)
    print(f'lookup N={n} K={k}: voxel means err {e:.2e}')


# ----------------------------------------------------------------------------------------------------------------------
# kNN branch and trained weights
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


def knn_branch_case(dev, b, n, slope, host, seed):
    from pvraft_b200 import _lib, ops
    g = torch.Generator().manual_seed(seed)
    sel = sample_scaled(g, b, n, 32, 4).to(dev)
    w = (torch.randn(64, 4, generator=g) * 0.5).to(dev)
    bk = torch.randn(64, generator=g).to(dev)
    gamma, beta = (torch.randn(64, generator=g) * 0.5 + 0.3).to(dev), (torch.randn(64, generator=g) * 0.2).to(dev)
    preluk = torch.tensor([slope], dtype=torch.float32, device=dev)
    flow = sample_scaled(g, b, n, 3).to(dev)
    w_cf, b_cf = torch.randn(64, 3, generator=g).to(dev), torch.randn(64, generator=g).to(dev)
    mom = knn_moments(sel.double())
    kfeat, cflow = torch.empty(b, n, 64, device=dev), torch.empty(b, n, 64, device=dev)
    a = _lib.KnnBranchArgs()
    a.knn_sel, a.moments = ops._p(sel), ops._p(mom, torch.float64)
    a.w_knn, a.b_knn, a.gnk_gamma, a.gnk_beta, a.preluk = ops._p(w), ops._p(bk), ops._p(gamma), ops._p(beta), ops._p(preluk)
    a.preluk_host = slope if host == 'given' else float('nan')
    a.kfeat, a.flow, a.w_cf, a.b_cf, a.cflow = ops._p(kfeat), ops._p(flow), ops._p(w_cf), ops._p(b_cf), ops._p(cflow)
    a.B, a.N = b, n
    ops.knn_branch(a)
    return dict(sel=sel, w=w, bk=bk, gamma=gamma, beta=beta, flow=flow, w_cf=w_cf, b_cf=b_cf, kfeat=kfeat, cflow=cflow)


@pytest.mark.parametrize('host', ['given', 'nan'])
@pytest.mark.parametrize('slope', [-0.3, 0.25, 1.0, 1.7])
@pytest.mark.parametrize('b,n', [(3, 1000), (8, 8192)])
def test_knn_branch_against_fp64(dev, b, n, slope, host):
    """kfeat = max over the 32 candidates of PReLU(GroupNorm(knn_conv.0(f))) with the GroupNorm statistics of all N*32
    vectors; cflow = relu(conv_flow(flow)).  Slopes below 0, inside (0, 1], at 1 and above 1; the slope passed from the host
    or read back from the device (NaN)."""
    c = knn_branch_case(dev, b, n, slope, host, seed=n + int(slope * 10))
    per = []
    for s in range(b):   # (one sample at a time: [N,32,64] float64)
        t = c['sel'][s].double() @ c['w'].double().t() + c['bk'].double()
        tg = t.reshape(-1, 8, 8)
        mean, var = tg.mean((0, 2)), tg.var((0, 2), unbiased=False)
        tn = ((tg - mean.view(1, 8, 1)) * (var.view(1, 8, 1) + 1e-5).rsqrt()).reshape(t.shape) * c['gamma'].double() + c['beta'].double()
        per.append(torch.where(tn >= 0, tn, slope * tn).amax(1))
    want = torch.stack(per)
    err = per_sample_err(c['kfeat'], want)
    cflow_ref = torch.relu(c['flow'].double() @ c['w_cf'].double().t() + c['b_cf'].double())
    e_cf = per_sample_err(c['cflow'], cflow_ref)
    print(f'knn_branch B={b} N={n} slope={slope} ({host}): kfeat err {err:.2e}, cflow err {e_cf:.2e}')
    assert err < 1e-5, err
    assert e_cf < 1e-6, e_cf


def test_knn_branch_instantiation_follows_the_slope(dev):
    """A slope above 1 runs the per-candidate instantiation, any other the max/min shortcut.  For a positive slope PReLU is
    monotone, so both give the same bits and only the launched kernel shows which one ran."""
    from torch.profiler import ProfilerActivity, profile
    seen = {}
    for slope in (-0.3, 1.0, 1.7):
        for host in ('given', 'nan'):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                knn_branch_case(dev, 2, 256, slope, host, seed=1)
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if 'k_knn_branch' in e.name]
            if not any(e.device_type == torch.autograd.DeviceType.CUDA for e in prof.events()):
                pytest.skip('the profiler records no device activity here')
            seen[(slope, host)] = names
            want = ('<false>', 'ILb0E') if slope > 1 else ('<true>', 'ILb1E')    # demangled or mangled name
            assert names and all(any(w in nm for w in want) for nm in names), (slope, host, names)
    print('knn_branch kernels by slope:', seen)


@pytest.mark.parametrize('slopes', [(-0.3, 1.7), (1.7, -0.3)])
@pytest.mark.parametrize('n', [1024, 1000])
def test_trained_weights_teacher_forced_loop(dev, n, slopes):
    """The RAFT loop's kernels with trained-looking weights on oracle-produced state, iteration by iteration: N = 1024 runs the
    tensor-core path (kNN branch kernel, wgmma layers with the PReLU slope in the prologue), N = 1000 the CUDA-core kernels."""
    from pvraft_b200 import RSF, Graph, ops
    b, k, iters = 2, 512, 3
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    m = RSF(args)
    m.load_state_dict(default_weights(args=args), strict=True)
    randomise_affine(m, 7, slopes)
    W = {key: v.detach().clone() for key, v in m.state_dict().items()}
    m = m.to(dev).eval()
    pc1, pc2 = O.synthetic_clouds(b, n, seed=n + 3)
    with torch.no_grad():
        li = O.prepare(W, pc1, pc2, k)
        trace = []
        O.raft_loop(W, li, pc1, iters, 3, 0.25, trace)
    assert any((W[key] < 0).any() for key in W if '.gn' in key and key.endswith('weight'))
    m.corr_block.set_state(li.state.truncated_corr.to(dev), li.state.indices.to(dev), pc2.to(dev))
    og = li.graph
    nbr = (og.edges.reshape(b, n, 32) - (torch.arange(b) * n).view(b, 1, 1)).to(torch.int32)
    graph = Graph(nbr.to(dev), og.edge_feats.reshape(b, n, 32, 3).to(dev).contiguous(), 32, [b * n, b * n])
    pc1d = pc1.to(dev)
    inp = li.inp.transpose(1, 2).contiguous().to(dev)
    net = li.net.transpose(1, 2).contiguous().to(dev)
    me = m.update_block.motion_encoder
    worst = dict(corr=0.0, motion=0.0, net=0.0, delta=0.0)
    with torch.no_grad():
        for it, t in enumerate(trace):
            coords = t['coords'].to(dev).contiguous()
            flow = (coords - pc1d).contiguous()
            if ops.tc_supported(n):
                corr_pm, motion_c = m.corr_block.feature_motion_tc(coords, flow, me, need_corr=True)
                _, motion = m.corr_block.feature_motion_tc(coords, flow, me, need_corr=False)     # what the loop runs
                assert per_sample_err(motion, motion_c) < 2e-5
            else:
                motion = torch.empty(b, n, 64, dtype=torch.float32, device=dev)

                def attach(a, keep, flow=flow, motion=motion):
                    me.fill(a, flow)
                    a.motion = ops._p(motion)
                    keep.append(motion)

                corr_pm, _ = m.corr_block.feature_point_major(coords, motion_args=attach)
            want_motion = O.motion_encoder(W, t['coords'] - pc1, t['corr'], 'update_block.motion_encoder')
            errs = dict(corr=per_sample_err(corr_pm.transpose(1, 2), t['corr']),
                        motion=per_sample_err(motion.transpose(1, 2), want_motion))
            net_new, delta = m.update_block.forward_pm(net, inp, motion, graph)
            errs.update(net=per_sample_err(net_new.transpose(1, 2), t['net']), delta=per_sample_err(delta, t['delta']))
            for key, e in errs.items():
                worst[key] = max(worst[key], e)
            assert errs['corr'] < 1e-5 and errs['motion'] < 2e-5 and errs['net'] < 2e-5 and errs['delta'] < 5e-5, (it, errs)
            net = t['net'].transpose(1, 2).contiguous().to(dev)
    print(f'trained-weight loop N={n} slopes (out_conv, knn_conv)={slopes}: worst per-sample err', {k: f'{v:.2e}' for k, v in worst.items()})


# ----------------------------------------------------------------------------------------------------------------------
# corr_topk at the configs[4] sizes
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('k', [1, 512, 1024])
@pytest.mark.parametrize('m', [16384, 32768, 49152])
def test_corr_topk_large_rows(dev, m, k):
    """Rows of up to 49152 columns (202 KB staged in shared memory), with ties; the last row is constant."""
    from pvraft_b200 import ops
    g = torch.Generator().manual_seed(m + k)
    corr = torch.randn(2, 3, m, generator=g)
    corr[:, :, ::7] = corr[:, :, 3:4]            # plenty of exact ties
    corr[1, 2] = 0.5
    val, idx = ops.corr_topk(corr.to(dev), k)
    top = torch.topk(corr, k, dim=2, sorted=True)
    assert torch.equal(val.cpu().sort(-1, descending=True).values, top.values)
    assert torch.equal(torch.gather(corr, 2, idx.cpu().long()), val.cpu())
    assert (idx.cpu()[..., 1:] > idx.cpu()[..., :-1]).all()
    assert torch.equal(idx.cpu()[1, 2].long(), torch.arange(k))      # all ties: the lowest columns win


def test_corr_topk_refuses_rows_beyond_the_staging_limit():
    """M = 49153 is refused before anything is launched (the pointers are never dereferenced)."""
    from pvraft_b200._lib import lib
    rc = lib().pvraft_corr_topk_fwd(16, 1, 1, 49153, 512, 16, 16, None)
    assert rc == -2 and b'49153' in lib().pvraft_last_error_string()
    assert lib().pvraft_corr_topk_fwd(16, 1, 1, 49152, 1025, 16, 16, None) == -2


# ----------------------------------------------------------------------------------------------------------------------
# SetConv edge kernel at the bench batch
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('c', [32, 64, 128])
def test_setconv_edge_bench_batch(dev, c):
    """y = P_j - P_i + W_e (x_j - x_i) over the 32 neighbours -> per-channel max / min and GroupNorm sums, B = 8, N = 8192, with
    and without the Morton processing order (which must change no bit of ymax / ymin)."""
    from pvraft_b200 import ops
    b, n, cin = 8, 8192, 64
    g = torch.Generator().manual_seed(c)
    pc, _ = O.synthetic_clouds(b, n, seed=c)
    pcd = pc.to(dev)
    nbr, rel = ops.knn(pcd, pcd, 32, mode=0, want_rel=True)
    order = ops.point_order(pcd)
    P = sample_scaled(g, b, n, c).to(dev)
    w = torch.randn(c, cin + 3, generator=g).to(dev)
    res = {}
    for name, o in (('plain', None), ('order', order)):
        stats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
        ymax, ymin = ops.setconv_edge(P, nbr, rel, w, cin, stats, order=o)
        res[name] = (ymax, ymin, stats)
    we = w[:, cin:].double()
    e_max = e_min = e_st = 0.0
    for s in range(b):   # float64 reference one sample at a time ([N,32,C])
        p = P[s].double()
        y = p[nbr[s].long()] - p.unsqueeze(1) + rel[s].double() @ we.t()
        ys = y.reshape(n * 32, 8, c // 8)
        s1, s2, sabs = ys.sum((0, 2)), (ys ** 2).sum((0, 2)), ys.abs().sum((0, 2))
        ymax, ymin, stats = res['plain']
        e_max = max(e_max, per_sample_err(ymax[s:s + 1], y.amax(1)[None]))
        e_min = max(e_min, per_sample_err(ymin[s:s + 1], y.amin(1)[None]))
        assert bool(((stats[s, :, 0] - s1).abs() <= 1e-5 * s1.abs() + 1e-7 * sabs).all()), (stats[s, :, 0], s1)
        assert bool(((stats[s, :, 1] - s2).abs() <= 1e-5 * s2).all()), (stats[s, :, 1], s2)
        e_st = max(e_st, float(((stats[s, :, 0] - s1).abs() / sabs).max()), float(((stats[s, :, 1] - s2).abs() / s2).max()))
        d = (res['order'][2][s] - stats[s]).abs()
        assert bool((d[:, 0] <= 1e-12 * sabs).all() and (d[:, 1] <= 1e-12 * s2).all()), d
    print(f'setconv_edge C={c}: ymax err {e_max:.2e}, ymin err {e_min:.2e}, stats err (relative to the sum of |y|) {e_st:.2e}')
    assert e_max < 1e-6 and e_min < 1e-6, (e_max, e_min)
    assert torch.equal(res['order'][0], res['plain'][0]) and torch.equal(res['order'][1], res['plain'][1])


# ----------------------------------------------------------------------------------------------------------------------
# remaining gradient instantiations
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('k', [512, 1024])
@pytest.mark.parametrize('c', [32, 256])
def test_corr_init_backward_channel_widths(dev, c, k):
    """d fmap1 = G fmap2 / sqrt(C), d fmap2 = G^T fmap1 / sqrt(C) with G the sparse [N,N] gradient of the kept entries."""
    from pvraft_b200 import ops
    b, n = 2, 1024
    g = torch.Generator().manual_seed(c + k)
    f1, f2 = sample_scaled(g, b, n, c).to(dev), sample_scaled(g, b, n, c, offset=-0.2).to(dev)
    idx = torch.rand(b, n, n, generator=g).argsort(-1)[..., :k]
    gv = torch.randn(b, n, k, generator=g)
    d1, d2 = ops.corr_init_bwd(gv.to(dev), idx.to(torch.int32).to(dev), f1, f2)
    G = torch.zeros(b, n, n, dtype=torch.float64).scatter_(2, idx, gv.double()).to(dev)
    want1 = G @ f2.double() / math.sqrt(c)
    want2 = G.transpose(1, 2) @ f1.double() / math.sqrt(c)
    e1, e2 = per_sample_err(d1, want1), per_sample_err(d2, want2)
    print(f'corr_init_bwd C={c} K={k}: d fmap1 err {e1:.2e}, d fmap2 err {e2:.2e}')
    assert e1 < 2e-5 and e2 < 2e-5, (e1, e2)


@pytest.mark.parametrize('c', [32, 64, 128])
def test_edge_forward_backward_widths(dev, c):
    """T = P[nbr] - P + E in place with GroupNorm sums; dP[nbr] += dT, dP -= sum_j dT."""
    from pvraft_b200 import ops
    b, n = 2, 1000
    g = torch.Generator().manual_seed(c)
    p, e = sample_scaled(g, b, n, c), sample_scaled(g, b, n * 32, c, offset=-0.2)
    nbr = torch.randint(0, n, (b, n, 32), generator=g)
    dt = torch.randn(b, n * 32, c, generator=g)
    stats = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev)
    t = ops.edge_fwd(p.to(dev), nbr.to(torch.int32).to(dev), e.to(dev).contiguous(), stats)
    dp = ops.edge_bwd(dt.to(dev), nbr.to(torch.int32).to(dev), torch.zeros(b, n, c, device=dev))
    pd = p.double()
    want = (torch.gather(pd.unsqueeze(1).expand(b, n, n, c), 2, nbr.unsqueeze(-1).expand(b, n, 32, c)) - pd.unsqueeze(2)
            + e.double().view(b, n, 32, c))
    dtv = dt.double().view(b, n, 32, c)
    want_dp = -dtv.sum(2)
    for s in range(b):
        want_dp[s].index_add_(0, nbr[s].reshape(-1), dtv[s].reshape(-1, c))
    e_t, e_dp = per_sample_err(t.view(b, n, 32, c), want), per_sample_err(dp, want_dp)
    e_st = check_out_stats(stats, t)
    print(f'edge C={c}: forward err {e_t:.2e}, stats {e_st:.2e}, backward err {e_dp:.2e}')
    assert e_t < 1e-6 and e_dp < 1e-5, (e_t, e_dp)
