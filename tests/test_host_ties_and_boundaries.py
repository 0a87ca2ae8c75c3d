"""The restatements of tests/ties_restated.py checked on the CPU: the pre-test threshold, the cell codes, the lookup's
32-NN tie rule and slot map, the exact fp32 fma and the graph distance against exact rational arithmetic, and that the
boundary generators reach the decisions they are written for."""
import fractions
import math

import numpy as np
import pytest
import torch

import ties_restated as R
from oracle import pvraft_oracle as O

F32 = np.float32
SCALES = [0.1, 0.2, 0.25, 0.3, 0.45, 0.7, float(F32(1 / 3))]


@pytest.mark.parametrize('base', SCALES)
def test_cube_threshold(base):
    """fl(t / r) >= 1.5 > fl(prev(t) / r) at every level's scale; t == 1.5 r for powers of two."""
    for r in R.level_scales(base, 4):
        t = R.cube_threshold(r)
        assert R.quotient(t, r) >= F32(1.5) > R.quotient(np.nextafter(t, F32(0)), r)
        if R.is_pow2(r):
            assert t == F32(1.5) * r
    # 0.45 is a scale where t lies one float above fl(1.5 r): a threshold of fl(1.5 r) would drop valid candidates there
    r = R.level_scales(0.45, 1)[0]
    assert R.cube_threshold(r) == np.nextafter(F32(1.5) * r, F32(np.inf))
    assert R.quotient(F32(1.5) * r, r) < F32(1.5)


def test_cube_threshold_equals_the_cell_test():
    """max|d| < t  <=>  every axis' cell is in {-1, 0, 1}, on every float in a window around each threshold."""
    for base in SCALES:
        r = R.level_scales(base, 3)[-1]
        t = R.cube_threshold(r)
        d = t + (np.arange(-64, 65) * np.spacing(t)).astype(F32)
        assert np.array_equal(np.abs(d) < t, np.abs(np.rint(R.quotient(d, r))) <= 1)
        assert np.array_equal(np.abs(-d) < t, np.abs(np.rint(R.quotient(-d, r))) <= 1)


@pytest.mark.parametrize('base,levels', [(0.25, 3), (0.125, 4), (0.5, 1), (0.3, 3), (0.1, 3), (0.7, 2), (1 / 3, 3), (0.45, 3)])
def test_cells_match_the_oracle(base, levels):
    """The restated cells equal O.voxel_cube_index (torch-CPU division) on every boundary candidate, and the pre-test
    never disagrees with the coarsest cube."""
    for kind in ('lattice', 'boundary'):
        c = R.make_case(kind, base, levels, 128, 64, seed=levels)
        cells = R.lookup_cells(c['cand'], c['coords'], base, levels)
        st = O.CorrState(torch.from_numpy(c['val']), torch.from_numpy(c['idx']), torch.from_numpy(c['cand']))
        for lvl in range(levels):
            cube, valid = O.voxel_cube_index(st, torch.from_numpy(c['coords']), float(R.level_scales(base, levels)[lvl]))
            assert np.array_equal(cells[..., lvl] >= 0, valid.numpy()), (kind, lvl)
            assert np.array_equal(np.maximum(cells[..., lvl], 0), cube.numpy()), (kind, lvl)
        d = R.offsets(c['cand'], c['coords'])
        assert np.array_equal(np.abs(d).max(-1) < R.cube_threshold(R.level_scales(base, levels)[-1]),
                              R.cell_codes(d, R.level_scales(base, levels)[-1]) >= 0)


def test_round_half_even_decides_on_the_lattice():
    """On the power-of-two lattice quotients of exactly +-0.5 occur, where rint and round disagree."""
    c = R.make_case('lattice', 0.25, 3, 128, 32, seed=1)
    d = R.offsets(c['cand'], c['coords'])
    q = R.quotient(d, F32(0.25))
    half = np.abs(q) == F32(0.5)
    assert half.sum() > 100
    assert (np.rint(q[half]) == 0).all() and (np.abs(np.trunc(q[half] + np.copysign(F32(0.5), q[half]))) == 1).all()


@pytest.mark.parametrize('k', [32, 64, 128, 256, 512, 1024])
def test_slot_map_is_a_permutation(k):
    m = R.slot_map(k)
    assert m.shape == (32, k // 32) and np.array_equal(np.sort(m.reshape(-1)), np.arange(k))
    if k <= 128:   # one block of 32*VEC slots: (lane, e) order is slot order
        assert np.array_equal(m.reshape(-1), np.arange(k))


@pytest.mark.parametrize('k', [32, 128, 256, 512, 1024])
def test_knn_select_rule(k):
    """The kernel's rule picks the 32 nearest.  On rows whose 32nd distance ties it equals the lowest-slot rule for
    K <= 128 and differs from it for K >= 256 (at K = 512 a tie between slot 4, lane 1 e 0, and slot 128, lane 0 e 4,
    goes to slot 128)."""
    rng = np.random.default_rng(k)
    dist = rng.integers(0, 6, (400, k)).astype(F32)    # heavy exact ties
    got = R.lookup_knn_select(dist)
    assert all(len(set(r)) == R.KNN for r in got.tolist())
    kth = np.sort(dist, -1)[:, R.KNN - 1]
    assert (np.take_along_axis(dist, got, -1).max(-1) == kth).all()
    low = R.lowest_slot_select(dist)
    same = (np.sort(got, -1) == low).all(-1)
    if k <= 128:
        assert same.all()
    else:
        assert (~same).sum() > 50
    if k == 512:
        d = np.full((1, k), 9.0, F32)
        d[0, [s for s in range(k) if s not in (4, 128)][:31]] = 1.0
        d[0, 4] = d[0, 128] = 2.0
        assert 128 in R.lookup_knn_select(d)[0] and 4 not in R.lookup_knn_select(d)[0]
        assert 4 in R.lowest_slot_select(d)[0]
    # without a tie at the 32nd place the order is (lane, e) over all 32
    dist = rng.permutation(k)[None, :].astype(F32)
    order = R.slot_map(k).reshape(-1)
    assert np.array_equal(R.lookup_knn_select(dist)[0], order[dist[0, order] < R.KNN])


# ------------------------------------------------------------------------------------------------------------------------
# exact rational reference of fp32 rounding
# ------------------------------------------------------------------------------------------------------------------------
def round32(x):
    """Fraction -> the nearest float32 (ties to even), exactly."""
    if x == 0:
        return F32(0.0)
    s = -1 if x < 0 else 1
    a = abs(x)
    e = math.floor(math.log2(a.numerator) - math.log2(a.denominator))
    while fractions.Fraction(2) ** e > a:
        e -= 1
    while fractions.Fraction(2) ** (e + 1) <= a:
        e += 1
    e = max(e, -126)
    m = a / fractions.Fraction(2) ** (e - 23)
    n = math.floor(m)
    rem = m - n
    if rem > fractions.Fraction(1, 2) or (rem == fractions.Fraction(1, 2) and n % 2 == 1):
        n += 1
    return F32(s * float(fractions.Fraction(n) * fractions.Fraction(2) ** (e - 23)))


def Fr(x):
    return fractions.Fraction(float(x))


def fma_triples(rng, n):
    """Random triples, and adversarial ones: a*b + c lands exactly on or next to a float32 midpoint after the double
    rounding of the product-sum."""
    a = rng.standard_normal(n).astype(F32) * F32(7)
    b = rng.standard_normal(n).astype(F32) * F32(3)
    c = rng.standard_normal(n).astype(F32)
    out = [(a, b, c)]
    # c = -(a*b rounded to fp32) + a tiny part: the sum is the product's rounding error, then the tiny part decides
    p = (a.astype(np.float64) * b.astype(np.float64))
    c2 = (-p).astype(F32)
    out.append((a, b, c2))
    # (1 + i 2^-12)(1 + j 2^-12) with ij odd is a float32 midpoint; a c far below double precision decides the rounding,
    # which a double-rounded product-sum loses
    a3 = (1 + rng.integers(0, 2 ** 9, n) * 2.0 ** -12).astype(F32)
    b3 = (1 + rng.integers(0, 2 ** 9, n) * 2.0 ** -12).astype(F32)
    c3 = (np.ldexp(rng.integers(1, 2 ** 10, n).astype(np.float64), -75) * rng.choice([-1, 1], n)).astype(F32)
    out.append((a3, b3, c3))
    c4 = (np.ldexp(np.ones(n), -24) + np.ldexp(rng.integers(-3, 4, n).astype(np.float64), -50)).astype(F32)
    out.append((a3, b3, c4))
    return out


def test_fma32_is_exact():
    rng = np.random.default_rng(0)
    hits = 0
    for a, b, c in fma_triples(rng, 3000):
        got = R.fma32(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(c)).numpy()
        want = np.array([round32(Fr(x) * Fr(y) + Fr(z)) for x, y, z in zip(a, b, c)], F32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)
        hits += int((naive != want).sum())
    print(f'fma32: exact on {4 * 3000} triples; the double-rounded product-sum is wrong on {hits} of them')
    assert hits > 0, 'the adversarial triples no longer reach a double-rounding case'


def exact_distance(q, p, mode):
    """One (query, point) distance with every op rounded to fp32 by exact rational arithmetic."""
    qf, pf = [Fr(v) for v in q], [Fr(v) for v in p]
    r = lambda x: Fr(round32(x))   # noqa: E731
    dot = r(qf[2] * pf[2] + r(qf[1] * pf[1] + r(qf[0] * pf[0])))
    qn = r(r(r(qf[0] * qf[0]) + r(qf[1] * qf[1])) + r(qf[2] * qf[2]))
    pn = r(r(r(pf[0] * pf[0]) + r(pf[1] * pf[1])) + r(pf[2] * pf[2]))
    if mode == 0:
        return round32(r(qn + pn) - 2 * dot)
    return round32(r(-2 * dot + qn) + pn)


@pytest.mark.parametrize('mode', [0, 1])
def test_graph_distance_against_rationals(mode):
    rng = np.random.default_rng(mode)
    q = (rng.uniform(-60, 60, (12, 3))).astype(F32)
    p = np.concatenate([rng.uniform(-60, 60, (40, 3)), q[:4] + rng.normal(0, 1e-3, (4, 3)), q[4:8],
                        np.round(rng.uniform(-60, 60, (20, 3)) * 16) / 16]).astype(F32)
    q = np.concatenate([q, np.round(q * 16) / 16]).astype(F32)
    got = R.graph_distance(torch.from_numpy(q), torch.from_numpy(p), mode).numpy()
    want = np.array([[exact_distance(a, b, mode) for b in p] for a in q], F32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_graph_ranking_is_distance_then_id():
    """Quantised and duplicated clouds: the restated ranking is a stable sort on (distance, id)."""
    g = torch.Generator().manual_seed(0)
    x = torch.round(torch.rand(300, 3, generator=g) * 16 * 8) / 16
    x[200:] = x[:100]
    for mode in (0, 1):
        ids, rel = R.knn_graph(x, x, 32, mode)
        d = R.graph_distance(x, x, mode)
        dd = torch.gather(d, 1, ids)
        assert bool((dd[:, 1:] >= dd[:, :-1]).all())
        tie = dd[:, 1:] == dd[:, :-1]
        assert bool((ids[:, 1:][tie] > ids[:, :-1][tie]).all()) and int(tie.sum()) > 1000
        assert torch.equal(rel, x[ids] - x[:, None])


# ------------------------------------------------------------------------------------------------------------------------
# generators
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('base,levels', [(0.25, 3), (0.125, 4), (0.5, 1)])
def test_lattice_cases_reach_every_half(base, levels):
    c = R.make_case('lattice', base, levels, 512, 64, seed=3)
    n = R.boundary_classes(c['cand'], c['coords'], c['intended'], base, levels)
    print(f'lattice {base} x {levels}: {n}')
    assert n['exact_offset'] == c['idx'].size   # every sum centre + offset is exact
    for lvl in range(levels):
        for h in (0.5, 1.5, 2.5):
            assert n[f'l{lvl}_q=={h}'] > 0, (lvl, h)
    assert n['max|d|==thr'] > 0


@pytest.mark.parametrize('base', [0.3, 0.1, 0.7, 1 / 3, 0.45])
def test_boundary_cases_reach_every_crossing(base):
    levels = 3
    c = R.make_case('boundary', base, levels, 512, 64, seed=4)
    n = R.boundary_classes(c['cand'], c['coords'], c['intended'], base, levels)
    print(f'boundary {base:.4f} x {levels}: {n}')
    exact = R.make_case('boundary', base, levels, 512, 64, seed=4, centres=[(0.0, 0.0, 0.0)])
    assert (R.offsets(exact['cand'], exact['coords']).astype(np.float64) == exact['intended']).all()
    for lvl in range(levels):
        for h in (0.5, 1.5):
            assert n[f'l{lvl}_at({h})'] > 0 and n[f'l{lvl}_below({h})'] > 0, (lvl, h)
    assert n['max|d|==thr'] > 0 and n['max|d|==prev(thr)'] > 0 and n['max|d|==next(thr)'] > 0
    # the centres near 35 and 1e3 move the offsets onto their own coarser grid
    assert n['exact_offset'] < c['idx'].size


def test_tie_pools():
    c = R.make_case('duplicate', 0.25, 3, 128, 10, seed=5)
    d = R.knn_sqdist(c['cand'], c['coords'])[0]
    assert ((d == 0).sum(-1) == 40).all()
    c = R.make_case('cluster_far', 0.25, 3, 512, 10, seed=6)
    d = R.knn_sqdist(c['cand'], c['coords'])[0]
    assert ((d < 3e-4).sum(-1) == 40).all() and (np.sort(d, -1)[:, 40] >= 100).all()
    # the 32nd distance lies more than 4 octaves (in the bit pattern: 2^25) below the largest lane minimum
    k = 512
    lane_min = d[:, R.slot_map(k)].min(-1).max(-1)
    kth = np.sort(d, -1)[:, 31]
    assert (lane_min.view(np.uint32) - kth.view(np.uint32) > 0x01FFFFFF).all()
