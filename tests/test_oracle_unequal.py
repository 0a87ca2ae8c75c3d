"""Pin the CPU oracle on pairs of clouds of different sizes against unequal_rsf.npz, produced by the unmodified reference
modules with a truncated state of N1 rows (tests/golden/make_golden_unequal.py).  CPU only; the tolerances are those of
test_oracle_golden.py."""
import pytest
import torch

import unequal_oracle as U
from conftest import load_golden, rel_err
from oracle import pvraft_oracle as O

TOL = 2e-5
CASES = ['a', 'b', 'c']   # (N1, N2) = (256, 384), (384, 256) at B = 2, K = 64; (100, 300) at B = 1, K = 128


@pytest.fixture(scope='module')
def golden():
    arr, W1 = load_golden('unequal_rsf.npz')
    return arr, U.golden_weights(arr, W1)


def case(arr, c):
    b, n1, n2, k, levels, iters, s = [int(v) for v in arr[f'{c}/meta']]
    return dict(b=b, n1=n1, n2=n2, k=k, levels=levels, iters=iters, s=s, bs=float(arr['base_scale']),
                get=lambda key: arr[f'{c}/{key}'])


def test_teacher_forced_lookup(golden):
    arr, W = golden
    q = case(arr, 'c')
    g = q['get']
    st = U.golden_state(q['get'])
    assert st.truncated_corr.shape == (q['b'], q['n1'], q['k'])
    for it, coords in enumerate((g('pc1'), g('it1/coords'))):
        vox = O.voxel_feature(W, st, coords, q['levels'], q['bs'])
        assert rel_err(vox[..., :q['s']], g(f'it{it}/voxel_feature')) < TOL
        corr = O.corr_lookup(W, st, coords, q['levels'], q['bs'])
        assert rel_err(corr[..., :q['s']], g(f'it{it}/corr')) < TOL


def test_indices_bit_exact(golden):
    arr, _ = golden
    q = case(arr, 'c')
    g = q['get']
    st = U.golden_state(q['get'])
    coords = g('it1/coords')
    for lvl in range(q['levels']):
        cube, valid = O.voxel_cube_index(st, coords, q['bs'] * 2 ** lvl)
        assert torch.equal(cube.to(torch.int8), g(f'it1/cube_idx_l{lvl}'))
        assert torch.equal(valid, g(f'it1/valid_l{lvl}'))
    slots = O.knn_select(st, coords)
    assert torch.equal(slots.sort(-1).values, g('it1/knn_slots').long().sort(-1).values)


def test_the_compact_case_reaches_the_count_clamp(golden):
    """Case c: some cell holds more candidates than there are query points (N1 = 100 < count <= K = 128 <= N2), so the
    mean divides by N1 rather than by the count -- in the golden itself, and in the oracle."""
    arr, W = golden
    q = case(arr, 'c')
    g = q['get']
    st = U.golden_state(q['get'])
    assert q['n1'] < q['k'] <= q['n2']
    reached = 0
    for coords in (g('pc1'), g('it1/coords')):
        for lvl in range(q['levels']):
            cube, valid = O.voxel_cube_index(st, coords, q['bs'] * 2 ** lvl)
            reached += int((torch.zeros(q['b'], q['n1'], 27).scatter_add_(2, cube, valid.float()) > q['n1']).sum())
    assert reached > 0
    # the clamp matters: dividing by the raw count gives other means at the coarsest level
    coords = g('pc1')
    got = O.voxel_means(st, coords, q['levels'], q['bs'])
    cube, valid = O.voxel_cube_index(st, coords, q['bs'] * 4)
    s = torch.zeros(q['b'], q['n1'], 27).scatter_add_(2, cube, st.truncated_corr * valid)
    cnt = torch.zeros(q['b'], q['n1'], 27).scatter_add_(2, cube, valid.float())
    assert not torch.allclose(got[:, 54:], (s / cnt.clamp_min(1)).transpose(1, 2), rtol=1e-3)


@pytest.mark.parametrize('c', CASES)
def test_encoder_corr_init_and_free_running(golden, c):
    arr, W = golden
    q = case(arr, c)
    g = q['get']
    pc1, pc2 = g('pc1'), g('pc2')
    li = U.prepare(W, pc1, pc2, q['k'])
    assert li.state.truncated_corr.shape == (q['b'], q['n1'], q['k'])
    cs = g('truncated_corr_checksum')
    assert abs(float(li.state.truncated_corr.double().sum()) - float(cs[0])) < 1e-6 * float(cs[1])
    if c == 'c':
        assert rel_err(li.state.truncated_corr, g('truncated_corr')) < TOL
        assert (li.state.indices.sort(-1).values != g('cand').long().sort(-1).values).any(-1).float().mean() <= 0.01
    trace = []
    flows = O.raft_loop(W, li, pc1, q['iters'], q['levels'], q['bs'], trace)
    for it in range(q['iters']):
        assert flows[it].shape == (q['b'], q['n1'], 3)
        assert rel_err(flows[it], g(f'it{it}/flow')) < 1e-4
        assert rel_err(trace[it]['corr'][..., :q['s']], g(f'it{it}/corr')) < 1e-4
        assert rel_err(trace[it]['net'][..., :q['s']], g(f'it{it}/net')) < 1e-4
    if c == 'a':
        refined = O.flot_refine(W, 'refine_block', flows[-1], li.feat_graph)
        assert rel_err(refined, g('refined')) < 1e-4
