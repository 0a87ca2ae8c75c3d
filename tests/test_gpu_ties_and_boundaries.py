"""The index-deciding kernels at the inputs where their rules decide: exact rounding boundaries and exact distance ties.

* k_corr_lookup: every candidate's cell (dbg_cube) bit-exact against the numpy float32 restatement of tests/ties_restated.py
  and against O.voxel_cube_index; the voxel means bit-identical to O.voxel_means; the 32 kNN
  slots in the kernel's exact order (the restated tie rule, no tie exemption), the gathered 4-vectors bitwise, the moments
  as test_gpu_parity.  Inputs: power-of-two scales on a lattice of step r0/4 (every quotient a multiple of 1/4: +-0.5, +-1.5,
  +-2.5 at every level), other scales at the floats where fl(d / r) reaches 0.5, passes 0.5 and reaches 1.5, at +-thr_c, and their
  neighbours, query centres near 0, 35 and 1e3; rows with 40 duplicates of the query (distance 0) and rows with 40
  candidates within 1 cm and the rest 10-60 m away.  Every K in {32, 128, 512, 1024}, shared-memory and global tables,
  fp32 and bf16 state; the DET form equals the default form.
* k_lookup_bwd: d_corr against a float64 gradient over the restated fp32 cells (no re-decision in float64).
* k_knn / k_knn_grid: ops.knn in modes 0 and 1, k in {16, 32}, at N = 40 (brute force), 4096 and 16 384 (shared-memory
  grid) and 20 000 (counting-sort grid) on a LiDAR-like cloud at KITTI extents, continuous, quantised to 1/16 m and with
  10 % duplicated points: ids in the exact (distance, id) order of the restated expanded distance, rel bitwise.
* The model on LiDAR-like scenes (the LiDAR-like cloud as pc1; pc2 = ego-motion + two moved objects + 1 cm noise;
  continuous, quantised to 1/16 m, duplicated points), with the oracle's kNN select following the kernel's tie rule:
  RSF teacher-forced per iteration and free-running at B = 2, N = 8192, K = 512 (tensor-core loop) and N = 4999, K = 256
  (CUDA-core kernels); RSF_refine free-running; a stage-1 training step's 95 parameter and 2 input gradients.

Worst errors and the boundary-class counts are printed (-s)."""
import contextlib
import math
import types

import numpy as np
import pytest
import torch

import ties_restated as R
from conftest import default_weights, rel_err
from oracle import pvraft_oracle as O
from test_gpu_grid_search import cloud

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@contextlib.contextmanager
def deterministic(flag):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(flag)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


# ------------------------------------------------------------------------------------------------------------------------
# lookup: cells, means, kNN select, backward
# ------------------------------------------------------------------------------------------------------------------------
FAMILIES = [('lattice', 0.25, 3), ('lattice', 0.125, 4), ('lattice', 0.5, 1),
            ('boundary', 0.3, 3), ('boundary', 0.1, 3), ('boundary', 0.7, 2), ('boundary', 1 / 3, 3), ('boundary', 0.45, 3),
            ('duplicate', 0.25, 3), ('cluster_far', 0.25, 3)]
CONFIGS = [(k, table, dtype) for k in (32, 128, 512, 1024) for table in ('smem', 'global') for dtype in ('fp32', 'bf16')
           if dtype == 'fp32' or k >= 128]
ROWS = 256
GLOBAL_ROWS = 20000   # table rows that keep the gather table out of shared memory at every K
WORST = {}


def report(name, value):
    WORST[name] = max(WORST.get(name, 0.0), value)


@pytest.fixture(scope='module', autouse=True)
def _print_worst():
    yield
    if WORST:
        print('\nworst over the file: ' + ', '.join(f'{k} {v:.2e}' for k, v in sorted(WORST.items())))


def lookup_case(family, base, levels, k, table, dtype, seed):
    c = R.make_case(family, base, levels, k, ROWS, seed, table_rows=GLOBAL_ROWS if table == 'global' else 0)
    if dtype == 'bf16':   # the state the kernel reads: values rounded to bf16 (nearest even), widened exactly
        c['val'] = torch.from_numpy(c['val']).to(torch.bfloat16).float().numpy()
    return c


def run_lookup(c, base, levels, dtype, det, dev):
    from pvraft_b200 import ops
    m = c['xyz2'].shape[1]
    val = torch.from_numpy(c['val']).to(dev)
    idx = torch.from_numpy(c['idx']).to(torch.int32).to(dev)
    if dtype == 'bf16':
        val, idx = ops.corr_state_pack_bf16(val, idx, m)
    xp = ops.xyz_pad(torch.from_numpy(c['xyz2']).to(dev))
    coords = torch.from_numpy(c['coords']).to(dev)
    with deterministic(det):
        out = ops.corr_lookup(val, idx, xp, coords, levels, base, want_slots=True, want_cube=True)
    torch.cuda.synchronize()
    return {key: v.cpu() for key, v in out.items()}, xp, coords


@pytest.mark.parametrize('k,table,dtype', CONFIGS, ids=[f'K{k}-{t}-{d}' for k, t, d in CONFIGS])
@pytest.mark.parametrize('family,base,levels', FAMILIES, ids=[f'{f}-{b:.4g}x{lv}' for f, b, lv in FAMILIES])
def test_lookup_at_boundaries_and_ties(dev, family, base, levels, k, table, dtype):
    from pvraft_b200 import ops
    seed = k * 7 + levels + int(base * 1000) + (1 if table == 'global' else 0)
    c = lookup_case(family, base, levels, k, table, dtype, seed)
    m = c['xyz2'].shape[1]
    assert ops.lookup_table_in_smem(m, k) == (table == 'smem')
    out, xp, coords = run_lookup(c, base, levels, dtype, False, dev)
    n = ROWS

    # (1) every candidate's cell at every level, as the fused kernel decided it
    cells = R.lookup_cells(c['cand'], c['coords'], base, levels)
    got = out['cube'].numpy().astype(np.int64)
    bad = got != cells
    assert not bad.any(), f'{int(bad.sum())} cell decisions differ from the restatement'
    st = O.CorrState(torch.from_numpy(c['val']), torch.from_numpy(c['idx']), torch.from_numpy(c['cand']))
    ct = torch.from_numpy(c['coords'])
    for lvl in range(levels):
        cube, valid = O.voxel_cube_index(st, ct, float(R.level_scales(base, levels)[lvl]))
        assert torch.equal(torch.from_numpy(cells[..., lvl] >= 0), valid), f'torch-CPU division decides level {lvl} differently'
        assert torch.equal(torch.from_numpy(np.maximum(cells[..., lvl], 0)), cube)

    # (2) voxel means (sequential ascending-slot sums == the oracle's scatter_add)
    want = O.voxel_means(st, ct, levels, base).transpose(1, 2)
    vox = out['vox'][..., :levels * 27]
    assert (out['vox'][..., levels * 27:] == 0).all()
    e_vox = rel_err(vox, want)
    assert torch.equal(bits(vox), bits(want)), f'voxel means differ from the oracle by up to {e_vox:.1e}'

    # (3) the 32 nearest, in the kernel's exact order
    dist = R.knn_sqdist(c['cand'], c['coords'])[0]
    want_slots = R.lookup_knn_select(dist)
    got_slots = out['knn_slot'][0].numpy()
    wrong = (got_slots != want_slots).any(-1)
    assert not wrong.any(), f'{int(wrong.sum())} rows select other slots or another order, e.g. row {int(np.argmax(wrong))}'
    kth = np.sort(dist, -1)[:, R.KNN - 1:R.KNN]
    tie_rows = int(((dist <= kth).sum(-1) > R.KNN).sum())
    split = np.zeros(n, bool)
    if k >= 256:   # rows where the kernel's tie rule and the lowest-slot rule pick different sets
        split = (np.sort(want_slots, -1) != R.lowest_slot_select(dist)).any(-1)

    # (4) the gathered 4-vectors, bitwise
    sl = torch.from_numpy(want_slots).long()[None]
    want_sel = O.knn_gather(st, ct, sl).permute(0, 2, 3, 1)
    assert torch.equal(bits(out['knn_sel']), bits(want_sel))

    # (5) moments of the 4-vectors in double
    f = out['knn_sel'].double().reshape(1, -1, 4)
    mo = out['moments']
    assert torch.allclose(mo[:, :4], f.sum(1), rtol=1e-12, atol=1e-9)
    iu = torch.triu_indices(4, 4)
    assert torch.allclose(mo[:, 4:14], torch.einsum('bni,bnj->bij', f, f)[:, iu[0], iu[1]], rtol=1e-12, atol=1e-9)
    assert float(mo[0, 14]) == n * 32

    # (6) DET: the same decisions and values
    det, _, _ = run_lookup(c, base, levels, dtype, True, dev)
    for key in ('cube', 'knn_slot', 'vox', 'knn_sel'):
        assert torch.equal(bits(det[key]), bits(out[key])), key
    assert torch.allclose(det['moments'][:, :15], mo[:, :15], rtol=1e-12, atol=1e-9)

    # (7) backward of the correlation values, float64 over the restated cells
    e_bwd = float('nan')
    if dtype == 'fp32':
        g = torch.Generator().manual_seed(seed)
        g_vox = torch.randn(1, n, levels * 27, generator=g)
        g_sel = torch.randn(1, n, 32, 4, generator=g)
        d_corr = ops.corr_lookup_bwd(torch.from_numpy(c['idx']).to(torch.int32).to(dev), xp, coords,
                                     torch.from_numpy(want_slots).to(torch.int32)[None].to(dev), g_vox.to(dev), g_sel.to(dev),
                                     levels, base).cpu()
        want_d = np.zeros((n, k))
        gv = g_vox[0].double().numpy()
        for lvl in range(levels):
            cl = cells[0, :, :, lvl]
            cnt = np.zeros((n, 27), np.int64)
            rows_i = np.repeat(np.arange(n), k).reshape(n, k)
            np.add.at(cnt, (rows_i[cl >= 0], cl[cl >= 0]), 1)
            cc = np.maximum(cl, 0)
            # clamp(count, 1, N) as the kernel and corr.py:65 (no cell of these 256-row cases holds more than N candidates)
            per = gv[rows_i, lvl * 27 + cc] / np.minimum(np.take_along_axis(cnt, cc, 1), n).clip(min=1)
            want_d += np.where(cl >= 0, per, 0.0)
        np.add.at(want_d, (np.repeat(np.arange(n), 32), want_slots.reshape(-1)), g_sel[0, :, :, 0].double().numpy().reshape(-1))
        want_d = torch.from_numpy(want_d)[None]
        e_bwd = rel_err(d_corr, want_d)
        assert e_bwd < 1e-6, e_bwd
        report('corr_lookup_bwd', e_bwd)
    report('voxel means', e_vox)
    classes = R.boundary_classes(c['cand'], c['coords'], c['intended'], base, levels)
    nz = {key: v for key, v in classes.items() if v}
    print(f'{family} {base:.4g}x{levels} K={k} {table} {dtype}: vox {e_vox:.1e}, bwd {e_bwd:.1e}; rows tied at the 32nd '
          f'place {tie_rows}/{n}, of them picked differently from lowest-slot {int(split.sum())}; classes {nz}')


# ------------------------------------------------------------------------------------------------------------------------
# kNN graph
# ------------------------------------------------------------------------------------------------------------------------
def lidar(n, variant, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = cloud(n, 'lidar', g, dev)[0]
    if variant == 'quantised':
        x = torch.round(x * 16) / 16
    elif variant == 'duplicated':
        pick = torch.randperm(n, generator=g, device=dev)[:n // 10]
        src = torch.randint(0, n, (n // 10,), generator=g, device=dev)
        x[pick] = x[src]
    return x.contiguous()


@pytest.mark.parametrize('variant', ['continuous', 'quantised', 'duplicated'])
@pytest.mark.parametrize('n', [40, 4096, 16384, 20000])
def test_knn_graph_exact_order(dev, n, variant):
    from pvraft_b200 import ops
    x = lidar(n, variant, dev, n + len(variant))
    for mode in (0, 1):
        for k in (16, 32):
            idx, rel = ops.knn(x[None], x[None], k, mode=mode, want_rel=True)
            want_idx, want_rel = R.knn_graph(x, x, k, mode)
            wrong = (idx[0].long() != want_idx).any(-1)
            assert not bool(wrong.any()), f'mode {mode}, k {k}: {int(wrong.sum())} rows differ, e.g. row {int(wrong.int().argmax())}'
            assert torch.equal(bits(rel[0]), bits(want_rel))
            d = torch.gather(R.graph_distance(x[:2048], x, mode), 1, want_idx[:2048])
            ties = int((d[:, 1:] == d[:, :-1]).any(-1).sum())
            print(f'knn graph N={n} {variant} mode {mode} k={k}: order exact; rows (of the first {min(n, 2048)}) with a '
                  f'distance tie among their neighbours {ties}')


# ------------------------------------------------------------------------------------------------------------------------
# model level on LiDAR-like scenes
# ------------------------------------------------------------------------------------------------------------------------
def lidar_scene(b, n, variant, seed):
    """pc1: the LiDAR-like cloud (rings on a ground plane, compact clusters, a sparse far range, tens of metres).  pc2: an
    ego-motion (yaw 0.5-2 degrees, horizontal translation 0.5-1.5 m), two objects (the points within 2 m of two pc1 points)
    moved 0.3-1 m more, and 1 cm noise.  'quantised': both clouds on a 1/16 m lattice; 'duplicated': 10 % of the points of
    each sample copies of others."""
    g = torch.Generator().manual_seed(seed)
    pc1s, pc2s = [], []
    for _ in range(b):
        p1 = cloud(n, 'lidar', g, torch.device('cpu'))[0]
        yaw = math.radians(0.5 + 1.5 * float(torch.rand(1, generator=g))) * (1 if float(torch.rand(1, generator=g)) < 0.5 else -1)
        c, s = math.cos(yaw), math.sin(yaw)
        rot = torch.tensor([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
        phi = float(torch.rand(1, generator=g)) * 2 * math.pi
        t = (0.5 + float(torch.rand(1, generator=g))) * torch.tensor([math.cos(phi), math.sin(phi), 0.0])
        p2 = p1 @ rot.T + t
        for _ in range(2):
            centre = p1[torch.randint(0, n, (1,), generator=g)]
            u = torch.randn(3, generator=g)
            move = u / u.norm() * (0.3 + 0.7 * float(torch.rand(1, generator=g)))
            p2 = torch.where(((p1 - centre).norm(dim=1, keepdim=True) < 2.0), p2 + move, p2)
        p2 = p2 + 0.01 * torch.randn(n, 3, generator=g)
        if variant == 'quantised':
            p1, p2 = torch.round(p1 * 16) / 16, torch.round(p2 * 16) / 16
        elif variant == 'duplicated':
            pick = torch.randperm(n, generator=g)[:n // 10]
            src = torch.randint(0, n, (n // 10,), generator=g)
            p1[pick], p2[pick] = p1[src], p2[src]
        pc1s.append(p1)
        pc2s.append(p2)
    return torch.stack(pc1s).contiguous(), torch.stack(pc2s).contiguous()


def restated_knn_select(state, coords, knn=R.KNN):
    """O.knn_select with the lookup kernel's tie rule: the rule is applied on the block's stored (bank-aware) candidate order,
    which is a function of the candidate ids alone (ops.corr_reorder), and the pick is mapped back to the state's slots."""
    from pvraft_b200 import ops
    idx = state.indices
    b, n, k = idx.shape
    d = R.knn_sqdist(state.truncate_xyz2.detach().numpy(), coords.detach().numpy())
    dev = torch.device('cuda:0')
    _, stored = ops.corr_reorder(torch.zeros(b, n, k, device=dev), idx.to(torch.int32).to(dev))
    stored = stored.long().cpu()
    perm = torch.empty_like(idx)   # perm[s] = the state's slot of stored slot s
    perm.scatter_(2, torch.argsort(stored, -1), torch.argsort(idx, -1))
    ds = np.take_along_axis(d, perm.numpy(), -1)
    sel = R.lookup_knn_select(ds.reshape(b * n, k)).reshape(b, n, knn)
    return torch.gather(perm, 2, torch.from_numpy(sel))


SCENE_ITERS = 8
SCENES = {}


def scene_reference(variant, n, k):
    """The oracle on a LiDAR-like scene, shared between the tests: weights, clouds, loop inputs, per-iteration trace, flows,
    and at N = 4999 the refined flow (RSF_refine's weights; RSF loads the same weights without refine_block)."""
    key = (variant, n, k)
    refine = n == 4999
    if key not in SCENES:
        args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
        W = default_weights(refine=refine, args=args)
        pc1, pc2 = lidar_scene(2, n, variant, seed=n + k + len(variant))
        with torch.no_grad():
            li = O.prepare(W, pc1, pc2, k)
            trace = []
            flows = O.raft_loop(W, li, pc1, SCENE_ITERS, 3, 0.25, trace)
            refined = O.flot_refine(W, 'refine_block', flows[-1], li.feat_graph) if refine else None
        SCENES[key] = dict(W=W, pc1=pc1, pc2=pc2, li=li, trace=trace, flows=flows, refined=refined)
    return SCENES[key]


def free_running_common(m, pc1, pc2, iters, dev):
    """The model's flows on the oracle's kNN graph (computed on the host, so eager: no CUDA-graph capture)."""
    from test_gpu_bench_path import oracle_adjacency
    auto, m.use_cuda_graph = m.use_cuda_graph, False
    try:
        with torch.no_grad(), oracle_adjacency():
            return m([pc1.to(dev), pc2.to(dev)], iters)
    finally:
        m.use_cuda_graph = auto


@pytest.mark.parametrize('variant', ['continuous', 'quantised', 'duplicated'])
@pytest.mark.parametrize('n,k', [(8192, 512), (4999, 256)], ids=['N8192-K512-tc', 'N4999-K256-cuda_core'])
def test_rsf_on_lidar_scenes(dev, monkeypatch, n, k, variant):
    """Teacher-forced per iteration through the loop's kernels on the oracle's state and adjacency (corr 1e-5, motion
    2e-5, net 2e-5, delta 5e-5), then free-running for 8 iterations on the oracle's adjacency (1e-4 mean-abs /
    mean|flow|).  The oracle's kNN select follows the kernel's tie rule, so no tie is exempt."""
    from test_gpu_bench_path import make_model, pm, product_graph
    monkeypatch.setattr(O, 'knn_select', restated_knn_select)
    c = scene_reference(variant, n, k)
    m, _ = make_model(dev, k=k, weights={key: v for key, v in c['W'].items() if not key.startswith('refine_block.')})
    li, b = c['li'], 2
    m.corr_block.set_state(li.state.truncated_corr.to(dev), li.state.indices.to(dev), c['pc2'].to(dev))
    g = product_graph(li.graph, b, n, dev)
    pc1 = c['pc1'].to(dev)
    me = m.update_block.motion_encoder
    tc = n % 128 == 0   # the tensor-core loop; otherwise the CUDA-core kernels behind the reference-layout module seams
    worst = dict(corr=0.0, motion=0.0, net=0.0, delta=0.0)
    with torch.no_grad():
        for it, t in enumerate(c['trace']):
            coords = t['coords'].to(dev).contiguous()
            flow = (coords - pc1).contiguous()
            net_in = li.net if it == 0 else c['trace'][it - 1]['net']   # teacher forcing: the oracle's hidden state
            if tc:
                corr_pm, motion = m.corr_block.feature_motion_tc(coords, flow, me, need_corr=True)
                corr = corr_pm.transpose(1, 2)
                want_motion = O.motion_encoder(c['W'], t['coords'] - c['pc1'], t['corr'], 'update_block.motion_encoder')
                e = rel_err(motion.transpose(1, 2).cpu(), want_motion)
                worst['motion'] = max(worst['motion'], e)
                assert e < 2e-5, (it, 'motion', e)
                _, motion_f = m.corr_block.feature_motion_tc(coords, flow, me, need_corr=False)
                net_new, delta = m.update_block.forward_pm(pm(net_in).to(dev), pm(li.inp).to(dev), motion_f, g)
                net_new = net_new.transpose(1, 2)
            else:
                corr = m.corr_block(coords)
                net_new, delta = m.update_block(net_in.to(dev), li.inp.to(dev), t['corr'].to(dev), flow, g)
            e = rel_err(corr.cpu(), t['corr'])
            worst['corr'] = max(worst['corr'], e)
            assert e < 1e-5, (it, 'corr', e)
            e = rel_err(net_new.cpu(), t['net'])
            worst['net'] = max(worst['net'], e)
            assert e < 2e-5, (it, 'net', e)
            e = rel_err(delta.cpu(), t['delta'])
            worst['delta'] = max(worst['delta'], e)
            assert e < 5e-5, (it, 'delta', e)
    common = free_running_common(m, c['pc1'], c['pc2'], SCENE_ITERS, dev)
    rel = [float((f.cpu() - r).abs().mean() / r.abs().mean()) for f, r in zip(common, c['flows'])]
    for key, v in worst.items():
        report(f'scene teacher-forced {key}', v)
    report('scene free-running', max(rel))
    print(f'lidar scene {variant} N={n} K={k}: teacher-forced worst {worst}; free-running per iteration '
          f'{[f"{r:.1e}" for r in rel]}, mean|flow| {float(c["flows"][-1].abs().mean()):.3f}')
    assert max(rel) < 1e-4, rel


@pytest.mark.parametrize('variant', ['continuous', 'quantised', 'duplicated'])
def test_rsf_refine_on_lidar_scenes(dev, monkeypatch, variant):
    """RSF_refine free-running for 8 iterations (N = 4999, K = 256) on the oracle's adjacency: 1e-4 mean-abs / mean|flow|."""
    from test_gpu_bench_path import make_model
    monkeypatch.setattr(O, 'knn_select', restated_knn_select)
    n, k = 4999, 256
    c = scene_reference(variant, n, k)
    m, _ = make_model(dev, k=k, refine=True, weights=c['W'])
    common = free_running_common(m, c['pc1'], c['pc2'], SCENE_ITERS, dev)
    e = float((common.cpu() - c['refined']).abs().mean() / c['refined'].abs().mean())
    report('scene refine free-running', e)
    print(f'lidar scene {variant} RSF_refine N={n} K={k}: refined flow {e:.2e} mean-abs / mean|flow|')
    assert e < 1e-4, e


def test_training_step_on_quantised_lidar_scene(dev, monkeypatch):
    """One stage-1 step (B = 2, N = 2048, K = 128, 3 iterations) on the quantised scene: all 95 parameter gradients and both
    input gradients against autograd through the oracle (with the kernel's kNN tie rule), on the oracle's kNN graph."""
    from pvraft_b200 import RSF
    from test_gpu_train_coverage import flows_close, model_step, oracle_step
    from train_helpers import compare_grads
    monkeypatch.setattr(O, 'knn_select', restated_knn_select)
    b, n, k, iters = 2, 2048, 128, 3
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    W = default_weights(args=args, seed=3)
    pc1, pc2 = lidar_scene(b, n, 'quantised', seed=2048)
    flows_ref, loss_ref, want = oracle_step(W, pc1, pc2, iters, k)
    m = RSF(args)
    m.load_state_dict(W)
    m = m.to(dev).train()
    flows, loss, got = model_step(m, pc1, pc2, iters, dev)
    e_f = flows_close(flows, flows_ref)
    e_l = abs(loss - loss_ref) / abs(loss_ref)
    print(f'quantised lidar scene training step: flows {e_f:.2e}, loss {e_l:.2e}')
    assert e_f < 1e-4 and e_l < 1e-4, (e_f, e_l)
    l2, mx, _ = compare_grads(got, want, 2e-2, 5e-2)
    report('scene training gradients relative L2', l2)
    report('scene training gradients max-abs', mx)
