"""The refinement of rigid fits against the second scan on the device (csrc/rigid_refine.cu, pvraft_b200.rigid_refine):
the normals against float64 eigh of the same brute-force neighbours, every iteration teacher-forced against the numpy
restatement of test_host_rigid_refine (the kernel's state k moved in fp32 gives the same correspondences, and their solve
gives state k + 1), recovery of a synthetic LiDAR-like scene from biased and noisy flow fits, degenerate geometry, masks
and non-finite input, determinism, batching, per-object equivalence, graph capture, and the fits' use downstream."""
import numpy as np
import pytest
import torch

import test_host_rigid_refine as H
from test_gpu_rigid_motion import same_bits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture
def det():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


@pytest.fixture(scope='module')
def sc():
    return H.scene(0)


@pytest.fixture(scope='module')
def normals(sc):
    return H.normals_ref(sc['xyz2'], 16)


def objects_fit(sc, fits, dev, segs=(0, 1, 2)):
    """A RigidObjects whose object o is segment segs[o] of the scene, with fit fits[o]."""
    import pvraft_b200
    seg = torch.as_tensor(sc['seg'], device=dev)
    labels = torch.full_like(seg, -1, dtype=torch.int32)
    for o, s in enumerate(segs):
        labels[seg == s] = o
    o = len(segs)
    R = torch.tensor(np.stack([fits[k][0] for k in range(o)]), dtype=torch.float32, device=dev)[None]
    t = torch.tensor(np.stack([fits[k][1] for k in range(o)]), dtype=torch.float32, device=dev)[None]
    cnt = torch.tensor([[int((sc['seg'] == s).sum()) for s in segs]], dtype=torch.int32, device=dev)
    return pvraft_b200.RigidObjects(labels[None], torch.tensor([o], dtype=torch.int32, device=dev), R, t, cnt,
                                    torch.zeros(1, o, dtype=torch.bool, device=dev), (labels >= 0)[None])


def call_trace(x1, x2, fit, dev, iterations=10, target_mask=None, max_distance=0.3, k_normal=16):
    """ops.rigid_refine with the trace (history, corr, normals, neighbours) of a RigidObjects fit."""
    from pvraft_b200 import ops
    b, n = x1.shape[:2]
    labels = torch.where(fit.inliers, fit.labels, -1).int().contiguous()
    tm = None if target_mask is None else target_mask.contiguous().view(torch.uint8)
    return ops.rigid_refine(x1.contiguous(), x2.contiguous(), labels, tm, fit.rotation.contiguous(), fit.translation.contiguous(),
                            fit.degenerate.contiguous().view(torch.uint8), iterations, max_distance, k_normal, want_trace=True)


def test_normals_match_float64_eigh_of_the_same_neighbours(sc, normals, dev):
    x1 = torch.tensor(sc['xyz1'], device=dev)[None]
    x2 = torch.tensor(sc['xyz2'], device=dev)[None]
    fits = H.flow_fits(sc, sc['truth'])
    out = call_trace(x1, x2, objects_fit(sc, fits, dev), dev, iterations=1)
    got = out[-2][0].cpu().numpy().astype(np.float64)
    nrm, valid, nbr = normals
    # the neighbour sets: the brute-force fp32 diff_sq search on (distance, id), bit for bit
    assert np.array_equal(out[-1][0].cpu().numpy(), nbr)
    assert np.array_equal(got[:, 3] == 1, valid)
    dots = np.abs((got[valid, :3] * nrm[valid]).sum(1))
    assert dots.min() >= 1 - 1e-6   # fp32 storage of the unit normal
    assert np.all(got[~valid] == 0)


@pytest.mark.parametrize('kind', ['biased', 'noisy'])
def test_every_iteration_teacher_forced_and_recovery(sc, dev, kind):
    import pvraft_b200
    rng = np.random.default_rng(7)
    flow = 0.8 * sc['truth'] if kind == 'biased' else sc['truth'] + rng.normal(0, 0.03, sc['truth'].shape)
    fits = H.flow_fits(sc, flow)
    x1 = torch.tensor(sc['xyz1'], device=dev)[None]
    x2 = torch.tensor(sc['xyz2'], device=dev)[None]
    fit = objects_fit(sc, fits, dev)
    R, t, degen, matched, rmse, rank, steps, hist, corr, kn, _ = call_trace(x1, x2, fit, dev)
    hist, corr, kn = hist[0].cpu().numpy(), corr[0].cpu().numpy(), kn[0].cpu().numpy()
    valid = kn[:, 3] == 1   # equal to the restatement's flags (test_normals_match_float64_eigh_of_the_same_neighbours)
    X1 = sc['xyz1']
    for o in range(3):
        mem = sc['seg'] == o
        X = X1[mem]
        cx = X.astype(np.float64).mean(0)
        rho = np.sqrt(((X - cx) ** 2).sum(1).mean())
        n_steps = int(steps[0, o])
        for k in range(n_steps):
            Rk, cyk = hist[o, k, :9].reshape(3, 3), hist[o, k, 9:]
            p = H.move32(Rk, cx, cyk, X)
            c = H.match_ref(p, sc['xyz2'], valid, 0.3)
            hit = c >= 0
            z, rk, _, _ = H.solve_ref(p[hit], sc['xyz2'][c[hit]], kn[c[hit], :3], cyk, rho)
            R1 = H.rodrigues(z[:3] / rho) @ Rk
            cy1 = cyk + z[3:]
            assert np.abs(R1 - hist[o, k + 1, :9].reshape(3, 3)).max() < 1e-9, (o, k)
            assert np.abs(cy1 - hist[o, k + 1, 9:]).max() < 1e-9 * max(1.0, np.abs(cy1).max()), (o, k)
        # the last iteration's correspondences, bit for bit: every iteration here updates, so the last one moved with
        # state steps - 1 (and a converged segment's later launches returned at once)
        last = n_steps - 1
        Rl, cyl = hist[o, last, :9].reshape(3, 3), hist[o, last, 9:]
        want = H.match_ref(H.move32(Rl, cx, cyl, X), sc['xyz2'], valid, 0.3)
        assert np.array_equal(corr[mem], want), o
        assert int(matched[0, o]) == int((want >= 0).sum())
    # recovery: the bounds of the CPU restatement
    after = H.errors([(R[0, o].double().cpu().numpy(), t[0, o].double().cpu().numpy()) for o in range(3)], sc['motions'])
    before = H.errors(fits, sc['motions'])
    for o in range(3):
        assert after[o][0] < H.REFINED[o][0] and after[o][1] < H.REFINED[o][1], (o, before[o], after[o])
        assert int(rank[0, o]) == 6 and not bool(degen[0, o])
        if kind == 'biased':
            assert after[o][1] * H.GAIN_BIASED < before[o][1]
    # rigid_flow with the refined fits has the lower error
    ref = pvraft_b200.RigidRefinement(fit._replace(rotation=R, translation=t), matched, rmse, rank, steps)
    f = torch.tensor(flow, dtype=torch.float32, device=dev)[None]
    truth = torch.tensor(sc['truth'], dtype=torch.float32, device=dev)[None]
    epe_in = (pvraft_b200.rigid_flow(x1, f, fit) - truth).norm(dim=-1).mean()
    epe_out = (pvraft_b200.rigid_flow(x1, f, ref.fit) - truth).norm(dim=-1).mean()
    if kind == 'biased':
        assert epe_out < 0.2 * epe_in, (float(epe_in), float(epe_out))
    else:
        assert epe_out < 0.03, float(epe_out)


def test_rigid_motion_then_refine_recovers_a_biased_ego_motion(sc, dev):
    import pvraft_b200
    x1 = torch.tensor(sc['xyz1'], device=dev)[None]
    x2 = torch.tensor(sc['xyz2'], device=dev)[None]
    f = torch.tensor(0.8 * sc['truth'], dtype=torch.float32, device=dev)[None]
    static = torch.tensor(sc['seg'] == 0, device=dev)[None]
    ego = pvraft_b200.rigid_motion(x1, f, mask=static)
    out = pvraft_b200.rigid_refine(x1, x2, ego)
    assert isinstance(out.fit, pvraft_b200.RigidMotion) and out.fit.rotation.shape == (1, 3, 3)
    assert out.matched.shape == (1, 1) and out.rank.shape == (1, 1)
    Rt, tt = sc['motions'][0]
    before = np.linalg.norm(ego.translation[0].double().cpu().numpy() - tt)
    after = np.linalg.norm(out.fit.translation[0].double().cpu().numpy() - tt)
    assert before > 0.15 * np.linalg.norm(tt)
    assert after < H.REFINED[0][1] and H.rot_deg(out.fit.rotation[0].double().cpu().numpy(), Rt) < H.REFINED[0][0]
    assert torch.equal(out.fit.inliers, ego.inliers) and torch.equal(out.fit.count, ego.count)
    rf = pvraft_b200.rigid_flow(x1, f, pvraft_b200.RigidObjects(torch.full((1, x1.shape[1]), -1, dtype=torch.int32, device=dev),
                                                                  torch.zeros(1, dtype=torch.int32, device=dev), torch.eye(3, device=dev).expand(1, 1, 3, 3),
                                                                  torch.zeros(1, 1, 3, device=dev), torch.zeros(1, 1, dtype=torch.int32, device=dev),
                                                                  torch.ones(1, 1, dtype=torch.bool, device=dev),
                                                                  torch.zeros(1, x1.shape[1], dtype=torch.bool, device=dev)), ego=out.fit)
    assert torch.isfinite(rf).all()


def test_a_ground_plane_leaves_x_y_and_yaw_alone(dev):
    import pvraft_b200
    rng = np.random.default_rng(3)
    g1 = np.stack([rng.uniform(-10, 10, 3000), rng.uniform(-10, 10, 3000), np.zeros(3000)], 1).astype(np.float32)
    g2 = np.stack([rng.uniform(-10, 10, 3000), rng.uniform(-10, 10, 3000), np.zeros(3000)], 1).astype(np.float32)
    R0 = np.array([[1, 0, 0], [0, np.cos(0.01), -np.sin(0.01)], [0, np.sin(0.01), np.cos(0.01)]]) @ H.yaw(2.0)
    t0 = np.array([0.3, -0.2, 0.05])
    x1, x2 = torch.tensor(g1, device=dev)[None], torch.tensor(g2, device=dev)[None]
    fit = pvraft_b200.RigidObjects(torch.zeros(1, 3000, dtype=torch.int32, device=dev), torch.ones(1, dtype=torch.int32, device=dev),
                                   torch.tensor(R0, dtype=torch.float32, device=dev)[None, None],
                                   torch.tensor(t0, dtype=torch.float32, device=dev)[None, None], torch.zeros(1, 1, dtype=torch.int32, device=dev),
                                   torch.ones(1, 1, dtype=torch.bool, device=dev), torch.ones(1, 3000, dtype=torch.bool, device=dev))
    R, t, degen, matched, rmse, rank, steps, hist, corr, _, _ = call_trace(x1, x2, fit, dev)
    assert int(rank[0, 0]) == 3 and bool(degen[0, 0])
    h = hist[0, 0].cpu().numpy()
    for k in range(int(steps[0, 0])):
        Ra, Rb = h[k, :9].reshape(3, 3), h[k + 1, :9].reshape(3, 3)
        w = Rb @ Ra.T
        assert abs(w[1, 0] - w[0, 1]) / 2 < 1e-9
        assert np.abs(h[k + 1, 9:11] - h[k, 9:11]).max() < 1e-9
    p = H.transform(R[0, 0].double().cpu().numpy(), t[0, 0].double().cpu().numpy(), g1.astype(np.float64))
    assert np.abs(p[:, 2]).max() < 1e-4


def test_masked_and_non_finite_points_and_empty_slots(sc, dev):
    x1 = torch.tensor(sc['xyz1'], device=dev)[None].clone()
    x2 = torch.tensor(sc['xyz2'], device=dev)[None].clone()
    fits = H.flow_fits(sc, 0.8 * sc['truth'])
    fit = objects_fit(sc, fits + [fits[0]], dev, segs=(0, 1, 2, 9))   # slot 3: no member
    x1[0, :50] = float('nan')
    x2[0, :50] = float('inf')
    tm = torch.rand(1, x2.shape[1], device=dev, generator=torch.Generator(dev).manual_seed(0)) < 0.7
    R, t, degen, matched, rmse, rank, steps, hist, corr, nrm, _ = call_trace(x1, x2, fit, dev, target_mask=tm)
    c = corr[0]
    hit = c >= 0
    assert bool(tm[0, c[hit].long()].all())
    assert not bool(hit[:50].any())
    assert bool((c[hit] >= 50).all())
    assert bool((nrm[0, ~tm[0], 3] == 0).all()) and bool((nrm[0, :50, 3] == 0).all())
    assert same_bits(R[0, 3], fit.rotation[0, 3]) and same_bits(t[0, 3], fit.translation[0, 3])
    assert int(steps[0, 3]) == 0 and int(matched[0, 3]) == 0 and int(rank[0, 3]) == 0
    assert all(int(steps[0, o]) > 0 for o in range(3))


def test_deterministic_batched_per_object_and_graph(sc, dev, det):
    import pvraft_b200
    x1 = torch.tensor(sc['xyz1'], device=dev)[None]
    x2 = torch.tensor(sc['xyz2'], device=dev)[None]
    fa = objects_fit(sc, H.flow_fits(sc, 0.8 * sc['truth']), dev)
    fb = objects_fit(sc, H.flow_fits(sc, sc['truth'] + np.random.default_rng(1).normal(0, 0.03, sc['truth'].shape)), dev)
    a1 = pvraft_b200.rigid_refine(x1, x2, fa)
    a2 = pvraft_b200.rigid_refine(x1, x2, fa)
    for u, v in zip(a1[1:], a2[1:]):
        assert torch.equal(u, v)
    assert same_bits(a1.fit.rotation, a2.fit.rotation) and same_bits(a1.fit.translation, a2.fit.translation)
    # batched equals per-sample
    batch = pvraft_b200.RigidObjects(*[torch.cat([u, v]) for u, v in zip(fa, fb)])
    ab = pvraft_b200.rigid_refine(torch.cat([x1, x1]), torch.cat([x2, x2]), batch)
    b1 = pvraft_b200.rigid_refine(x1, x2, fb)
    assert same_bits(ab.fit.rotation, torch.cat([a1.fit.rotation, b1.fit.rotation]))
    assert same_bits(ab.fit.translation, torch.cat([a1.fit.translation, b1.fit.translation]))
    assert torch.equal(ab.steps, torch.cat([a1.steps, b1.steps])) and torch.equal(ab.rmse, torch.cat([a1.rmse, b1.rmse]))
    # object o equals the object refined alone
    for o in range(3):
        single = pvraft_b200.RigidObjects(fa.labels, fa.num_objects, fa.rotation[:, o:o + 1], fa.translation[:, o:o + 1],
                                          fa.count[:, o:o + 1], fa.degenerate[:, o:o + 1], fa.inliers & (fa.labels == o))
        so = pvraft_b200.rigid_refine(x1, x2, single)
        assert same_bits(so.fit.rotation[:, 0], a1.fit.rotation[:, o]) and same_bits(so.fit.translation[:, 0], a1.fit.translation[:, o]), o
        assert torch.equal(so.steps[:, 0], a1.steps[:, o]) and torch.equal(so.rank[:, 0], a1.rank[:, o])
    # eager equals a CUDA-graph replay (no host synchronisation inside the call)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pvraft_b200.rigid_refine(x1, x2, fa)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gout = pvraft_b200.rigid_refine(x1, x2, fa)
    g.replay()
    torch.cuda.synchronize()
    assert same_bits(gout.fit.rotation, a1.fit.rotation) and same_bits(gout.fit.translation, a1.fit.translation)
    # the default mode agrees with the deterministic one
    torch.use_deterministic_algorithms(False)
    nd = pvraft_b200.rigid_refine(x1, x2, fa)
    assert (nd.fit.rotation - a1.fit.rotation).abs().max() < 1e-6
    assert (nd.fit.translation - a1.fit.translation).abs().max() < 1e-6


def test_the_tracker_takes_refined_fits(sc, dev):
    import pvraft_b200
    x1 = torch.tensor(sc['xyz1'], device=dev)[None]
    x2 = torch.tensor(sc['xyz2'], device=dev)[None]
    f = torch.tensor(0.8 * sc['truth'], dtype=torch.float32, device=dev)[None]
    ego = pvraft_b200.rigid_motion(x1, f, mask=torch.tensor(sc['seg'] == 0, device=dev)[None])
    obj = pvraft_b200.rigid_objects(x1, f, mask=~ego.inliers, flow_radius=0.3)
    ego_r = pvraft_b200.rigid_refine(x1, x2, ego)
    obj_r = pvraft_b200.rigid_refine(x1, x2, obj)
    tr = pvraft_b200.ObjectTracker()
    tracks = tr.step(x1, f, obj_r.fit, ego_r.fit)
    assert tracks is not None
    assert torch.isfinite(pvraft_b200.rigid_flow(x1, f, obj_r.fit, ego=ego_r.fit)).all()


def expected_last(x1, x2, fit, hist, corr, kn, steps):
    """matched and rmse of the last iteration from the kernel's own state, correspondences and normals (numpy, float64 sums
    of the fp32 values)."""
    labels = torch.where(fit.inliers, fit.labels, -1)[0].cpu().numpy()
    X1, X2 = x1[0].cpu().numpy(), x2[0].cpu().numpy()
    out = []
    for o in range(fit.rotation.shape[1]):
        mem = labels == o
        X = X1[mem]
        cx = X.astype(np.float64).mean(0)
        last = max(int(steps[0, o]) - 1, 0)   # every iteration that ran updated, so the last moved with state steps - 1
        Rl, cyl = hist[0, o, last, :9].cpu().numpy().reshape(3, 3), hist[0, o, last, 9:].cpu().numpy()
        p = H.move32(Rl, cx, cyl, X)
        c = corr[0].cpu().numpy()[mem]
        hit = c >= 0
        n = kn[0].cpu().numpy()[c[hit], :3].astype(np.float64)
        r = (n * (p[hit].astype(np.float64) - X2[c[hit]].astype(np.float64))).sum(1)
        out.append((int(hit.sum()), float(np.sqrt((r * r).mean())) if hit.any() else 0.0))
    return out


@pytest.mark.parametrize('deterministic', [False, True])
@pytest.mark.parametrize('iterations,segs', [(1, (0,)), (1, (0, 1, 2)), (3, (1, 2, 0))])
def test_matched_and_rmse_over_a_stale_workspace(sc, dev, deterministic, iterations, segs):
    """An odd number of segments, with one running the last iteration: every accumulator starts from zero even when the
    workspace held other values."""
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        x1 = torch.tensor(sc['xyz1'], device=dev)[None]
        x2 = torch.tensor(sc['xyz2'], device=dev)[None]
        fits = H.flow_fits(sc, 0.8 * sc['truth'])
        fit = objects_fit(sc, [fits[s] for s in segs], dev, segs=segs)
        for _ in range(2):
            junk = torch.full((64 << 20,), 3.0e5, dtype=torch.float64, device=dev)   # leave large values in the cache
            del junk
            R, t, degen, matched, rmse, rank, steps, hist, corr, kn, _ = call_trace(x1, x2, fit, dev, iterations=iterations)
            for o, (m, e) in enumerate(expected_last(x1, x2, fit, hist, corr, kn, steps)):
                assert int(matched[0, o]) == m, (o, int(matched[0, o]), m)
                assert abs(float(rmse[0, o]) - e) <= 1e-6 * e + 1e-12, (o, float(rmse[0, o]), e)
    finally:
        torch.use_deterministic_algorithms(was)


def test_matches_at_the_exact_gate_and_ties_by_id(dev):
    """Points exactly fl(max_distance^2) from a target match it; points one step beyond do not; a point equidistant from
    two targets matches the lower id.  Coordinates are multiples of 2^-10 and the source cloud is symmetric about 0, so the
    centroid is 0, the identity fit moves every point onto itself, and every diff_sq below is exact."""
    import pvraft_b200
    gx, gy = np.meshgrid(np.arange(-8, 9), np.arange(-8, 9))
    tgt = np.stack([gx.ravel(), gy.ravel(), np.zeros(gx.size)], 1).astype(np.float32)
    tgt = tgt[np.random.default_rng(5).permutation(len(tgt))]          # ids not in grid order
    eps = 2.0 ** -10
    half = [(2, 3, 0.25), (-5, 1, 0.25), (4, -6, 0.25 + eps), (0, 7, 0.25 + eps),   # on the gate / just beyond (0.25 m)
            (1.5, 2, 0.25), (-3, -2.5, 0.25)]                                        # ties at 0.3125 with r = 0.75
    src = np.array(half + [(-a, -b, -c) for a, b, c in half], np.float32)
    x1, x2 = torch.tensor(src, device=dev)[None], torch.tensor(tgt, device=dev)[None]

    def refine(max_distance):
        fit = pvraft_b200.RigidObjects(torch.zeros(1, len(src), dtype=torch.int32, device=dev), torch.ones(1, dtype=torch.int32, device=dev),
                                       torch.eye(3, device=dev)[None, None], torch.zeros(1, 1, 3, device=dev),
                                       torch.zeros(1, 1, dtype=torch.int32, device=dev), torch.ones(1, 1, dtype=torch.bool, device=dev),
                                       torch.ones(1, len(src), dtype=torch.bool, device=dev))
        out = call_trace(x1, x2, fit, dev, iterations=1, max_distance=max_distance)
        kn = out[-2][0].cpu().numpy()
        p = H.move32(np.eye(3), np.zeros(3), np.zeros(3), src)
        assert np.array_equal(p, src)                                    # the move is exact here
        want = H.match_ref(p, tgt, kn[:, 3] == 1, max_distance)
        got = out[8][0].cpu().numpy()
        assert np.array_equal(got, want)
        return got

    def target_at(x, y):
        return int(np.nonzero((tgt[:, 0] == x) & (tgt[:, 1] == y))[0][0])

    got = refine(0.25)
    n = len(half)
    for j, (a, b, c) in enumerate(half[:4]):
        on = c == 0.25
        for k, (u, v) in ((j, (a, b)), (n + j, (-a, -b))):
            assert got[k] == (target_at(u, v) if on else -1), (k, got[k])
    got = refine(0.75)
    for j, (a, b, c) in enumerate(half[4:], start=4):
        for k, sgn in ((j, 1), (n + j, -1)):
            u, v = sgn * a, sgn * b
            pair = [target_at(np.floor(u), v), target_at(np.ceil(u), v)] if u % 1 else [target_at(u, np.floor(v)), target_at(u, np.ceil(v))]
            assert got[k] == min(pair), (k, got[k], pair)


def test_two_walls_and_a_ground_leave_one_direction(dev):
    import pvraft_b200
    rng = np.random.default_rng(3)
    g1 = np.stack([rng.uniform(-10, 10, 3000), rng.uniform(-10, 10, 3000), np.zeros(3000)], 1)
    g2 = np.stack([rng.uniform(-10, 10, 3000), rng.uniform(-10, 10, 3000), np.zeros(3000)], 1)
    walls = [np.concatenate([np.stack([np.full(1500, s), rng.uniform(-10, 10, 1500), rng.uniform(1.5, 4.5, 1500)], 1)
                             for s in (-5.0, 5.0)]) for _ in range(2)]
    a = torch.tensor(np.concatenate([g1, walls[0]]), dtype=torch.float32, device=dev)[None]
    b = torch.tensor(np.concatenate([g2, walls[1]]), dtype=torch.float32, device=dev)[None]
    n = a.shape[1]
    fit = pvraft_b200.RigidMotion(torch.tensor(H.yaw(1.0), dtype=torch.float32, device=dev)[None],
                                  torch.tensor([[0.1, -0.2, 0.05]], dtype=torch.float32, device=dev),
                                  torch.ones(1, n, dtype=torch.bool, device=dev), torch.full((1,), n, dtype=torch.int32, device=dev),
                                  torch.ones(1, dtype=torch.bool, device=dev))
    out = pvraft_b200.rigid_refine(a, b, fit)
    assert int(out.rank[0, 0]) == 5 and bool(out.fit.degenerate[0])
    ref = H.icp_ref(a[0].cpu().numpy(), b[0].cpu().numpy(), np.ones(n, bool), H.yaw(1.0), np.array([0.1, -0.2, 0.05]))
    assert ref['rank'] == 5


def test_fit_tensors_off_the_device_are_refused(sc, dev):
    import pvraft_b200
    from pvraft_b200._lib import PvraftError
    x1 = torch.tensor(sc['xyz1'], device=dev)[None]
    x2 = torch.tensor(sc['xyz2'], device=dev)[None]
    fit = objects_fit(sc, H.flow_fits(sc, sc['truth']), dev)
    for name in ('labels', 'inliers', 'degenerate', 'translation'):
        with pytest.raises(PvraftError):
            pvraft_b200.rigid_refine(x1, x2, fit._replace(**{name: getattr(fit, name).cpu()}))
