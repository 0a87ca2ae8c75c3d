"""Object tracking on the device (csrc/tracks.cu, pvraft_b200.track): the votes and the greedy assignment against numpy
restatements, bit for bit; identities and composed poses along a synthetic scan sequence with boxes that enter, leave, pass
close by and split; repeatability, batching, no host synchronisation, CUDA-graph capture, and the grid form of the search at
131 072 points."""
import math

import numpy as np
import pytest
import torch

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


def same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


# ---- numpy restatements ----------------------------------------------------------------------------------------------------
def restate_votes(xp, gp, lp, tp, x, lab, num, nn, o, gate):
    """members [B,O], overlap [B,O,O_prev] as pvraft_track_objects_fwd states them; every input a numpy array."""
    b, n = lab.shape
    o_prev = tp.shape[1]
    g2 = np.float32(gate) * np.float32(gate)
    members = np.zeros((b, o), np.int64)
    overlap = np.zeros((b, o, o_prev), np.int64)
    for s in range(b):
        nb = min(int(num[s]), o)
        c = lab[s].astype(np.int64)
        take = (c >= 0) & (c < nb)
        np.add.at(members[s], c[take], 1)
        if xp is None:
            continue
        m = xp.shape[1]
        i = nn[s].astype(np.int64)
        ok = take & (i >= 0) & (i < m)
        a = np.full(n, -1, np.int64)
        a[ok] = lp[s][i[ok]]
        ok &= (a >= 0) & (a < o_prev)
        ok[ok] &= tp[s][a[ok]] >= 0
        w = (xp[s] + gp[s]).astype(np.float32)
        d = (x[s] - w[np.where(ok, i, 0)]).astype(np.float32)
        d2 = ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(np.float32)
        ok &= d2 <= g2
        np.add.at(overlap[s], (c[ok], a[ok]), 1)
    return members, overlap


def compose(Ra, ta, Q):
    """(R_a R_p, R_a t_p + t_a) in double, each entry (x0 y0 + x1 y1) + x2 y2 (numpy never contracts) -> [12]."""
    Ra, ta = Ra.astype(np.float64).reshape(3, 3), ta.astype(np.float64)
    Rp, tp = Q[:9].reshape(3, 3), Q[9:]
    out = np.zeros(12)
    for i in range(3):
        for k in range(3):
            out[3 * i + k] = (Ra[i, 0] * Rp[0, k] + Ra[i, 1] * Rp[1, k]) + Ra[i, 2] * Rp[2, k]
        out[9 + i] = ((Ra[i, 0] * tp[0] + Ra[i, 1] * tp[1]) + Ra[i, 2] * tp[2]) + ta[i]
    return out


def restate_assign(overlap, members, num, tp, ap, pp, Rp, tq, min_overlap, next_id):
    """(match, track, age [B,O], pose [B,O,12], next_id [B]) as pvraft_track_objects_fwd states them."""
    b, o, _ = overlap.shape
    match, track, age = (np.full((b, o), -1, np.int64) for _ in range(3))
    pose = np.zeros((b, o, 12))
    pose[:, :, [0, 4, 8]] = 1.0
    nid = next_id.astype(np.int64).copy()
    for s in range(b):
        nb = max(0, min(int(num[s]), o))
        pairs = sorted((-int(overlap[s, c, a]), c, a) for c in range(nb) for a in range(overlap.shape[2])
                       if overlap[s, c, a] >= 1 and float(overlap[s, c, a]) >= float(min_overlap) * float(members[s, c]))
        taken = set()
        for _, c, a in pairs:
            if match[s, c] < 0 and a not in taken:
                match[s, c] = a
                taken.add(a)
        for c in range(nb):
            a = match[s, c]
            if a < 0:
                track[s, c], age[s, c] = nid[s], 0
                nid[s] += 1
            else:
                track[s, c], age[s, c] = tp[s, a], ap[s, a] + 1
                pose[s, c] = compose(Rp[s, a], tq[s, a], pp[s, a])
    return match, track, age, pose, nid


def cpu(*ts):
    return [None if t is None else t.cpu().numpy() for t in ts]


def run_and_check(dev, prev, x, lab, num, o, nn, gate, min_overlap, next_id):
    """ops.track_objects against both restatements; returns its outputs."""
    from pvraft_b200 import ops
    nid0 = next_id.clone()
    overlap, members, match, track, age, pose = ops.track_objects(prev, x, lab, num, o, nn, gate, min_overlap, next_id)
    xp, gp, lp, tp, ap, pp, Rp, tq = cpu(*prev) if prev is not None else (None,) * 8
    o_prev = 0 if prev is None else tp.shape[1]
    tp = np.zeros((x.shape[0], 0), np.int64) if prev is None else tp
    want_m, want_o = restate_votes(xp, gp, lp, tp, *cpu(x, lab, num, nn), o, gate)
    assert np.array_equal(members.cpu().numpy(), want_m)
    assert np.array_equal(overlap.cpu().numpy(), want_o) and overlap.shape[2] == o_prev
    want = restate_assign(want_o, want_m, num.cpu().numpy(), tp, ap, pp, Rp, tq, min_overlap, nid0.cpu().numpy())
    for got, w in zip((match, track, age), want[:3]):
        assert np.array_equal(got.cpu().numpy(), w)
    assert np.array_equal(pose.cpu().numpy().view(np.uint64), want[3].view(np.uint64))
    assert np.array_equal(next_id.cpu().numpy(), want[4])
    return overlap, members, match, track, age, pose


def random_prev(g, b, m, o_prev, dev, xp=None, gp=None, lp=None, empty=0.2):
    """A previous step's state: random ids (a share `empty` of the slots empty), ages, double poses and fp32 fits."""
    tp = torch.randint(0, 1000, (b, o_prev), generator=g, dtype=torch.int32)
    tp[torch.rand(b, o_prev, generator=g) < empty] = -1
    ap = torch.randint(0, 9, (b, o_prev), generator=g, dtype=torch.int32)
    pp = torch.randn(b, o_prev, 12, generator=g, dtype=torch.float64)
    Rp = torch.randn(b, o_prev, 3, 3, generator=g)
    tq = torch.randn(b, o_prev, 3, generator=g) * 10
    return tuple(t.to(dev).contiguous() for t in (xp, gp, lp, tp, ap, pp, Rp, tq))


# ---- 1. votes ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('grid', [False, True])
@pytest.mark.parametrize('o_prev,o,gate', [(12, 12, 0.5), (7, 20, 0.5), (30, 5, 0.3)])
def test_votes_equal_restatement(dev, grid, o_prev, o, gate):
    """Quantised coordinates (a 1/8 m lattice) put many pairs at exactly fl(gate^2); NaN points, nn = -1 and nn >= M, labels
    outside their ranges, num_objects above O, and empty previous slots are all in the draw."""
    from pvraft_b200 import ops
    g = torch.Generator().manual_seed(o_prev * 100 + o + int(grid))
    b, m, n = 3, 3000, 2500
    xp = torch.randint(0, 24, (b, m, 3), generator=g).float() / 8
    gp = torch.randint(-2, 3, (b, m, 3), generator=g).float() / 8
    x = torch.randint(0, 24, (b, n, 3), generator=g).float() / 8
    x[:, ::97, 1] = float('nan')
    lp = torch.randint(-2, o_prev + 2, (b, m), generator=g, dtype=torch.int32)
    lab = torch.randint(-2, o + 2, (b, n), generator=g, dtype=torch.int32)
    num = torch.tensor([o, o - 3, o + 5], dtype=torch.int32)
    prev = random_prev(g, b, m, o_prev, dev, xp, gp, lp)
    x, lab, num = x.to(dev), lab.to(dev), num.to(dev)
    nn = ops.flow_propagate(prev[0], prev[1], x, k=1, want_idx=True, use_grid=grid)[1].view(b, n).contiguous()
    if not grid:
        assert bool((nn[:, ::97] == -1).all())   # a NaN query has no nearest point
    nn[:, 1::53] = -1
    nn[:, 2::61] = m
    next_id = torch.tensor([0, 5, 1000], dtype=torch.int32, device=dev)
    overlap, members, *_ = run_and_check(dev, prev, x, lab, num, o, nn, gate, 0.5, next_id)
    assert int(overlap.sum()) > 100 and int(members.sum()) > 1000


def test_votes_at_exactly_gate_squared_and_the_next_float(dev):
    from pvraft_b200 import ops
    up = float(np.nextafter(np.float32(0.5), np.float32(1)))
    xp = torch.tensor([[[0.0, 0.0, 0.0], [0.0, 10.0, 0.0], [0.0, 20.0, 0.0]]], device=dev)
    x = torch.tensor([[[0.5, 0.0, 0.0], [up, 10.0, 0.0], [0.0, 20.0, -0.5]]], device=dev)
    lp = torch.tensor([[0, 1, 2]], dtype=torch.int32, device=dev)
    g = torch.Generator().manual_seed(3)
    prev = random_prev(g, 1, 3, 3, dev, xp, torch.zeros_like(xp), lp)
    prev = prev[:3] + (torch.tensor([[4, 5, 6]], dtype=torch.int32, device=dev),) + prev[4:]
    nn = ops.flow_propagate(prev[0], prev[1], x, k=1, want_idx=True)[1].view(1, 3).contiguous()
    assert nn.tolist() == [[0, 1, 2]]
    num = torch.tensor([3], dtype=torch.int32, device=dev)
    overlap, members, match, track, *_ = run_and_check(dev, prev, x, lp.clone(), num, 3, nn, 0.5, 0.5,
                                                       torch.zeros(1, dtype=torch.int32, device=dev))
    assert overlap[0].diagonal().tolist() == [1, 0, 1] and members.tolist() == [[1, 1, 1]]
    assert track.tolist() == [[4, 0, 6]]


# ---- 2. assignment -------------------------------------------------------------------------------------------------------------
def planted(g, dev, o_prev, o, counts, extra, num, empty=0.2):
    """Inputs whose votes are exactly counts [B,O,O_prev] (+ extra [B,O] members with no vote): previous slot a has one
    point W_a = (2a, 0, 0); each vote is a current point at W_a with nn = a; each extra member has nn = -1."""
    b = counts.shape[0]
    m = o_prev + 1
    xp = torch.zeros(b, m, 3)
    xp[:, :, 0] = 2.0 * torch.arange(m)
    lp = torch.arange(m, dtype=torch.int32).expand(b, m).clone()
    lp[:, -1] = -1
    rows = []
    for s in range(b):
        pts, lab, nn = [], [], []
        for c in range(o):
            for a in range(o_prev):
                k = int(counts[s, c, a])
                pts += [xp[s, a]] * k; lab += [c] * k; nn += [a] * k
            k = int(extra[s, c])
            pts += [torch.zeros(3)] * k; lab += [c] * k; nn += [-1] * k
        rows.append((pts, lab, nn))
    n = max(1, max(len(r[1]) for r in rows))
    x = torch.zeros(b, n, 3)
    labels = torch.full((b, n), -1, dtype=torch.int32)
    nns = torch.full((b, n), -1, dtype=torch.int32)
    for s, (pts, lab, nn) in enumerate(rows):
        if lab:
            x[s, :len(lab)] = torch.stack(pts)
            labels[s, :len(lab)] = torch.tensor(lab, dtype=torch.int32)
            nns[s, :len(lab)] = torch.tensor(nn, dtype=torch.int32)
    prev = random_prev(g, b, m, o_prev, dev, xp, torch.zeros_like(xp), lp, empty)
    return prev, x.to(dev), labels.to(dev), torch.tensor(num, dtype=torch.int32, device=dev), nns.to(dev)


@pytest.mark.parametrize('min_overlap', [1 / 16, 0.5, 1.0])
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_assignment_equals_restatement_with_ties(dev, min_overlap, seed):
    g = torch.Generator().manual_seed(10 + seed)
    b, o_prev, o = 4, 24, 40
    counts = torch.randint(1, 4, (b, o, o_prev), generator=g) * (torch.rand(b, o, o_prev, generator=g) < 0.12)
    extra = torch.randint(0, 3, (b, o), generator=g)
    counts[:, ::3] = 0   # every third slot votes for one previous object only, so that min_overlap = 1 has pairs too
    for c in range(0, o, 3):
        counts[:, c, (c // 3) % o_prev] = 2
    extra[:, ::3] = 0
    prev, x, lab, num, nn = planted(g, dev, o_prev, o, counts, extra, [o, 31, 0, o + 9])
    next_id = torch.tensor([0, 3, 7, 2 ** 20], dtype=torch.int32, device=dev)
    _, _, match, *_ = run_and_check(dev, prev, x, lab, num, o, nn, 0.5, min_overlap, next_id)
    assert int((match >= 0).sum()) >= 3


def test_sixteen_eligible_pairs_per_slot_at_the_least_min_overlap(dev):
    """min_overlap = 1/16 with 16 single votes for 16 previous objects in every one of 256 slots: 4096 eligible pairs."""
    g = torch.Generator().manual_seed(20)
    o = 256
    counts = torch.zeros(1, o, o, dtype=torch.int64)
    for c in range(o):
        counts[0, c, (c + 7 * torch.arange(16)) % o] = 1
    prev, x, lab, num, nn = planted(g, dev, o, o, counts, torch.zeros(1, o, dtype=torch.int64), [o], empty=0.0)
    next_id = torch.zeros(1, dtype=torch.int32, device=dev)
    overlap, _, match, *_ = run_and_check(dev, prev, x, lab, num, o, nn, 0.5, 1 / 16, next_id)
    assert int((overlap >= 1).sum()) == 16 * o
    _, _, match1, *_ = run_and_check(dev, prev, x, lab, num, o, nn, 0.5, 1 / 16 + 1e-9, next_id.clone())
    assert int((match1 >= 0).sum()) == 0 and int((match >= 0).sum()) > 0


def test_first_step_births_every_object(dev):
    g = torch.Generator().manual_seed(21)
    b, n, o = 3, 500, 9
    x = torch.randn(b, n, 3, generator=g).to(dev)
    lab = torch.randint(-1, o, (b, n), generator=g, dtype=torch.int32).to(dev)
    num = torch.tensor([o, 4, 0], dtype=torch.int32, device=dev)
    next_id = torch.tensor([0, 10, 3], dtype=torch.int32, device=dev)
    overlap, members, match, track, age, pose = run_and_check(dev, None, x, lab, num, o, None, 0.5, 0.5, next_id)
    assert overlap.shape == (b, o, 0)
    assert track[0].tolist() == list(range(o)) and track[1].tolist() == [10, 11, 12, 13] + [-1] * 5 and track[2].tolist() == [-1] * o
    assert next_id.tolist() == [o, 14, 3] and int(match.max()) == -1


# ---- 3. a synthetic sequence -------------------------------------------------------------------------------------------------
def rot_z(deg):
    a = math.radians(deg)
    return torch.tensor([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]], dtype=torch.float64)


def se3(R, t):
    T = torch.eye(4, dtype=torch.float64)
    T[:3, :3], T[:3, 3] = R, torch.as_tensor(t, dtype=torch.float64)
    return T


SCANS = 9
SPLIT = 5   # F's two parts move together up to scan SPLIT and apart after it


def sensor(t):
    return se3(rot_z(1.0 * t), [1.0 * t, 0.2 * t, 0.0])


def boxes(t, every=False):
    """{name: (world pose [4,4], local box (lo, hi))} of the boxes present at scan t (every: also those absent, whose pose
    still moves the points of a scan they are in towards the next).  A runs through; B enters at scan 3; C leaves after scan
    4; D and E pass each other at scan 4 with 0.3 m between them; F1 (2/3) and F2 (1/3) are one box until scan SPLIT, then
    F2 moves away sideways."""
    out = {'A': (se3(rot_z(2.0 * t), [5.0 + 1.5 * t, -4.0, 0.0]), ((-1.0, -0.5, -0.5), (1.0, 0.5, 0.5)))}
    if t >= 3 or every:
        out['B'] = (se3(rot_z(-3.0 * t), [-6.0 + 0.8 * t, 9.0 - 0.2 * t, 0.0]), ((-1.0, -0.5, -0.5), (1.0, 0.5, 0.5)))
    if t <= 4 or every:
        out['C'] = (se3(torch.eye(3, dtype=torch.float64), [12.0 - 1.0 * t, 8.0, 0.0]), ((-1.0, -0.5, -0.5), (1.0, 0.5, 0.5)))
    out['D'] = (se3(torch.eye(3, dtype=torch.float64), [-10.0 + 2.0 * t, 2.0, 0.0]), ((-1.0, -0.5, -0.5), (1.0, 0.5, 0.5)))
    out['E'] = (se3(rot_z(180.0), [6.0 - 2.0 * t, 3.3, 0.0]), ((-1.0, -0.5, -0.5), (1.0, 0.5, 0.5)))
    F = se3(rot_z(1.5 * t), [-5.0 + 1.2 * t, -10.0, 0.0])
    out['F1'] = (F, ((-1.5, -0.5, -0.5), (0.5, 0.5, 0.5)))
    F2 = F if t <= SPLIT else se3(torch.eye(3, dtype=torch.float64), [0.6 * (t - SPLIT), -1.5 * (t - SPLIT), 0.0]) @ F
    out['F2'] = (F2, ((0.5, -0.5, -0.5), (1.5, 0.5, 0.5)))
    return out


DENSITY = 300.0   # points per cubic metre of a box: about 0.15 m apart, well inside the clustering radius


def scan(g, t):
    """Scan t in its sensor frame: a re-sampled static scene and boxes -> (points [n,3] f64, owner names per point
    ('' static), their world points)."""
    pts, owner = [], []
    ground = torch.rand(5000, 3, generator=g, dtype=torch.float64) * torch.tensor([50.0, 40.0, 0.0]) - torch.tensor([20.0, 20.0, 1.5])
    walls = torch.rand(3000, 3, generator=g, dtype=torch.float64) * torch.tensor([50.0, 0.0, 4.0]) + torch.tensor([-20.0, 0.0, -1.5])
    walls[:, 1] = torch.where(torch.rand(3000, generator=g) < 0.5, -20.0, 20.0).double()
    pts += [ground, walls]
    owner += [''] * 8000
    for name, (T, (lo, hi)) in sorted(boxes(t).items()):
        lo, hi = torch.tensor(lo, dtype=torch.float64), torch.tensor(hi, dtype=torch.float64)
        k = int(DENSITY * float((hi - lo).prod()))
        local = lo + torch.rand(k, 3, generator=g, dtype=torch.float64) * (hi - lo)
        pts.append(local @ T[:3, :3].T + T[:3, 3])
        owner += [name] * k
    world = torch.cat(pts)
    S = torch.linalg.inv(sensor(t))
    return world @ S[:3, :3].T + S[:3, 3], owner, world


def true_flow(world, owner, t):
    """Each point's displacement from scan t to scan t + 1 in the sensor frames: static points stay in the world, a box's
    points ride on its pose."""
    nxt, now = boxes(t + 1, every=True), boxes(t)
    moved = world.clone()
    for name in set(owner) - {''}:
        sel = torch.tensor([o == name for o in owner])
        M = nxt[name][0] @ torch.linalg.inv(now[name][0])
        moved[sel] = world[sel] @ M[:3, :3].T + M[:3, 3]
    S1, S0 = torch.linalg.inv(sensor(t + 1)), torch.linalg.inv(sensor(t))
    return (moved @ S1[:3, :3].T + S1[:3, 3]) - (world @ S0[:3, :3].T + S0[:3, 3])


def key(name, t):
    """The true object a box's points belong to at scan t: F1 is F, and so is F2 until it moves apart."""
    return 'F' if name == 'F1' or (name == 'F2' and t < SPLIT) else name


def true_pose(name, born, t):
    """The motion of a box from sensor frame `born` to sensor frame t."""
    return torch.linalg.inv(sensor(t)) @ boxes(t)[name][0] @ torch.linalg.inv(boxes(born)[name][0]) @ sensor(born)


def sequence(seeds, noise):
    """Per scan t < SCANS - 1: (x [B,n,3] f32, flow [B,n,3] f32, owners of sample 0) with one sequence per seed; the
    seeds share the scene (same point counts), not the sampling or the noise."""
    gs = [torch.Generator().manual_seed(s) for s in seeds]
    out = []
    for t in range(SCANS - 1):
        xs, fs = [], []
        for g in gs:
            x, owner, world = scan(g, t)
            f = true_flow(world, owner, t) + torch.randn(len(owner), 3, generator=g, dtype=torch.float64) * noise
            xf = x.float()
            xs.append(xf)
            fs.append((x + f - xf.double()).float())
        out.append((torch.stack(xs), torch.stack(fs), owner))
    return out


def detect(x, f):
    import pvraft_b200
    ego = pvraft_b200.rigid_motion(x, f)
    obj = pvraft_b200.rigid_objects(x, f, mask=~ego.inliers, radius=0.5, min_points=20, max_objects=16, flow_radius=0.3)
    return ego, obj


def corners(name, t):
    lo, hi = boxes(t)[name][1]
    c = torch.tensor([[(lo, hi)[i >> k & 1][k] for k in range(3)] for i in range(8)], dtype=torch.float64)
    T = torch.linalg.inv(sensor(t)) @ boxes(t)[name][0]
    return c @ T[:3, :3].T + T[:3, 3]


@pytest.mark.parametrize('noise', [0.0, 0.01])
def test_sequence_keeps_identities_and_composes_poses(dev, noise):
    """Every true object keeps one id over its life and no id is reused.  Pose tolerance: a least-squares rigid fit over n
    points with flow noise sigma errs at those points by about sigma sqrt(6 / n) (six degrees of freedom); a pose composed
    over k fits errs by at most the sum (each later fit is rigid), so the corners of a box must lie within 5 k sigma
    sqrt(6 / n_min) of the truth, plus 2e-4 m for fp32 coordinates.  The noise-free rotations agree to 1e-5 per step."""
    import pvraft_b200
    seq = sequence([7], noise)
    tr = pvraft_b200.ObjectTracker()
    ids, born, retired = {}, {}, set()
    n_min = min(int(DENSITY * 1.0), int(DENSITY * 2.0))
    worst_rot, worst_pt = 0.0, 0.0
    for t, (x, f, owner) in enumerate(seq):
        x, f = x.to(dev), f.to(dev)
        ego, obj = detect(x, f)
        out = tr.step(x, f, obj, ego)
        labels = out.labels[0].cpu()
        present = sorted(set(owner) - {''})
        for name in present:
            sel = torch.tensor([o == name for o in owner])
            got = torch.unique(labels[sel])
            assert got.numel() == 1 and int(got) >= 0, (t, name, got.tolist())
            tid = int(got)
            k_ = key(name, t)
            if k_ not in ids:
                assert tid not in retired and tid not in ids.values(), (t, name, tid)
                ids[k_], born[k_] = tid, t
            assert ids[k_] == tid, (t, name, tid, ids)
            slot = int((out.track_id[0] == tid).nonzero()[0, 0])
            assert int(out.age[0, slot]) == t - born[k_]
            truth = true_pose(name, born[k_], t)
            R, tt = out.rotation[0, slot].cpu().double(), out.translation[0, slot].cpu().double()
            c0 = corners(name, born[k_])
            err = float(((c0 @ R.T + tt) - (c0 @ truth[:3, :3].T + truth[:3, 3])).norm(dim=1).max())
            rot = float((R - truth[:3, :3]).abs().max())
            worst_rot, worst_pt = max(worst_rot, rot), max(worst_pt, err)
            k = t - born[k_]
            if noise == 0.0:
                assert rot < 1e-5 * max(k, 1) and err < 2e-4, (t, name, rot, err)
            else:
                assert err < 5 * k * noise * math.sqrt(6 / n_min) + 2e-4, (t, name, err)
        gone = {ids[n] for n in ids if n not in {key(p, t) for p in present}}
        retired |= gone
        assert not (set(out.track_id[0].tolist()) - {-1}) & retired, t
    assert set(ids) == {'A', 'B', 'C', 'D', 'E', 'F', 'F2'} and born['B'] == 3 and born['F2'] == SPLIT
    print(f'noise {noise}: worst rotation entry error {worst_rot:.2e}, worst corner error {worst_pt:.2e} m')


# ---- 4. repeatability, batching, synchronisation, capture ---------------------------------------------------------------------
def run_tracker(dev, inputs, sl=slice(None)):
    import pvraft_b200
    tr = pvraft_b200.ObjectTracker()
    outs = []
    for x, f, ego, obj in inputs:
        pick = lambda nt: type(nt)(*(v[sl] for v in nt))   # noqa: E731
        outs.append(tr.step(x[sl], f[sl], pick(obj), pick(ego)))
    return outs


@pytest.mark.parametrize('mode', ['default', 'deterministic'])
def test_repeatable_and_batched_equals_per_sample(dev, mode, request):
    if mode == 'deterministic':
        request.getfixturevalue('det')
    seq = sequence([11, 12, 13], 0.01)[:5]
    inputs = []
    for x, f, _ in seq:
        x, f = x.to(dev), f.to(dev)
        inputs.append((x, f) + detect(x, f))
    a, b = run_tracker(dev, inputs), run_tracker(dev, inputs)
    for p, q in zip(a, b):
        assert all(same_bits(u, v) for u, v in zip(p, q))
    for s in range(3):
        one = run_tracker(dev, inputs, slice(s, s + 1))
        for p, q in zip(one, a):
            assert all(same_bits(u[0], v[s]) for u, v in zip(p, q)), s
    assert int(a[-1].age.max()) == 4


def test_step_never_synchronises(dev):
    seq = sequence([21], 0.01)[:3]
    inputs = []
    for x, f, _ in seq:
        x, f = x.to(dev), f.to(dev)
        inputs.append((x, f) + detect(x, f))
    import pvraft_b200
    tr = pvraft_b200.ObjectTracker()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for x, f, ego, obj in inputs:
            tr.step(x, f, obj, ego)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert int(tr._next_id[0]) == 5   # A, C, D, E and F: B enters later


def test_captured_call_equals_eager(dev):
    from pvraft_b200 import ops
    g = torch.Generator().manual_seed(30)
    b, o_prev, o = 2, 24, 40
    counts = torch.randint(1, 4, (b, o, o_prev), generator=g) * (torch.rand(b, o, o_prev, generator=g) < 0.12)
    prev, x, lab, num, nn = planted(g, dev, o_prev, o, counts, torch.randint(0, 3, (b, o), generator=g), [o, 17])
    nid0 = torch.tensor([4, 9], dtype=torch.int32, device=dev)
    next_id = nid0.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.track_objects(prev, x, lab, num, o, nn, 0.5, 0.5, next_id)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = ops.track_objects(prev, x, lab, num, o, nn, 0.5, 0.5, next_id)
    next_id.copy_(nid0)
    graph.replay()
    eager_id = nid0.clone()
    eager = ops.track_objects(prev, x, lab, num, o, nn, 0.5, 0.5, eager_id)
    assert all(same_bits(p, q) for p, q in zip(static, eager)) and torch.equal(next_id, eager_id)


# ---- 5. large clouds -------------------------------------------------------------------------------------------------------------
def test_grid_search_at_131072_points_equals_brute_force(dev):
    from pvraft_b200 import ops
    g = torch.Generator().manual_seed(40)
    b, n, o = 1, 131072, 64
    assert ops.use_grid_search('flow_propagate', n)
    xp = (torch.rand(b, n, 3, generator=g) * torch.tensor([80.0, 80.0, 4.0])).to(dev)
    gp = (torch.randn(b, n, 3, generator=g) * 0.3).to(dev)
    x = (torch.rand(b, n, 3, generator=g) * torch.tensor([80.0, 80.0, 4.0])).to(dev)
    lp = (torch.arange(n, dtype=torch.int32)[None] * o // n).to(dev)
    lab = ((x[..., 0] / 80.0 * o).clamp(0, o - 1)).to(torch.int32)
    num = torch.tensor([o], dtype=torch.int32, device=dev)
    prev = random_prev(g, b, n, o, dev, xp, gp, lp)
    outs = []
    for grid in (True, False):
        nn = ops.flow_propagate(xp, gp, x, k=1, want_idx=True, use_grid=grid)[1].view(b, n).contiguous()
        outs.append((nn,) + ops.track_objects(prev, x, lab, num, o, nn, 0.5, 0.5, torch.zeros(b, dtype=torch.int32, device=dev)))
    assert all(same_bits(p, q) for p, q in zip(*outs))
    assert int(outs[0][1].sum()) > 1000
