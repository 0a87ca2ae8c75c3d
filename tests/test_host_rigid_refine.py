"""The refinement of rigid fits against the second scan without a GPU: the entry points are declared, bound and size their
workspaces, and refuse bad arguments before any launch; pvraft_b200.rigid_refine refuses bad clouds, fits, masks and
parameters with ValueError; and a float64 numpy restatement of the whole point-to-plane ICP (fp32 where the kernels
decide: the move and the diff_sq gate) recovers the motions of a synthetic LiDAR-like scene from noisy and from biased
flow fits -- the accuracy the GPU tests then assert of the kernels.

    normal of target j:  eigenvector of the smallest eigenvalue of its k nearest targets' covariance, valid when
                         lambda0 < lambda1 / 4
    match of member i:   nearest valid target of p = R (x - c_x) + c_y (fp32) on (diff_sq, id), diff_sq <= fl(max_distance^2)
    step:                z = -sum_{lambda > 1e-4 lambda_max} (v . g) / lambda v of the rho-scaled J^T J, g = J^T r
"""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 256   # never dereferenced: every call below fails its argument check
BAD = -1
NAMES = ('pvraft_rigid_refine_fwd', 'pvraft_rigid_refine_workspace_bytes', 'pvraft_rigid_refine_det_workspace_bytes')
KAPPA, RANK_TOL, CONVERGED = 0.25, 1e-4, 1e-6


def r16(v):
    return (v + 15) // 16 * 16


# ---- numpy restatement ---------------------------------------------------------------------------------------------------
def diff_sq32(a, b):
    """fp32 (dx dx + dy dy) + dz dz of broadcastable [..., 3] float32 arrays, every operation rounded."""
    d = (a - b).astype(np.float32)
    return ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(np.float32)


def targets_of(x2, mask=None):
    on = np.isfinite(x2).all(1)
    return on if mask is None else on & mask


def normals_ref(x2, k, mask=None, chunk=512):
    """-> (normals [M,3] float64, valid [M] bool, neighbours [M,k] int (-1 for a point that is no target))."""
    x2 = x2.astype(np.float32)
    on = targets_of(x2, mask)
    ids = np.nonzero(on)[0]
    T = x2[ids]
    M = len(x2)
    nrm, valid, nbr = np.zeros((M, 3)), np.zeros(M, bool), -np.ones((M, k), np.int64)
    for c0 in range(0, len(ids), chunk):
        q = T[c0:c0 + chunk]
        D = diff_sq32(q[:, None, :], T[None, :, :])
        order = np.argsort(D, axis=1, kind='stable')[:, :k]   # stable: ties by id (ids ascending)
        for r, j in enumerate(ids[c0:c0 + chunk]):
            if len(ids) < k:
                continue
            nb = ids[order[r]]
            nbr[j] = nb
            d = x2[nb].astype(np.float64) - x2[j].astype(np.float64)
            e = d - d.mean(0)
            lam, V = np.linalg.eigh(e.T @ e)
            nrm[j] = V[:, 0]
            valid[j] = lam[0] < KAPPA * lam[1]
    return nrm, valid, nbr


def rodrigues(w):
    th = np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    a = np.sin(th) / th if th > 0 else 1.0
    b = 2 * (np.sin(th / 2) / th) ** 2 if th > 0 else 0.5
    return np.eye(3) + a * K + b * (K @ K)


def move32(R, cx, cy, x):
    """p = R (x - c_x) + c_y in fp32 with the kernel's order; R, c_x, c_y rounded from double."""
    m, cxf, cyf = R.astype(np.float32), cx.astype(np.float32), cy.astype(np.float32)
    d = (x - cxf).astype(np.float32)
    return np.stack([((m[k, 0] * d[:, 0] + m[k, 1] * d[:, 1]) + m[k, 2] * d[:, 2]) + cyf[k] for k in range(3)], 1).astype(np.float32)


def match_ref(p, x2, valid, max_distance, chunk=1024):
    """Nearest valid target of each p on (diff_sq, id) within fl(max_distance^2) -> ids (-1 for none)."""
    r2 = np.float32(max_distance) * np.float32(max_distance)
    ids = np.nonzero(valid)[0]
    Q = x2[ids].astype(np.float32)
    out = -np.ones(len(p), np.int64)
    if len(ids) == 0:
        return out
    for c0 in range(0, len(p), chunk):
        D = diff_sq32(p[c0:c0 + chunk, None, :], Q[None, :, :])
        D = np.where(D <= r2, D, np.inf)   # NaN and beyond the gate
        j = np.argmin(D, axis=1)           # the first minimum: the lowest id
        hit = np.isfinite(D[np.arange(len(j)), j])
        out[c0:c0 + chunk] = np.where(hit, ids[j], -1)
    return out


def solve_ref(p, q, n, cy, rho):
    """The degeneracy-aware step from correspondences (p, q, n fp32 values as float64) -> (z [6], rank, eigvals, V)."""
    p, q, n = p.astype(np.float64), q.astype(np.float64), n.astype(np.float64)
    a = p - cy.astype(np.float32).astype(np.float64)
    J = np.concatenate([np.cross(a, n), n], 1)
    r = ((p - q) * n).sum(1)
    s = np.array([1 / rho] * 3 + [1.0] * 3)
    H = (J.T @ J) * s[:, None] * s[None, :]
    g = (J.T @ r) * s
    lam, V = np.linalg.eigh(H)
    keep = lam > RANK_TOL * lam.max()
    z = -(V[:, keep] @ ((V[:, keep].T @ g) / lam[keep]))
    return z, int(keep.sum()), lam, V


def icp_ref(x1, x2, members, R0, t0, max_distance=0.3, iterations=10, k_normal=16, target_mask=None, normals=None):
    """The whole refinement of one segment -> dict(R, t, history [(R, c_y)], rank, steps, matched, corr, rho)."""
    x1 = x1.astype(np.float32)
    nrm, valid, _ = normals if normals is not None else normals_ref(x2, k_normal, target_mask)
    mem = members & np.isfinite(x1).all(1)
    X = x1[mem]
    cx = X.astype(np.float64).mean(0)
    rho = np.sqrt(((X - cx) ** 2).sum(1).mean()) or 1.0
    R, cy = R0.astype(np.float64), R0.astype(np.float64) @ cx + t0.astype(np.float64)
    hist, rank, steps, matched, corr = [(R.copy(), cy.copy())], 0, 0, 0, None
    for _ in range(iterations):
        p = move32(R, cx, cy, X)
        corr = match_ref(p, x2, valid, max_distance)
        hit = corr >= 0
        matched = int(hit.sum())
        if matched < 6:
            rank = 0
            hist.append((R.copy(), cy.copy()))
            continue
        z, rank, _, _ = solve_ref(p[hit], x2[corr[hit]], nrm[corr[hit]].astype(np.float32), cy, rho)
        R = rodrigues(z[:3] / rho) @ R
        cy = cy + z[3:]
        steps += 1
        hist.append((R.copy(), cy.copy()))
        if np.linalg.norm(z[:3]) + np.linalg.norm(z[3:]) <= CONVERGED:
            break
    return dict(R=R, t=cy - R @ cx, history=hist, rank=rank, steps=steps, matched=matched, corr=corr, rho=rho, cx=cx)


def kabsch(x, y):
    """The least-squares rigid motion x -> y (float64)."""
    cx, cy = x.mean(0), y.mean(0)
    U, _, Vt = np.linalg.svd((x - cx).T @ (y - cy))
    D = np.diag([1, 1, np.sign(np.linalg.det(Vt.T @ U.T))])
    R = Vt.T @ D @ U.T
    return R, cy - R @ cx


def rot_deg(Ra, Rb):
    return float(np.degrees(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1) / 2, -1, 1))))


def yaw(deg):
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


# ---- the synthetic scene -------------------------------------------------------------------------------------------------
BOXES = ((np.array([4.0, 3.0, 0.0]), np.array([4.0, 1.8, 1.6])), (np.array([-5.0, -4.0, 0.0]), np.array([4.5, 2.0, 1.8])))
BOX_MOTIONS = ((yaw(4.0), np.array([1.2, 0.3, 0.0])), (yaw(-3.0), np.array([-0.8, 1.0, 0.0])))
EGO = (yaw(1.5) @ np.array([[1, 0, 0], [0, np.cos(0.01), -np.sin(0.01)], [0, np.sin(0.01), np.cos(0.01)]]), np.array([0.9, 0.15, 0.03]))


def sample_static(rng, n):
    """Ground (z = 0, 30 x 30 m) and three walls (x = -14, x = 14, y = 12, 3 m high)."""
    k = rng.integers(0, 4, n)
    u, v = rng.uniform(-15, 15, n), rng.uniform(0, 3, n)
    g = np.stack([rng.uniform(-15, 15, n), rng.uniform(-15, 15, n), np.zeros(n)], 1)
    w0 = np.stack([np.full(n, -14.0), u, v], 1)
    w1 = np.stack([np.full(n, 14.0), u, v], 1)
    w2 = np.stack([u * 0.9, np.full(n, 12.0), v], 1)
    pick = np.where(k[:, None] == 0, g, np.where(k[:, None] == 1, w0, np.where(k[:, None] == 2, w1, w2)))
    return np.where((k == 0)[:, None] & (rng.random(n) < 0.6)[:, None], g, pick)


def sample_box(rng, n, centre, size):
    """Points on the four sides and the top of a box standing on the ground."""
    face = rng.integers(0, 5, n)
    u, v = rng.random(n), rng.random(n)
    lo = centre - size * np.array([0.5, 0.5, 0.0])
    pts = np.empty((n, 3))
    for f, (a, b, c, val) in enumerate(((1, 2, 0, 0.0), (1, 2, 0, 1.0), (0, 2, 1, 0.0), (0, 2, 1, 1.0), (0, 1, 2, 1.0))):
        sel = face == f
        pts[sel, a] = lo[a] + u[sel] * size[a]
        pts[sel, b] = lo[b] + v[sel] * size[b]
        pts[sel, c] = lo[c] + val * size[c]
    return pts


def transform(R, t, x):
    return x @ R.T + t


def scene(seed, n_static=4000, n_box=1500, noise=0.01):
    """A pair of scans of a static scene seen from a moving sensor, with two boxes that move on their own.  xyz2 is
    sampled independently of xyz1 (no exact point pairs) from the moved surfaces, with `noise` metres of Gaussian noise.
    -> dict(xyz1, xyz2 float32, truth [N,3] the true flow, seg [N] (0 static, 1 + o box o), motions [(R, t)] per segment)."""
    rng = np.random.default_rng(seed)
    Re, te = EGO
    x1, x2, seg, motions = [sample_static(rng, n_static)], [transform(Re, te, sample_static(rng, n_static))], [np.zeros(n_static, int)], [EGO]
    for o, ((c, sz), (Rb, tb)) in enumerate(zip(BOXES, BOX_MOTIONS)):
        # the box moves by (Rb about its centre, tb) in the world; the sensor sees the world through the ego motion
        Rw, tw = Rb, c + tb - Rb @ c
        R, t = Re @ Rw, Re @ tw + te
        x1.append(sample_box(rng, n_box, c, sz))
        x2.append(transform(R, t, sample_box(rng, n_box, c, sz)))
        seg.append(np.full(n_box, 1 + o))
        motions.append((R, t))
    x1, x2, seg = np.concatenate(x1), np.concatenate(x2), np.concatenate(seg)
    # the static scene under a box is hidden in both scans: drop ground points inside a box footprint
    keep1 = np.ones(len(x1), bool)
    for c, sz in BOXES:
        keep1 &= ~((seg == 0) & (np.abs(x1[:, :2] - c[:2]) < sz[:2] / 2).all(1))
    x1, seg = x1[keep1], seg[keep1]
    x2 = x2 + rng.normal(0, noise, x2.shape)
    x1 = x1 + rng.normal(0, noise, x1.shape)
    truth = np.empty_like(x1)
    for s, (R, t) in enumerate(motions):
        truth[seg == s] = transform(R, t, x1[seg == s]) - x1[seg == s]
    perm = rng.permutation(len(x2))
    return dict(xyz1=x1.astype(np.float32), xyz2=x2[perm].astype(np.float32), truth=truth, seg=seg, motions=motions)


def flow_fits(sc, flow):
    """The flow fit of every segment (Kabsch of x -> x + flow on its points; rigid_motion / rigid_objects' role)."""
    x = sc['xyz1'].astype(np.float64)
    return [kabsch(x[sc['seg'] == s], (x + flow)[sc['seg'] == s]) for s in range(len(sc['motions']))]


def errors(fits, motions):
    return [(rot_deg(R, Rt), float(np.linalg.norm(t - tt))) for (R, t), (Rt, tt) in zip(fits, motions)]


# Accuracy the refinement reaches on scene(seed), seeds 0 and 1 (the CPU restatement below), with margin; the GPU tests
# assert the same bounds of the kernels.  Both flows lead to the same fixed point of the ICP: a few mm and under 0.1 degree
# for the static scene, 1-3 cm and under 0.5 degree for the boxes (their 16-neighbour normals straddle the edges).  With
# 3 cm of random noise over thousands of points the flow fit itself is already that close, so only the biased flow is
# required to improve.
REFINED = ((0.1, 0.01), (0.5, 0.05), (0.5, 0.05))   # per segment (static, box 0, box 1): (degrees, metres)
GAIN_BIASED = 5.0                                    # the biased fit's translation error over the refined one, at least


def refine_all(sc, fits, normals=None):
    normals = normals if normals is not None else normals_ref(sc['xyz2'], 16)
    return [icp_ref(sc['xyz1'], sc['xyz2'], sc['seg'] == s, R, t, normals=normals) for s, (R, t) in enumerate(fits)], normals


@pytest.mark.parametrize('seed', [0, 1])
def test_restatement_recovers_the_motions_from_noisy_and_biased_flow(seed):
    sc = scene(seed)
    rng = np.random.default_rng(100 + seed)
    normals = normals_ref(sc['xyz2'], 16)
    for kind in ('noisy', 'biased'):
        flow = sc['truth'] + rng.normal(0, 0.03, sc['truth'].shape) if kind == 'noisy' else 0.8 * sc['truth']
        fits = flow_fits(sc, flow)
        before = errors(fits, sc['motions'])
        out, _ = refine_all(sc, fits, normals)
        after = errors([(o['R'], o['t']) for o in out], sc['motions'])
        for s, ((rb, tb), (ra, ta), o) in enumerate(zip(before, after, out)):
            assert ra < REFINED[s][0] and ta < REFINED[s][1], (kind, s, before[s], after[s], o['steps'], o['rank'])
            assert o['rank'] == 6
            if kind == 'biased':   # the flow fit is 20 % short of the motion
                assert tb > 0.15 * np.linalg.norm(sc['motions'][s][1]) and ta * GAIN_BIASED < tb, (s, tb, ta)


def test_restatement_leaves_unobservable_directions_alone():
    """A noise-free ground plane alone constrains z, roll and pitch only: rank 3, and the steps have no component along x,
    y or yaw; two parallel walls (clear of the ground, so that no normal mixes the two) and the ground leave only the
    translation along the walls free: rank 5."""
    rng = np.random.default_rng(3)
    g1 = np.stack([rng.uniform(-10, 10, 3000), rng.uniform(-10, 10, 3000), np.zeros(3000)], 1).astype(np.float32)
    g2 = np.stack([rng.uniform(-10, 10, 3000), rng.uniform(-10, 10, 3000), np.zeros(3000)], 1).astype(np.float32)
    R0 = np.array([[1, 0, 0], [0, np.cos(0.01), -np.sin(0.01)], [0, np.sin(0.01), np.cos(0.01)]]) @ yaw(2.0)
    t0 = np.array([0.3, -0.2, 0.05])
    out = icp_ref(g1, g2, np.ones(3000, bool), R0, t0)
    assert out['rank'] == 3
    for (Ra, ca), (Rb, cb) in zip(out['history'][:-1], out['history'][1:]):
        w = Rb @ Ra.T
        assert abs(w[1, 0] - w[0, 1]) / 2 < 1e-9 * out['rho'] + 1e-12   # no yaw step
        assert np.abs((cb - ca)[:2]).max() < 1e-9
    # the plane: z = 0 after the refinement (roll, pitch and z are observed)
    p = transform(out['R'], out['t'], g1.astype(np.float64))
    assert np.abs(p[:, 2]).max() < 1e-4
    walls = np.concatenate([np.stack([np.full(1500, s), rng.uniform(-10, 10, 1500), rng.uniform(1.5, 4.5, 1500)], 1) for s in (-5.0, 5.0)])
    a = np.concatenate([g1, walls.astype(np.float32)])
    walls2 = np.concatenate([np.stack([np.full(1500, s), rng.uniform(-10, 10, 1500), rng.uniform(1.5, 4.5, 1500)], 1) for s in (-5.0, 5.0)])
    b = np.concatenate([g2, walls2.astype(np.float32)])
    out = icp_ref(a, b, np.ones(len(a), bool), yaw(1.0), np.array([0.1, -0.2, 0.05]))
    assert out['rank'] == 5


# ---- the C ABI -----------------------------------------------------------------------------------------------------------
def test_header_declares_and_lib_binds_the_refinement_entry_points():
    from pvraft_b200 import _lib, build
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    for name in NAMES:
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert name in _lib.EXPORTS
    assert [len(_lib._SIGNATURES[n][1]) for n in NAMES] == [28, 5, 3]
    assert 'rigid_refine.cu' in build.SOURCES
    assert [d.pointee for d in _lib.FUNCTIONS['pvraft_rigid_refine_fwd'][1][21:25]] == ['double', 'int32_t', 'float', 'int32_t']


def test_refinement_workspace_sizes():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    b, n, m, o, it = 3, 1001, 777, 5, 10
    g = b * o
    assert lib.pvraft_rigid_refine_det_workspace_bytes(b, o, it) == g * (5 + it * 29) * 24
    for bad in ((0, o, it), (b, 0, it), (b, 257, it), (b, o, 0), (b, o, 65), (65536, 1, it)):
        assert lib.pvraft_rigid_refine_det_workspace_bytes(*bad) == 0, bad
    c = (n + 255) // 256
    s = (n + 1023) // 1024 + o
    grouping = r16(4 * b * n) + 2 * r16(4 * g) + 2 * r16(4 * b * c * o) + r16(4 * b * n) + r16(4 * b) + r16(4 * b * s) + r16(4 * b)
    want = (r16(lib.pvraft_grid_index_workspace_bytes(b, m)) + r16(12 * b * m) + r16(16 * b * m) + grouping + r16(4 * g * 16)
            + r16(8 * g * 21) + r16(8 * g * 5) + r16(8 * it * g * 29))
    assert lib.pvraft_rigid_refine_workspace_bytes(b, n, m, o, it) == want
    # one segment per sample needs no grouping: its windows are the sample's
    want = (r16(lib.pvraft_grid_index_workspace_bytes(b, m)) + r16(12 * b * m) + r16(16 * b * m) + r16(4 * b * 16) + r16(8 * b * 21)
            + r16(8 * b * 5) + r16(8 * it * b * 29))
    assert lib.pvraft_rigid_refine_workspace_bytes(b, n, m, 1, it) == want
    for bad in ((0, n, m, o, it), (b, 0, m, o, it), (b, n, 0, o, it), (b, n, m, 0, it), (b, n, m, 257, it), (b, n, m, o, 0),
                (b, n, m, o, 65), (1 << 16, 1 << 15, m, 1, it), (300, n, m, 256, it)):
        assert lib.pvraft_rigid_refine_workspace_bytes(*bad) == 0, bad


def test_refinement_entry_point_refuses_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def fwd(x1=P, x2=P, lab=P, tm=None, Ri=P, ti=P, di=P, B=2, N=64, M=64, O=4, it=10, md=0.3, k=16, R=P, t=P, d=P, mt=P, rm=P,
            rk=P, sp=P, ws=P):
        return lib.pvraft_rigid_refine_fwd(x1, x2, lab, tm, Ri, ti, di, B, N, M, O, it, md, k, R, t, d, mt, rm, rk, sp, None, None,
                                           None, None, ws, None, None)

    nan, inf = float('nan'), float('inf')
    cases = (dict(B=0), dict(N=0), dict(M=0), dict(O=0), dict(O=257), dict(B=300, O=256), dict(B=1 << 16, N=1 << 15, O=1),
             dict(B=1 << 16, M=1 << 15, O=1), dict(it=0), dict(it=65), dict(md=0.0), dict(md=-0.3), dict(md=nan), dict(md=inf),
             dict(md=1e20), dict(k=2), dict(k=33), dict(M=8, k=9), dict(lab=None))
    for kw in cases:
        assert fwd(**kw) == BAD, kw
        assert b'rigid_refine_fwd' in lib.pvraft_last_error_string()
    for name in ('x1', 'x2', 'Ri', 'ti', 'di', 'R', 't', 'd', 'mt', 'rm', 'rk', 'sp', 'ws'):
        assert fwd(**{name: None}) == BAD, name
    assert fwd(ws=P + 8) == BAD   # unaligned workspace


def test_public_function_refuses_bad_arguments():
    import pvraft_b200
    from pvraft_b200._lib import PvraftError
    b, n, m, o = 2, 50, 40, 4
    x1, x2 = torch.rand(b, n, 3), torch.rand(b, m, 3)
    ego = pvraft_b200.RigidMotion(torch.eye(3).expand(b, 3, 3), torch.zeros(b, 3), torch.ones(b, n, dtype=torch.bool),
                                  torch.zeros(b, dtype=torch.int32), torch.zeros(b, dtype=torch.bool))
    obj = pvraft_b200.RigidObjects(torch.zeros(b, n, dtype=torch.int32), torch.ones(b, dtype=torch.int32), torch.eye(3).expand(b, o, 3, 3),
                                   torch.zeros(b, o, 3), torch.zeros(b, o, dtype=torch.int32), torch.zeros(b, o, dtype=torch.bool),
                                   torch.ones(b, n, dtype=torch.bool))
    calls = [dict(xyz1=x1[..., :2], xyz2=x2, fit=ego), dict(xyz1=x1, xyz2=x2[..., :2], fit=ego), dict(xyz1=x1.long(), xyz2=x2, fit=ego),
             dict(xyz1=x1, xyz2=x2[:1], fit=ego), dict(xyz1=x1[:, :0], xyz2=x2, fit=ego), dict(xyz1=x1, xyz2=x2[:, :0], fit=ego),
             dict(xyz1=x1, xyz2=x2, fit=None), dict(xyz1=x1, xyz2=x2, fit=(ego.rotation, ego.translation)),
             dict(xyz1=x1[:, :49], xyz2=x2, fit=ego), dict(xyz1=x1[:, :49], xyz2=x2, fit=obj),
             dict(xyz1=x1, xyz2=x2, fit=ego._replace(rotation=torch.eye(3).expand(b, 1, 3, 3))),
             dict(xyz1=x1, xyz2=x2, fit=obj._replace(translation=torch.zeros(b, o + 1, 3))),
             dict(xyz1=x1, xyz2=x2, fit=obj._replace(degenerate=torch.zeros(b, dtype=torch.bool))),
             dict(xyz1=x1, xyz2=x2, fit=obj._replace(degenerate=torch.zeros(b, o, dtype=torch.int32))),
             dict(xyz1=x1, xyz2=x2, fit=obj._replace(inliers=torch.ones(b, n))), dict(xyz1=x1, xyz2=x2, fit=obj._replace(labels=obj.labels.float())),
             dict(xyz1=x1, xyz2=x2, fit=ego._replace(inliers=torch.ones(b, n, dtype=torch.uint8))),
             dict(xyz1=x1, xyz2=x2, fit=ego._replace(rotation=torch.eye(3, dtype=torch.int32).expand(b, 3, 3))),
             dict(xyz1=x1, xyz2=x2, fit=ego, target_mask=torch.ones(b, m)), dict(xyz1=x1, xyz2=x2, fit=ego, target_mask=torch.ones(b, n, dtype=torch.bool)),
             dict(xyz1=x1, xyz2=x2, fit=ego, target_mask=[True] * m)]
    calls += [dict(xyz1=x1, xyz2=x2, fit=ego, iterations=v) for v in (0, 65, 2.0, True, None)]
    calls += [dict(xyz1=x1, xyz2=x2, fit=ego, max_distance=v) for v in (0.0, -0.3, float('nan'), float('inf'), True, '0.3', 1e20)]
    calls += [dict(xyz1=x1, xyz2=x2, fit=ego, k_normal=v) for v in (2, 33, 41, 16.0, True, None)]
    for kw in calls:
        with pytest.raises(ValueError, match='rigid_refine'):
            pvraft_b200.rigid_refine(**kw)
    with pytest.raises(ValueError, match='rigid_refine'):   # k_normal above M
        pvraft_b200.rigid_refine(x1, x2[:, :10], ego, k_normal=11)
    with pytest.raises(PvraftError):
        pvraft_b200.rigid_refine(x1, x2, ego)
    with pytest.raises(PvraftError):
        pvraft_b200.rigid_refine(x1, x2, obj, target_mask=torch.ones(b, m, dtype=torch.bool), iterations=64, max_distance=1.0, k_normal=32)
    assert pvraft_b200.RigidRefinement._fields == ('fit', 'matched', 'rmse', 'rank', 'steps')
