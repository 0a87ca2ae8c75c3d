"""The rigid-motion fit (csrc/rigid_motion.cu, pvraft_b200.rigid_motion): the sampler bit for bit against a numpy uint64
restatement of the hash and the rejection tests, the counts and the selection against a float64 restatement, exact recovery of
noise-free motions, robustness to moving objects, the refit against a float64 Horn fit, degenerate samples, gradients against
float64 autograd through a torch Horn fit, determinism and batching, graph capture, and a training step of the model.

    j_r = splitmix64((seed << 32) | (h << 2) | r) mod n_allowed   (r = 0, 1, 2: an index into the ascending allowed points)
    model (R, c_x, c_y) = Horn's fit of the triple about its centroids;  inlier: ||R (x - c_x) - (y - c_y)||^2 <= threshold^2
    refit: Horn on the inliers, `rounds` times;  t = y-bar - R x-bar
"""
import math
import types

import numpy as np
import pytest
import torch

from conftest import default_weights
from oracle import pvraft_oracle as O
from train_helpers import compare_grads, oracle_adjacency

pytestmark = pytest.mark.gpu

M64 = (1 << 64) - 1


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
    a, b = a.detach().contiguous(), b.detach().contiguous()
    if a.is_floating_point():
        a, b = (t.view(torch.int64 if t.element_size() == 8 else torch.int32) for t in (a, b))
    return torch.equal(a, b)


# ---- host restatements ---------------------------------------------------------------------------------------------------
def splitmix64(k):
    z = (k + 0x9e3779b97f4a7c15) & M64
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & M64
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & M64
    return z ^ (z >> 31)


def draws(seed, h_count, n_allowed):
    """[H,3] positions in the allowed list, in uint64 arithmetic."""
    return np.array([[splitmix64((seed << 32) | (h << 2) | r) % n_allowed for r in range(3)] for h in range(h_count)], np.int64)


def rejected(x, y, thr):
    """The triple tests in float64 (numpy rounds every operation and never contracts): x, y [3,3] float64."""
    a, b = x[1] - x[0], x[2] - x[0]
    c = np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])
    d3 = lambda u: (u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]   # noqa: E731
    if not d3(c) > (1e-6 * d3(a)) * d3(b):
        return True
    for i, j in ((0, 1), (0, 2), (1, 2)):
        if not abs(math.sqrt(d3(x[i] - x[j])) - math.sqrt(d3(y[i] - y[j]))) <= 2.0 * thr:
            return True
    return False


def rotq(q):
    w, x, y, z = q
    return np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


def horn_np(x, y):
    """float64 Horn fit -> (R, x-bar, y-bar)."""
    xb, yb = x.mean(0), y.mean(0)
    S = (x - xb).T @ (y - yb)
    (xx, xy, xz), (yx, yy, yz), (zx, zy, zz) = S
    N = np.array([[xx + yy + zz, yz - zy, zx - xz, xy - yx], [yz - zy, xx - yy - zz, xy + yx, zx + xz],
                  [zx - xz, xy + yx, -xx + yy - zz, yz + zy], [xy - yx, zx + xz, yz + zy, -xx - yy + zz]])
    _, V = np.linalg.eigh(N)
    return rotq(V[:, -1]), xb, yb


def horn_torch(x, y):
    """The same fit in torch (differentiable through torch.linalg.eigh): x, y [n,3] float64 -> (R, t)."""
    xb, yb = x.mean(0), y.mean(0)
    S = (x - xb).T @ (y - yb)
    xx, xy, xz, yx, yy, yz, zx, zy, zz = S.reshape(9)
    N = torch.stack([torch.stack([xx + yy + zz, yz - zy, zx - xz, xy - yx]), torch.stack([yz - zy, xx - yy - zz, xy + yx, zx + xz]),
                     torch.stack([zx - xz, xy + yx, -xx + yy - zz, yz + zy]), torch.stack([xy - yx, zx + xz, yz + zy, -xx - yy + zz])])
    _, V = torch.linalg.eigh(N)
    w, a, b, c = V[:, -1]
    R = torch.stack([torch.stack([w * w + a * a - b * b - c * c, 2 * (a * b - w * c), 2 * (a * c + w * b)]),
                     torch.stack([2 * (a * b + w * c), w * w - a * a + b * b - c * c, 2 * (b * c - w * a)]),
                     torch.stack([2 * (a * c - w * b), 2 * (b * c + w * a), w * w - a * a - b * b + c * c])])
    return R, yb - R @ xb


def resid2(R, cx, cy, x, y):
    return (((x - cx) @ R.T - (y - cy)) ** 2).sum(-1)


def random_rotation(g, max_deg):
    axis = torch.randn(3, generator=g, dtype=torch.float64)
    axis = axis / axis.norm()
    ang = math.radians(max_deg) * float(torch.rand(1, generator=g, dtype=torch.float64))
    K = torch.tensor([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]], dtype=torch.float64)
    return torch.eye(3, dtype=torch.float64) + math.sin(ang) * K + (1 - math.cos(ang)) * K @ K


def cloud(n, kind, g, shift=0.0):
    """[n,3] float64: 'uniform' in [-20, 20]^3, or 'lidar' (the distribution of test_gpu_grid_search.cloud): rings on a ground
    plane, dense clusters and a sparse far range."""
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)   # noqa: E731
    if kind == 'uniform':
        x = r(n, 3) * 40 - 20
    else:
        n1, n2 = n // 2, n // 4
        n3 = n - n1 - n2
        ring = torch.randint(0, 32, (n1,), generator=g).double()
        rad = 3 + ring * 1.5 + r(n1) * 0.02
        th = r(n1) * 2 * math.pi
        ground = torch.stack([rad * torch.cos(th), rad * torch.sin(th), -1.7 + r(n1) * 0.05], 1)
        ctr = (r(8, 3) * 30 - 15)[torch.randint(0, 8, (n2,), generator=g)]
        clusters = ctr + torch.randn(n2, 3, generator=g, dtype=torch.float64) * 0.3
        far = torch.cat([r(n3, 2) * 160 - 80, r(n3, 1) * 6 - 2], 1)
        x = torch.cat([ground, clusters, far])[torch.randperm(n, generator=g)]
    return x + shift


def rigid_flow(x64, R, t):
    """fp32 xyz1 and flow of the motion y = R x + t."""
    x = x64.float()
    return x, ((x.double() @ R.T + t) - x.double()).float()


def yf32(x, f):
    return (x.float() + f.float()).double()


def rot_err(Ra, Rb):
    """The angle of Ra^T Rb, from atan2 of its sine (the skew part) and cosine: arccos of the trace alone loses half the
    digits near zero."""
    M = Ra.double().T @ Rb.double()
    sin = 0.5 * float(torch.stack([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]]).norm())
    return math.atan2(sin, (float(torch.trace(M)) - 1) / 2)


def scene(n, g, objects, noise=0.01, shift=0.0):
    """A LiDAR-like pair: ego-motion (R_e, t_e) for the static scene, and `objects` = fractions of the points, each a cluster
    moving by the ego-motion plus its own translation of 0.5 to 2 m -> (xyz1, flow fp32, R_e, t_e, moving mask)."""
    x = cloud(n, 'lidar', g, shift)
    R, t = random_rotation(g, 5.0), (torch.rand(3, generator=g, dtype=torch.float64) * 2 - 1) * 2.0
    y = x @ R.T + t
    moving = torch.zeros(n, dtype=torch.bool)
    start = 0
    perm = torch.randperm(n, generator=g)
    for frac in objects:
        k = int(frac * n)
        idx = perm[start:start + k]
        start += k
        ctr = (torch.rand(3, generator=g, dtype=torch.float64) * 40 - 20) + shift
        x[idx] = ctr + torch.randn(k, 3, generator=g, dtype=torch.float64) * 1.5
        d = torch.randn(3, generator=g, dtype=torch.float64)
        off = d / d.norm() * (0.5 + 1.5 * float(torch.rand(1, generator=g, dtype=torch.float64)))
        y[idx] = x[idx] @ R.T + t + off
        moving[idx] = True
    y = y + torch.randn(n, 3, generator=g, dtype=torch.float64) * noise
    xf = x.float()
    return xf, (y - xf.double()).float(), R, t, moving


def fit(dev, x, f, mask=None, **kw):
    import pvraft_b200
    return pvraft_b200.rigid_motion(x.to(dev), f.to(dev), None if mask is None else mask.to(dev), **kw)


def raw(dev, x, f, mask=None, threshold=0.1, hypotheses=256, rounds=2, seed=0):
    """The one-segment fit rigid_motion makes, with the sampler's triples and counts: (R, t, inliers, count, degenerate,
    state, triples [B,H,3], hypothesis counts [B,H])."""
    from pvraft_b200 import ops
    lab = None if mask is None else torch.add(mask.to(dev), -1).int()
    R, t, inl, count, degen, state, triples, hcount = ops.rigid_objects(x.to(dev).contiguous(), f.to(dev).contiguous(), lab, 1, threshold,
                                                                        hypotheses, rounds, seed, want_samples=True)
    return R[:, 0], t[:, 0], inl, count[:, 0], degen[:, 0], state[:, 0], triples, hcount


# ---- 1. sampler ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('masked', [False, True])
def test_one_segment_sampler_bit_exact(dev, masked):
    g = torch.Generator().manual_seed(1)
    b, n, hc, thr, seed = 2, 3000, 1024, 0.1, 12345
    x = torch.rand(b, n, 3, generator=g) * 10
    f = torch.randn(b, n, 3, generator=g) * 0.05           # random flows: many triples break the distance test
    x[1, :200] = x[1, 200:400]                              # coincident points
    x[1, 400:600, 1] = x[1, 400:600, 0]
    x[1, 400:600, 2] = 2 * x[1, 400:600, 0]                 # a collinear stretch
    mask = torch.rand(b, n, generator=g) < 0.6 if masked else None
    out = raw(dev, x, f, mask, threshold=thr, hypotheses=hc, seed=seed)
    triples, hcount = out[6].cpu().numpy(), out[7].cpu().numpy()
    x64, y64 = x.double().numpy(), yf32(x, f).numpy()
    thr64 = float(np.float32(thr))                          # the fp32 threshold, widened
    nrej = 0
    for s in range(b):
        allowed = np.nonzero(mask[s].numpy())[0] if masked else np.arange(n)
        j = draws(seed, hc, len(allowed))
        assert np.array_equal(triples[s], allowed[j]), s
        for h in range(hc):
            idx = allowed[j[h]]
            rej = len(set(j[h].tolist())) < 3 or rejected(x64[s][idx], y64[s][idx], thr64)
            nrej += rej
            assert (hcount[s, h] == -1) == rej, (s, h)
    print(f'{nrej} of {b * hc} triples rejected')
    assert 0 < nrej < b * hc


# ---- 2. counts and selection ---------------------------------------------------------------------------------------------
def test_one_segment_counts_and_selection_against_float64(dev):
    g = torch.Generator().manual_seed(2)
    n, hc, thr = 4000, 512, 0.5
    x64 = torch.rand(n, 3, generator=g, dtype=torch.float64) * 5
    R, t = random_rotation(g, 20.0), torch.tensor([0.3, -0.2, 0.1], dtype=torch.float64)
    y = x64 @ R.T + t + torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.25
    y[: n // 3] += torch.randn(n // 3, 3, generator=g, dtype=torch.float64) * 2.0
    x = x64.float()
    f = (y - x.double()).float()
    out = raw(dev, x[None], f[None], threshold=thr, hypotheses=hc, rounds=1, seed=7)
    triples, hcount = out[6][0].cpu().numpy(), out[7][0].cpu().numpy()
    xs, ys = x.double().numpy(), yf32(x, f).numpy()
    boundary, checked = 0, 0
    for h in range(hc):
        if hcount[h] < 0:
            continue
        idx = triples[h]
        Rh, cx, cy = horn_np(xs[idx], ys[idx])
        Rh, cx, cy = (v.astype(np.float32).astype(np.float64) for v in (Rh, cx, cy))
        r2 = resid2(Rh, cx, cy, xs, ys)
        edge = np.abs(r2 - thr * thr) <= 1e-5 * thr * thr
        boundary += int(edge.sum())
        lo, hi = int((r2 <= thr * thr)[~edge].sum()), int((r2 <= thr * thr)[~edge].sum() + edge.sum())
        assert lo <= hcount[h] <= hi, (h, hcount[h], lo, hi)
        checked += 1
    print(f'{checked} accepted hypotheses checked, {boundary} boundary (point, hypothesis) pairs exempt')
    best = int(np.argmax(hcount))                                       # the lowest index among the largest
    assert int(out[3][0]) == hcount[best]                               # round 1 refits on the best hypothesis's inliers
    assert checked > hc // 4


# ---- 3. exact recovery ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['uniform', 'lidar'])
@pytest.mark.parametrize('shift', [0.0, 1e3])
def test_exact_recovery(dev, kind, shift):
    g = torch.Generator().manual_seed(3 + int(shift))
    b, n = 3, 8192
    xs, fs, Rs, ts = [], [], [], []
    for _ in range(b):
        R, t = random_rotation(g, 30.0), (torch.rand(3, generator=g, dtype=torch.float64) * 2 - 1) * 5.0
        x, f = rigid_flow(cloud(n, kind, g, shift), R, t)
        xs.append(x); fs.append(f); Rs.append(R); ts.append(t)
    out = fit(dev, torch.stack(xs), torch.stack(fs))
    t_tol = 1e-4 if shift == 0 else 1e-3
    for s in range(b):
        assert not bool(out.degenerate[s])
        assert bool(out.inliers[s].all()) and int(out.count[s]) == n
        assert rot_err(out.rotation[s].cpu(), Rs[s]) < 1e-5, rot_err(out.rotation[s].cpu(), Rs[s])
        assert float((out.translation[s].cpu().double() - ts[s]).abs().max()) < t_tol


# ---- 4. robustness -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('objects', [(0.05, 0.08, 0.04), (0.08,) * 5, (0.45,)], ids=['scene', 'five_objects', 'one_large_object'])
def test_ego_motion_among_moving_objects(dev, objects):
    g = torch.Generator().manual_seed(4)
    x, f, R, t, moving = scene(16384, g, objects)
    out = fit(dev, x[None], f[None], threshold=0.05)
    inl = out.inliers[0].cpu()
    re, te = rot_err(out.rotation[0].cpu(), R), float((out.translation[0].cpu().double() - t).norm())
    static_share = float(inl[~moving].float().mean())
    print(f'ego-motion error {re:.2e} rad, {te * 1e3:.2f} mm; static inliers {static_share:.5f}')
    assert not bool(out.degenerate[0])
    assert re < 1e-4 and te < 5e-3
    assert not bool(inl[moving].any())
    assert static_share >= 0.999


# ---- 5. refit ------------------------------------------------------------------------------------------------------------
def test_refit_against_float64_horn(dev):
    g = torch.Generator().manual_seed(5)
    n, thr = 6000, 0.5
    x64 = torch.rand(n, 3, generator=g, dtype=torch.float64) * 5
    R, t = random_rotation(g, 25.0), torch.tensor([1.0, 0.5, -0.7], dtype=torch.float64)
    y = x64 @ R.T + t + torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.2
    y[: n // 4] += torch.randn(n // 4, 3, generator=g, dtype=torch.float64)
    x = x64.float()
    f = (y - x.double()).float()
    xs, ys = x.double().numpy(), yf32(x, f).numpy()
    prev = None
    for rounds in (1, 2, 3):
        out = fit(dev, x[None], f[None], threshold=thr, rounds=rounds)
        inl = out.inliers[0].cpu().numpy()
        Rw, xb, yb = horn_np(xs[inl], ys[inl])
        assert np.abs(out.rotation[0].cpu().double().numpy() - Rw).max() < 4 * 2.0 ** -24
        tw = yb - Rw @ xb
        assert np.abs(out.translation[0].cpu().double().numpy() - tw).max() < 4 * 2.0 ** -24 * (1 + np.abs(tw).max())
        if prev is not None:   # this round's inliers: within the threshold of the previous round's model, stored in fp32
            Rp, cx, cy = (np.asarray(v, np.float32).astype(np.float64) for v in prev)
            r2 = resid2(Rp, cx, cy, xs, ys)
            edge = np.abs(r2 - thr * thr) <= 1e-5 * thr * thr
            print(f'rounds={rounds}: {int(edge.sum())} boundary points exempt')
            assert np.array_equal(inl[~edge], (r2 <= thr * thr)[~edge])
        prev = (out.rotation[0].cpu().numpy(), xs[inl].mean(0), ys[inl].mean(0))


# ---- 6. degenerate cases -------------------------------------------------------------------------------------------------
def test_degenerate_samples(dev):
    import pvraft_b200
    g = torch.Generator().manual_seed(6)
    n = 500
    good_x, good_f = rigid_flow(cloud(n, 'uniform', g), random_rotation(g, 10.0), torch.tensor([0.5, 0.1, 0.0], dtype=torch.float64))
    tt = torch.rand(n, 1, generator=g) * 50 - 25
    collinear = torch.cat([tt, 2 * tt, -tt], 1)                    # exactly collinear in fp32
    dup = torch.rand(1, 3, generator=g).expand(n, 3).contiguous() * 10
    xs = torch.stack([good_x, collinear, good_x, good_x, dup])
    fs = torch.stack([good_f] + [torch.randn(n, 3, generator=g) * 0.01 for _ in range(4)])
    mask = torch.ones(5, n, dtype=torch.bool)
    mask[2] = False                   # all masked
    mask[3] = False
    mask[3, [10, 300]] = True         # two points left
    xd, fd = xs.to(dev).requires_grad_(True), fs.to(dev).requires_grad_(True)
    out = pvraft_b200.rigid_motion(xd, fd, mask=mask.to(dev))
    assert out.degenerate.cpu().tolist() == [False, True, True, True, True]
    ys = yf32(xs, fs)
    for s in (1, 2, 3, 4):
        assert torch.equal(out.rotation[s].cpu(), torch.eye(3))
        inl = out.inliers[s].cpu()
        assert torch.equal(inl, mask[s])                                # no accepted hypothesis: every allowed point
        want = (ys[s][inl] - xs[s][inl].double()).mean(0) if inl.any() else torch.zeros(3, dtype=torch.float64)
        assert float((out.translation[s].detach().cpu().double() - want).abs().max()) < 1e-5, s
    assert int(out.count[2]) == 0 and int(out.count[3]) == 2
    gR, gt = torch.randn(5, 3, 3, device=dev), torch.randn(5, 3, device=dev)
    ((out.rotation * gR).sum() + (out.translation * gt).sum()).backward()
    assert torch.isfinite(xd.grad).all() and torch.isfinite(fd.grad).all()
    for s in (1, 3, 4):   # the translation only: d flow = dt / n on the inliers, d xyz1 = 0
        inl = out.inliers[s]
        assert float(xd.grad[s].abs().max()) == 0.0
        assert torch.allclose(fd.grad[s][inl], (gt[s] / int(out.count[s])).expand(int(inl.sum()), 3), rtol=1e-6, atol=0)
    assert float(fd.grad[2].abs().max()) == 0.0


def test_a_degenerate_sample_leaves_its_neighbours_alone(dev, det):
    g = torch.Generator().manual_seed(7)
    n = 2048
    x0, f0 = rigid_flow(cloud(n, 'lidar', g), random_rotation(g, 10.0), torch.tensor([1.0, 0.0, 0.2], dtype=torch.float64))
    x2, f2 = rigid_flow(cloud(n, 'uniform', g), random_rotation(g, 10.0), torch.tensor([0.0, -1.0, 0.2], dtype=torch.float64))
    tt = torch.rand(n, 1, generator=g)
    x1 = torch.cat([tt, 2 * tt, 4 * tt], 1)
    batch = fit(dev, torch.stack([x0, x1, x2]), torch.stack([f0, f0, f2]))
    assert batch.degenerate.cpu().tolist() == [False, True, False]
    for s, (x, f) in ((0, (x0, f0)), (2, (x2, f2))):
        one = fit(dev, x[None], f[None])
        for a, b in zip(one, batch):
            assert same_bits(a[0], b[s])


# ---- 7. gradients --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [64, 8192])
@pytest.mark.parametrize('shift', [0.0, 1e3])
def test_gradients_against_float64_autograd(dev, n, shift):
    import pvraft_b200
    g = torch.Generator().manual_seed(n + int(shift))
    b = 2
    xs, fs = [], []
    for _ in range(b):
        R, t = random_rotation(g, 20.0), (torch.rand(3, generator=g, dtype=torch.float64) * 2 - 1) * 3.0
        x64 = cloud(n, 'uniform', g, shift)
        y = x64 @ R.T + t + torch.randn(n, 3, generator=g, dtype=torch.float64) * 0.02
        y[: n // 8] += 1.0                                               # outliers
        x = x64.float()
        xs.append(x); fs.append((y - x.double()).float())
    x, f = torch.stack(xs), torch.stack(fs)
    gR, gt = torch.randn(b, 3, 3, generator=g), torch.randn(b, 3, generator=g)
    xd, fd = x.to(dev).requires_grad_(True), f.to(dev).requires_grad_(True)
    out = pvraft_b200.rigid_motion(xd, fd, threshold=0.1)
    ((out.rotation * gR.to(dev)).sum() + (out.translation * gt.to(dev)).sum()).backward()
    x64, f64 = x.double().requires_grad_(True), f.double().requires_grad_(True)
    y64 = x64 + f64 + (yf32(x, f) - (x.double() + f.double()))       # the fp32 sum y = x + f, differentiable
    loss = 0
    for s in range(b):
        inl = out.inliers[s].cpu()
        assert not bool(out.degenerate[s]) and int(inl.sum()) >= 3
        R, t = horn_torch(x64[s][inl], y64[s][inl])
        assert float((out.rotation[s].cpu().double() - R.detach()).abs().max()) < 1e-6
        loss = loss + (R * gR[s].double()).sum() + (t * gt[s].double()).sum()
    loss.backward()
    for got, want, name in ((xd.grad, x64.grad, 'd_xyz1'), (fd.grad, f64.grad, 'd_flow')):
        err = float((got.cpu().double() - want).norm() / want.norm())
        print(f'n={n} shift={shift}: {name} relative error {err:.2e}')
        assert err < 1e-5, (name, err)
        assert float(got[~out.inliers].abs().max()) == 0.0


# ---- 8. batch and determinism --------------------------------------------------------------------------------------------
def batch_case(g, b=4, n=5000):
    xs, fs = [], []
    for s in range(b):
        x, f, _, _, _ = scene(n, g, (0.1, 0.05), shift=100.0 * s)
        xs.append(x); fs.append(f)
    return torch.stack(xs), torch.stack(fs)


def test_one_segment_deterministic_repeatable_and_batched_equals_per_sample(dev, det):
    g = torch.Generator().manual_seed(8)
    x, f = batch_case(g)
    mask = torch.rand(x.shape[:2], generator=g) < 0.9
    for m in (None, mask):
        a, b = fit(dev, x, f, m, threshold=0.05), fit(dev, x, f, m, threshold=0.05)
        assert all(same_bits(p, q) for p, q in zip(a, b))
        for s in range(x.shape[0]):
            one = fit(dev, x[s:s + 1], f[s:s + 1], None if m is None else m[s:s + 1], threshold=0.05)
            assert all(same_bits(p[0], q[s]) for p, q in zip(one, a)), s
    full = fit(dev, x, f, torch.ones(x.shape[:2], dtype=torch.bool), threshold=0.05)
    none = fit(dev, x, f, None, threshold=0.05)
    assert all(same_bits(p, q) for p, q in zip(full, none))
    ra, rb = raw(dev, x, f, threshold=0.05), raw(dev, x, f, torch.ones(x.shape[:2], dtype=torch.bool), threshold=0.05)
    assert all(same_bits(p, q) for p, q in zip(ra, rb))


def test_one_segment_default_mode_agrees_with_deterministic_mode(dev):
    g = torch.Generator().manual_seed(9)
    x, f = batch_case(g)
    a = raw(dev, x, f, threshold=0.05)
    torch.use_deterministic_algorithms(True)
    try:
        d = raw(dev, x, f, threshold=0.05)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(a[7], d[7]) and torch.equal(a[6], d[6])           # the same hypotheses, counts and so selection
    differ = int((a[2] != d[2]).sum())
    print(f'{differ} inlier decisions differ between the modes')
    assert differ <= 10
    assert float((a[0] - d[0]).abs().max()) < 1e-6 and float((a[1] - d[1]).abs().max()) < 1e-6 * (1 + float(d[1].abs().max()))


# ---- 9. capture ----------------------------------------------------------------------------------------------------------
def test_captured_forward_and_backward_equal_eager(dev, det):
    import pvraft_b200
    g = torch.Generator().manual_seed(10)
    x1, f1 = batch_case(g, b=2, n=3000)
    x2, f2 = batch_case(g, b=2, n=3000)
    gR, gt = torch.randn(2, 3, 3, generator=g).to(dev), torch.randn(2, 3, generator=g).to(dev)
    sx, sf = x1.to(dev).requires_grad_(True), f1.to(dev).requires_grad_(True)

    def step(x, f):
        out = pvraft_b200.rigid_motion(x, f, threshold=0.05)
        dx, df = torch.autograd.grad((out.rotation * gR).sum() + (out.translation * gt).sum(), (x, f))
        return out.rotation, out.translation, out.inliers, out.count, out.degenerate, dx, df

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step(sx, sf)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step(sx, sf)
    with torch.no_grad():
        sx.copy_(x2.to(dev))
        sf.copy_(f2.to(dev))
    graph.replay()
    eager = step(x2.to(dev).requires_grad_(True), f2.to(dev).requires_grad_(True))
    assert all(same_bits(p, q) for p, q in zip(static, eager))


# ---- 10. composition with the model --------------------------------------------------------------------------------------
def test_rsf_training_step_through_the_fit_matches_oracle(dev):
    """A 3-iteration stage-1 step whose loss is ||R - R_gt||^2 + ||t - t_gt||^2 of rigid_motion(xyz1, flows[-1]) (every point
    an inlier) against autograd through the oracle's rsf_forward and the float64 torch Horn fit: all 95 parameter gradients,
    with the bounds of test_gpu_laplacian.py::test_rsf_gradients_match_oracle."""
    import pvraft_b200
    from pvraft_b200 import RSF
    b, n, k, iters = 2, 1024, 128, 3
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)
    W = default_weights(args=args, seed=2)
    pc1, pc2 = O.synthetic_clouds(b, n, seed=11)
    pc1, pc2 = pc1 * 0.4, pc2 * 0.4
    g = torch.Generator().manual_seed(12)
    R_gt, t_gt = random_rotation(g, 3.0), torch.tensor([0.05, -0.02, 0.01], dtype=torch.float64)
    Wr = {kk: v.detach().clone().requires_grad_(True) for kk, v in W.items()}
    flow_ref = O.rsf_forward(Wr, pc1, pc2, iters, 3, 0.25, k)[-1]
    want_loss = 0
    for s in range(b):
        R, t = horn_torch(pc1[s].double(), (pc1[s] + flow_ref[s]).double())
        want_loss = want_loss + ((R - R_gt) ** 2).sum() + ((t - t_gt) ** 2).sum()
    want_loss.backward()
    want = {kk: v.grad for kk, v in Wr.items()}
    m = RSF(args)
    m.load_state_dict(W)
    m = m.to(dev).train()
    with oracle_adjacency():
        flows = m([pc1.to(dev), pc2.to(dev)], num_iters=iters)
    out = pvraft_b200.rigid_motion(pc1.to(dev), flows[-1], threshold=1e3)
    assert bool(out.inliers.all()) and not bool(out.degenerate.any())
    loss = ((out.rotation.double() - R_gt.to(dev)) ** 2).sum() + ((out.translation.double() - t_gt.to(dev)) ** 2).sum()
    assert abs(float(loss.detach()) - float(want_loss.detach())) < 1e-3 * abs(float(want_loss.detach()))
    loss.backward()
    got = {kk: p.grad for kk, p in m.named_parameters()}
    assert len(got) == 95 and all(v is not None for v in got.values())
    compare_grads(got, want, 2e-2, 5e-2)
