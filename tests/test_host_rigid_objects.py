"""The moving-object fit without a GPU: the clustering and per-object fit entry points are declared, bound, size their
workspaces and refuse bad arguments before any launch; pvraft_b200.rigid_objects and rigid_flow refuse bad shapes, masks,
radii, counts, thresholds, hypothesis and round counts and seeds with ValueError, and CPU tensors with PvraftError."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 256   # never dereferenced: every call below fails its argument check
BAD = -1
NAMES = ('pvraft_euclidean_clusters_fwd', 'pvraft_euclidean_clusters_workspace_bytes', 'pvraft_rigid_objects_fwd',
         'pvraft_rigid_objects_workspace_bytes', 'pvraft_rigid_objects_fwd_det_workspace_bytes', 'pvraft_rigid_objects_bwd')


def r16(v):
    return (v + 15) // 16 * 16


def test_header_declares_and_lib_binds_the_clustering_and_fit_entry_points():
    from pvraft_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    for name in NAMES:
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert name in _lib.EXPORTS
    assert [len(_lib._SIGNATURES[n][1]) for n in NAMES] == [14, 2, 21, 5, 3, 13]
    from pvraft_b200 import build
    assert 'clusters.cu' in build.SOURCES


def test_workspace_sizes():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    b, n, o, h, r = 3, 1001, 5, 37, 2
    assert lib.pvraft_rigid_objects_fwd_det_workspace_bytes(b, o, r) == r * b * o * 16 * 24
    for bad in ((0, o, r), (b, 0, r), (b, 257, r), (b, o, 0), (b, o, 9)):
        assert lib.pvraft_rigid_objects_fwd_det_workspace_bytes(*bad) == 0, bad
    c = (n + 255) // 256
    s = (n + 1023) // 1024 + o
    g = b * o
    want = (r16(4 * b * n) + 2 * r16(4 * g) + 2 * r16(4 * b * c * o) + r16(4 * b * n) + r16(4 * b) + r16(4 * b * s) + r16(4 * b)
            + r16(4 * g * h * 16) + r16(4 * g * h) + r16(4 * g * 16) + r16(8 * r * g * 16))
    assert lib.pvraft_rigid_objects_workspace_bytes(b, n, o, h, r) == want
    for bad in ((0, n, o, h, r), (b, 0, o, h, r), (b, n, 0, h, r), (b, n, 257, h, r), (b, n, o, 0, r), (b, n, o, 4097, r),
                (b, n, o, h, 0), (b, n, o, h, 9), (1 << 16, 1 << 15, o, h, r)):
        assert lib.pvraft_rigid_objects_workspace_bytes(*bad) == 0, bad
    grid = lib.pvraft_grid_index_workspace_bytes(b, n)
    assert lib.pvraft_euclidean_clusters_workspace_bytes(b, n) == r16(grid) + r16(12 * b * n) + 3 * r16(4 * b * n) + r16(8 * b * n)
    for bad in ((0, n), (b, 0), (1 << 16, 1 << 15)):
        assert lib.pvraft_euclidean_clusters_workspace_bytes(*bad) == 0, bad


def test_clustering_and_fit_entry_points_refuse_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def clusters(x=P, f=None, mask=None, B=2, N=64, radius=0.5, fr=0.5, minp=10, O=64, lab=P, num=P, sizes=P, ws=P):
        return lib.pvraft_euclidean_clusters_fwd(x, f, mask, B, N, radius, fr, minp, O, lab, num, sizes, ws, None)

    def fwd(x=P, f=P, lab=P, B=2, N=64, O=8, thr=0.1, H=256, rounds=2, seed=0, R=P, t=P, inl=P, cnt=P, deg=P, st=P, ws=P):
        return lib.pvraft_rigid_objects_fwd(x, f, lab, B, N, O, thr, H, rounds, seed, R, t, inl, cnt, deg, st, None, None, ws, None, None)

    def bwd(x=P, f=P, lab=P, inl=P, st=P, dR=P, dt=P, B=2, N=64, O=8, dx=P, df=P):
        return lib.pvraft_rigid_objects_bwd(x, f, lab, inl, st, dR, dt, B, N, O, dx, df, None)

    nan, inf = float('nan'), float('inf')
    cases = (dict(B=0), dict(N=0), dict(N=-1), dict(B=1 << 16, N=1 << 15), dict(radius=0.0), dict(radius=-1.0), dict(radius=nan),
             dict(radius=inf), dict(radius=1e20), dict(f=P, fr=0.0), dict(f=P, fr=nan), dict(f=P, fr=inf), dict(f=P, fr=1e20),
             dict(minp=0), dict(O=0), dict(O=257))
    for kw in cases:
        assert clusters(**kw) == BAD, kw
        assert b'euclidean_clusters_fwd' in lib.pvraft_last_error_string()
    for name in ('x', 'lab', 'num', 'sizes', 'ws'):
        assert clusters(**{name: None}) == BAD, name
    assert clusters(ws=P + 8) == BAD   # unaligned workspace
    cases = (dict(B=0), dict(N=0), dict(O=0), dict(O=257), dict(H=0), dict(H=4097), dict(rounds=0), dict(rounds=9), dict(seed=-1),
             dict(thr=0.0), dict(thr=-0.1), dict(thr=nan), dict(thr=inf), dict(B=1 << 16, N=1 << 15))
    for kw in cases:
        assert fwd(**kw) == BAD, kw
        assert b'rigid_objects_fwd' in lib.pvraft_last_error_string()
    for name in ('x', 'f', 'lab', 'R', 't', 'inl', 'cnt', 'deg', 'st', 'ws'):
        assert fwd(**{name: None}) == BAD, name
    for kw in (dict(B=0), dict(N=0), dict(O=0), dict(O=257), dict(B=1 << 16, N=1 << 15)):
        assert bwd(**kw) == BAD, kw
        assert b'rigid_objects_bwd' in lib.pvraft_last_error_string()
    for name in ('x', 'f', 'lab', 'inl', 'st', 'dR', 'dt', 'dx', 'df'):
        assert bwd(**{name: None}) == BAD, name


def test_public_functions_refuse_bad_arguments():
    import pvraft_b200
    from pvraft_b200._lib import PvraftError
    x = torch.rand(2, 50, 3)
    f = torch.rand(2, 50, 3)
    calls = [
        dict(xyz1=torch.rand(2, 50), flow=torch.rand(2, 50)),
        dict(xyz1=torch.rand(2, 50, 4), flow=torch.rand(2, 50, 4)),
        dict(xyz1=x, flow=torch.rand(2, 49, 3)),
        dict(xyz1=torch.rand(2, 0, 3), flow=torch.rand(2, 0, 3)),
        dict(xyz1=torch.rand(0, 50, 3), flow=torch.rand(0, 50, 3)),
        dict(xyz1=x.long(), flow=f.long()),
        dict(xyz1=x, flow=f, mask=torch.ones(2, 50)),
        dict(xyz1=x, flow=f, mask=torch.ones(2, 49, dtype=torch.bool)),
        dict(xyz1=x, flow=f, mask=[True] * 50),
    ]
    for name in ('radius', 'flow_radius', 'threshold'):
        calls += [dict(xyz1=x, flow=f, **{name: v}) for v in (0.0, -0.1, float('nan'), float('inf'), True, '0.1', 1e20)]
    calls += [dict(xyz1=x, flow=f, min_points=v) for v in (0, -1, 2.0, True, None)]
    calls += [dict(xyz1=x, flow=f, max_objects=v) for v in (0, 257, 2.0, True, None)]
    calls += [dict(xyz1=x, flow=f, hypotheses=v) for v in (0, 4097, 2.0, True, None)]
    calls += [dict(xyz1=x, flow=f, rounds=v) for v in (0, 9, 2.0, False)]
    calls += [dict(xyz1=x, flow=f, seed=v) for v in (-1, 2 ** 31, 1.0, True, None)]
    for kw in calls:
        with pytest.raises(ValueError, match='rigid_objects'):
            pvraft_b200.rigid_objects(**kw)
    with pytest.raises(PvraftError):
        pvraft_b200.rigid_objects(x, f)
    with pytest.raises(PvraftError):
        pvraft_b200.rigid_objects(x, f, mask=torch.ones(2, 50, dtype=torch.bool), radius=1.0, min_points=1, max_objects=256,
                                  flow_radius=0.3, threshold=0.5, hypotheses=4096, rounds=8, seed=2 ** 31 - 1)
    assert pvraft_b200.RigidObjects._fields == ('labels', 'num_objects', 'rotation', 'translation', 'count', 'degenerate', 'inliers')

    o = 4
    obj = pvraft_b200.RigidObjects(torch.zeros(2, 50, dtype=torch.int32), torch.zeros(2, dtype=torch.int32), torch.eye(3).expand(2, o, 3, 3),
                                   torch.zeros(2, o, 3), torch.zeros(2, o, dtype=torch.int32), torch.zeros(2, o, dtype=torch.bool),
                                   torch.ones(2, 50, dtype=torch.bool))
    ego = pvraft_b200.RigidMotion(torch.eye(3).expand(2, 3, 3), torch.zeros(2, 3), torch.ones(2, 50, dtype=torch.bool),
                                  torch.zeros(2, dtype=torch.int32), torch.zeros(2, dtype=torch.bool))
    for kw in (dict(xyz1=x, flow=f, objects=None), dict(xyz1=x, flow=f, objects=obj, ego=obj), dict(xyz1=x[..., :2], flow=f, objects=obj),
               dict(xyz1=x, flow=f[:, :49], objects=obj), dict(xyz1=x[:, :49], flow=f[:, :49], objects=obj),
               dict(xyz1=x, flow=f, objects=obj, ego=ego._replace(inliers=torch.ones(2, 49, dtype=torch.bool)))):
        with pytest.raises(ValueError, match='rigid_flow'):
            pvraft_b200.rigid_flow(**kw)
    # rigid_flow is ATen glue: identity fits keep every point where it is
    assert torch.equal(pvraft_b200.rigid_flow(x, f, obj, ego=ego), torch.zeros_like(x))
    assert torch.equal(pvraft_b200.rigid_flow(x, f, obj._replace(inliers=torch.zeros(2, 50, dtype=torch.bool))), f)
