"""The rigid-motion fit without a GPU: the C entry points are declared, bound, size their workspaces and refuse bad arguments
before any launch; pvraft_b200.rigid_motion refuses bad shapes, masks, thresholds, hypothesis and round counts and seeds with
ValueError, and CPU tensors with PvraftError."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 256   # never dereferenced: every call below fails its argument check
BAD = -1


def test_header_declares_and_lib_binds_the_entry_points():
    from pvraft_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    names = ('pvraft_rigid_motion_fwd', 'pvraft_rigid_motion_bwd', 'pvraft_rigid_motion_workspace_bytes',
             'pvraft_rigid_motion_fwd_det_workspace_bytes')
    for name in names:
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert name in _lib.EXPORTS
    assert [len(_lib._SIGNATURES[n][1]) for n in names] == [20, 11, 4, 2]


def test_workspace_sizes():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    assert lib.pvraft_rigid_motion_fwd_det_workspace_bytes(3, 2) == 2 * 3 * 16 * 24
    assert lib.pvraft_rigid_motion_fwd_det_workspace_bytes(0, 2) == 0
    assert lib.pvraft_rigid_motion_fwd_det_workspace_bytes(3, 9) == 0
    r16 = lambda v: (v + 15) // 16 * 16   # noqa: E731
    b, n, h, r = 3, 1001, 37, 2
    want = r16(4 * b * n) + r16(4 * b) + r16(4 * b * h * 16) + r16(4 * b * h) + r16(4 * b * 16) + r16(8 * r * b * 16)
    assert lib.pvraft_rigid_motion_workspace_bytes(b, n, h, r) == want
    for bad in ((0, n, h, r), (b, 2, h, r), (b, n, 0, r), (b, n, 4097, r), (b, n, h, 0), (b, n, h, 9)):
        assert lib.pvraft_rigid_motion_workspace_bytes(*bad) == 0, bad


def test_entry_points_refuse_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def fwd(x=P, f=P, mask=None, B=2, N=64, thr=0.1, H=256, rounds=2, seed=0, R=P, t=P, inl=P, cnt=P, deg=P, st=P, ws=P):
        return lib.pvraft_rigid_motion_fwd(x, f, mask, B, N, thr, H, rounds, seed, R, t, inl, cnt, deg, st, None, None, ws, None, None)

    def bwd(x=P, f=P, inl=P, st=P, dR=P, dt=P, B=2, N=64, dx=P, df=P):
        return lib.pvraft_rigid_motion_bwd(x, f, inl, st, dR, dt, B, N, dx, df, None)

    cases = (dict(B=0), dict(N=2), dict(N=-1), dict(H=0), dict(H=4097), dict(rounds=0), dict(rounds=9), dict(seed=-1),
             dict(thr=0.0), dict(thr=-0.1), dict(thr=float('nan')), dict(thr=float('inf')), dict(B=1 << 16, N=1 << 15))
    for kw in cases:
        assert fwd(**kw) == BAD, kw
        assert b'rigid_motion_fwd' in lib.pvraft_last_error_string()
    for name in ('x', 'f', 'R', 't', 'inl', 'cnt', 'deg', 'st', 'ws'):
        assert fwd(**{name: None}) == BAD, name
    for kw in (dict(B=0), dict(N=2), dict(B=1 << 16, N=1 << 15)):
        assert bwd(**kw) == BAD, kw
        assert b'rigid_motion_bwd' in lib.pvraft_last_error_string()
    for name in ('x', 'f', 'inl', 'st', 'dR', 'dt', 'dx', 'df'):
        assert bwd(**{name: None}) == BAD, name


def test_public_function_refuses_bad_arguments():
    import pvraft_b200
    from pvraft_b200._lib import PvraftError
    x = torch.rand(2, 50, 3)
    f = torch.rand(2, 50, 3)
    calls = [
        dict(xyz1=torch.rand(2, 50), flow=torch.rand(2, 50)),
        dict(xyz1=torch.rand(2, 50, 4), flow=torch.rand(2, 50, 4)),
        dict(xyz1=x, flow=torch.rand(2, 49, 3)),
        dict(xyz1=torch.rand(2, 2, 3), flow=torch.rand(2, 2, 3)),
        dict(xyz1=torch.rand(0, 50, 3), flow=torch.rand(0, 50, 3)),
        dict(xyz1=x.long(), flow=f.long()),
        dict(xyz1=x, flow=f, mask=torch.ones(2, 50)),
        dict(xyz1=x, flow=f, mask=torch.ones(2, 49, dtype=torch.bool)),
        dict(xyz1=x, flow=f, mask=torch.ones(1, 50, dtype=torch.bool)),
        dict(xyz1=x, flow=f, mask=[True] * 50),
    ]
    calls += [dict(xyz1=x, flow=f, threshold=v) for v in (0.0, -0.1, float('nan'), float('inf'), True, '0.1', 1e20)]
    calls += [dict(xyz1=x, flow=f, hypotheses=v) for v in (0, 4097, 2.0, True, None)]
    calls += [dict(xyz1=x, flow=f, rounds=v) for v in (0, 9, 2.0, False)]
    calls += [dict(xyz1=x, flow=f, seed=v) for v in (-1, 2 ** 31, 1.0, True, None)]
    for kw in calls:
        with pytest.raises(ValueError, match='rigid_motion'):
            pvraft_b200.rigid_motion(**kw)
    with pytest.raises(PvraftError):
        pvraft_b200.rigid_motion(x, f)
    with pytest.raises(PvraftError):
        pvraft_b200.rigid_motion(x, f, mask=torch.ones(2, 50, dtype=torch.bool), threshold=0.5, hypotheses=4096, rounds=8,
                                 seed=2 ** 31 - 1)
    assert pvraft_b200.RigidMotion._fields == ('rotation', 'translation', 'inliers', 'count', 'degenerate')
