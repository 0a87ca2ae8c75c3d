"""The rigid-motion fit without a GPU: the C entry points of its one-segment case are declared, bound, size their workspaces
and refuse bad arguments before any launch; pvraft_b200.rigid_motion refuses bad shapes, masks, thresholds, hypothesis and round counts and seeds with
ValueError, and CPU tensors with PvraftError."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 256   # never dereferenced: every call below fails its argument check
BAD = -1


def test_header_declares_and_lib_binds_the_one_segment_entry_points():
    """The ego-motion fit is the one-segment case of the rigid fit: its entry points are the pvraft_rigid_objects_* family."""
    from pvraft_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    names = ('pvraft_rigid_objects_fwd', 'pvraft_rigid_objects_bwd', 'pvraft_rigid_objects_workspace_bytes',
             'pvraft_rigid_objects_fwd_det_workspace_bytes')
    for name in names:
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert name in _lib.EXPORTS
    assert [len(_lib._SIGNATURES[n][1]) for n in names] == [21, 13, 5, 3]


def test_one_segment_workspace_sizes():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    assert lib.pvraft_rigid_objects_fwd_det_workspace_bytes(3, 1, 2) == 2 * 3 * 16 * 24
    assert lib.pvraft_rigid_objects_fwd_det_workspace_bytes(0, 1, 2) == 0
    assert lib.pvraft_rigid_objects_fwd_det_workspace_bytes(3, 1, 9) == 0
    r16 = lambda v: (v + 15) // 16 * 16   # noqa: E731
    b, n, h, r = 3, 1001, 37, 2
    c, s = (n + 255) // 256, (n + 1023) // 1024 + 1
    want = (r16(4 * b * n) + 2 * r16(4 * b) + 2 * r16(4 * b * c) + r16(4 * b * n) + r16(4 * b) + r16(4 * b * s) + r16(4 * b)
            + r16(4 * b * h * 16) + r16(4 * b * h) + r16(4 * b * 16) + r16(8 * r * b * 16))
    assert lib.pvraft_rigid_objects_workspace_bytes(b, n, 1, h, r) == want
    for bad in ((0, n, 1, h, r), (b, 0, 1, h, r), (b, n, 1, 0, r), (b, n, 1, 4097, r), (b, n, 1, h, 0), (b, n, 1, h, 9)):
        assert lib.pvraft_rigid_objects_workspace_bytes(*bad) == 0, bad


def test_one_segment_entry_points_refuse_bad_arguments():
    """The one-segment calls rigid_motion makes (labels NULL without a mask, O = 1); N >= 3 is rigid_motion's own rule,
    checked in Python (test_public_function_refuses_bad_arguments)."""
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def fwd(x=P, f=P, lab=None, B=2, N=64, O=1, thr=0.1, H=256, rounds=2, seed=0, R=P, t=P, inl=P, cnt=P, deg=P, st=P, ws=P):
        return lib.pvraft_rigid_objects_fwd(x, f, lab, B, N, O, thr, H, rounds, seed, R, t, inl, cnt, deg, st, None, None, ws, None, None)

    def bwd(x=P, f=P, lab=None, inl=P, st=P, dR=P, dt=P, B=2, N=64, O=1, dx=P, df=P):
        return lib.pvraft_rigid_objects_bwd(x, f, lab, inl, st, dR, dt, B, N, O, dx, df, None)

    cases = (dict(B=0), dict(N=0), dict(N=-1), dict(H=0), dict(H=4097), dict(rounds=0), dict(rounds=9), dict(seed=-1),
             dict(thr=0.0), dict(thr=-0.1), dict(thr=float('nan')), dict(thr=float('inf')), dict(B=1 << 16, N=1 << 15), dict(O=2))
    for kw in cases:
        assert fwd(**kw) == BAD, kw
        assert b'rigid_objects_fwd' in lib.pvraft_last_error_string()
    for name in ('x', 'f', 'R', 't', 'inl', 'cnt', 'deg', 'st', 'ws'):
        assert fwd(**{name: None}) == BAD, name
    for kw in (dict(B=0), dict(N=0), dict(B=1 << 16, N=1 << 15), dict(O=2)):
        assert bwd(**kw) == BAD, kw
        assert b'rigid_objects_bwd' in lib.pvraft_last_error_string()
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
