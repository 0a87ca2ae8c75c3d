"""Object tracking without a GPU: the association entry point is declared, bound and built, and refuses bad arguments before
any launch; pvraft_b200.ObjectTracker refuses bad parameters, shapes and types with ValueError and CPU tensors with
PvraftError."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 256   # never dereferenced: every call below fails its argument check
BAD, UNSUPPORTED = -1, -2
NAME = 'pvraft_track_objects_fwd'


def test_header_declares_and_lib_binds_the_tracking_entry_point():
    from pvraft_b200 import _lib, build, ops
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    assert re.search(r'PVRAFT_API int ' + NAME + r'\(', header)
    assert NAME in _lib.EXPORTS
    params = _lib._SIGNATURES[NAME][1]
    assert len(params) == 27
    assert [d.pointee for d in _lib.FUNCTIONS[NAME][1] if d.pointee == 'double'] == ['double', 'double']   # pose_prev, pose
    assert 'tracks.cu' in build.SOURCES
    assert ops.TRACK_MIN_OVERLAP == 1 / 16 and ops.RIGID_MAX_OBJECTS == 256


def test_tracking_entry_point_refuses_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def fwd(xp=P, fp=P, lp=P, tp=P, ap=P, pp=P, Rp=P, tq=P, x=P, lab=P, num=P, nn=P, B=2, M=64, N=64, O_prev=8, O=8, gate=0.5,
            mo=0.5, nid=P, ov=P, mem=P, match=P, track=P, age=P, pose=P):
        return lib.pvraft_track_objects_fwd(xp, fp, lp, tp, ap, pp, Rp, tq, x, lab, num, nn, B, M, N, O_prev, O, gate, mo, nid, ov,
                                            mem, match, track, age, pose, None)

    nan, inf = float('nan'), float('inf')
    cases = (dict(B=0), dict(N=0), dict(N=-1), dict(M=-1), dict(O=0), dict(O=257), dict(O_prev=-1), dict(O_prev=257),
             dict(M=0), dict(M=0, O_prev=3), dict(gate=0.0), dict(gate=-0.5), dict(gate=nan), dict(gate=inf), dict(gate=1e20),
             dict(mo=0.0), dict(mo=1 / 16 - 1e-9), dict(mo=1.0 + 1e-9), dict(mo=nan), dict(mo=-0.5), dict(mo=inf))
    for kw in cases:
        assert fwd(**kw) == BAD, kw
        assert b'track_objects_fwd' in lib.pvraft_last_error_string()
    for name in ('xp', 'fp', 'lp', 'tp', 'ap', 'pp', 'Rp', 'tq', 'x', 'lab', 'num', 'nn', 'nid', 'ov', 'mem', 'match', 'track', 'age',
                 'pose'):
        assert fwd(**{name: None}) == BAD, name
    # the first step's previous pointers are not required, the current ones still are
    first = dict(xp=None, fp=None, lp=None, tp=None, ap=None, pp=None, Rp=None, tq=None, nn=None, ov=None, M=0, O_prev=0)
    for name in ('x', 'lab', 'num', 'nid', 'mem', 'match', 'track', 'age', 'pose'):
        assert fwd(**first, **{name: None}) == BAD, name
    assert fwd(**first, gate=nan) == BAD
    assert fwd(B=1 << 16) == UNSUPPORTED
    assert b'65535' in lib.pvraft_last_error_string()


def _objects(b, n, o, device='cpu'):
    import pvraft_b200
    return pvraft_b200.RigidObjects(torch.zeros(b, n, dtype=torch.int32, device=device), torch.ones(b, dtype=torch.int32, device=device),
                                    torch.eye(3, device=device).expand(b, o, 3, 3), torch.zeros(b, o, 3, device=device),
                                    torch.zeros(b, o, dtype=torch.int32, device=device), torch.zeros(b, o, dtype=torch.bool, device=device),
                                    torch.ones(b, n, dtype=torch.bool, device=device))


def test_tracker_refuses_bad_arguments():
    import pvraft_b200
    from pvraft_b200._lib import PvraftError
    for kw in [dict(gate=v) for v in (0.0, -0.5, float('nan'), float('inf'), True, '0.5', 1e20, None)] + \
              [dict(min_overlap=v) for v in (0.0, 0.06, 1.01, float('nan'), True, '0.5', None)]:
        with pytest.raises(ValueError, match='ObjectTracker'):
            pvraft_b200.ObjectTracker(**kw)
    pvraft_b200.ObjectTracker(gate=0.1, min_overlap=1 / 16)
    pvraft_b200.ObjectTracker(min_overlap=1)

    x, f = torch.rand(2, 50, 3), torch.rand(2, 50, 3)
    obj = _objects(2, 50, 4)
    ego = pvraft_b200.RigidMotion(torch.eye(3).expand(2, 3, 3), torch.zeros(2, 3), torch.ones(2, 50, dtype=torch.bool),
                                  torch.zeros(2, dtype=torch.int32), torch.zeros(2, dtype=torch.bool))
    tr = pvraft_b200.ObjectTracker()
    calls = [dict(xyz1=x[..., :2], flow=f[..., :2], objects=obj), dict(xyz1=x, flow=f[:, :49], objects=obj),
             dict(xyz1=x.long(), flow=f.long(), objects=obj), dict(xyz1=x[:, :0], flow=f[:, :0], objects=obj),
             dict(xyz1=x[:0], flow=f[:0], objects=obj), dict(xyz1=x, flow=f, objects=None), dict(xyz1=x, flow=f, objects=tuple(obj)),
             dict(xyz1=x, flow=f, objects=obj, ego=obj), dict(xyz1=x, flow=f, objects=obj, ego=tuple(ego)),
             dict(xyz1=x, flow=f, objects=_objects(2, 49, 4)), dict(xyz1=x, flow=f, objects=_objects(3, 50, 4)),
             dict(xyz1=x, flow=f, objects=_objects(2, 50, 257)),
             dict(xyz1=x, flow=f, objects=obj._replace(labels=obj.labels.long())),
             dict(xyz1=x, flow=f, objects=obj._replace(translation=torch.zeros(2, 5, 3))),
             dict(xyz1=x, flow=f, objects=obj, ego=ego._replace(inliers=torch.ones(2, 49, dtype=torch.bool)))]
    for kw in calls:
        with pytest.raises(ValueError, match='ObjectTracker'):
            tr.step(**kw)
    tr.gate = float('nan')
    with pytest.raises(ValueError, match='gate'):
        tr.step(x, f, obj)
    tr.gate, tr.min_overlap = 0.5, 2.0
    with pytest.raises(ValueError, match='min_overlap'):
        tr.step(x, f, obj)
    tr.min_overlap = 0.5
    with pytest.raises(PvraftError):
        tr.step(x, f, obj, ego)
    assert pvraft_b200.ObjectTracks._fields == ('track_id', 'labels', 'matched', 'age', 'rotation', 'translation')


def test_tracker_refuses_a_changed_batch_or_device():
    """The batch size and device checks compare against the kept state; it is set here by hand, so no device is needed."""
    import pvraft_b200
    tr = pvraft_b200.ObjectTracker()
    tr._prev = (torch.zeros(2, 50, 3, device='meta'),) + (None,) * 7
    with pytest.raises(ValueError, match='batch size'):
        tr.step(torch.rand(3, 50, 3), torch.rand(3, 50, 3), _objects(3, 50, 4))
    with pytest.raises(ValueError, match='previous step'):
        tr.step(torch.rand(2, 50, 3), torch.rand(2, 50, 3), _objects(2, 50, 4))
    tr.reset()
    assert tr._prev is None and tr._next_id is None
