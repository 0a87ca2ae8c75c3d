"""The object boxes without a GPU: a float32 numpy restatement of the rule of pvraft_object_boxes_fwd (extents, choice, box,
displacement, heading) recovers synthetic boxes -- full and L-shaped views at yaws off the angle grid -- and the two moving
boxes of test_host_rigid_refine's scene with their world motion and heading; the entry points are declared, bound and
size their workspace, and refuse bad arguments before any launch; pvraft_b200.object_boxes refuses bad arguments with
ValueError.

    direction a:  (c_a, s_a) = fp32(cos, sin)(a pi / (2 A))
    extents:      u = fl(fl(c P) + fl(s Q)), v = fl(fl(c Q) - fl(s P)) of the members, P = x_p, Q = x_q
    choice:       a* = lowest argmin of (umax - umin)(vmax - vmin) in double
    heading:      the length axis turned by pi when the centre's displacement points against it
"""
import os
import re

import numpy as np
import pytest
import torch

import test_host_rigid_refine as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 256   # never dereferenced: every call below fails its argument check
BAD, UNSUPPORTED = -1, -2
NAMES = ('pvraft_object_boxes_fwd', 'pvraft_object_boxes_workspace_bytes')


def r16(v):
    return (v + 15) // 16 * 16


# ---- numpy restatement ---------------------------------------------------------------------------------------------------
def dirs_ref(A):
    """(c_a, s_a) [A,2] float32: the double cos and sin of a pi / (2 A), rounded."""
    th = np.pi * (np.arange(A) / (2.0 * A))
    return np.stack([np.cos(th), np.sin(th)], 1).astype(np.float32)


def axes(up):
    return (up + 1) % 3, (up + 2) % 3


def boxes_ref(x, labels, R, t, up, A, ego=None, dirs=None):
    """The rule for one sample: x [N,3] float32, labels [N], fits R [O,3,3], t [O,3] float32, ego None or (R_e, t_e,
    degenerate) -> dict(center, size, displacement [O,3] f32, yaw [O] f32, rotation [O,3,3] f32, count [O], extents
    [O,A,4] f32, astar [O], phi [O] float64)."""
    x = np.asarray(x, np.float32)
    O = len(R)
    p, q = axes(up)
    d = dirs_ref(A) if dirs is None else np.asarray(dirs, np.float32)
    c, s = d[:, 0:1], d[:, 1:2]
    out = dict(center=np.zeros((O, 3), np.float32), size=np.zeros((O, 3), np.float32), displacement=np.zeros((O, 3), np.float32),
               yaw=np.zeros(O, np.float32), rotation=np.zeros((O, 3, 3), np.float32), count=np.zeros(O, np.int64),
               extents=np.tile(np.array([np.inf, -np.inf, np.inf, -np.inf], np.float32), (O, A, 1)), astar=np.zeros(O, np.int64),
               phi=np.zeros(O))
    use_ego = ego is not None and not ego[2]
    for o in range(O):
        mem = (labels == o) & np.isfinite(x).all(1)
        out['count'][o] = mem.sum()
        out['rotation'][o][p, 0] = out['rotation'][o][q, 1] = out['rotation'][o][up, 2] = 1
        if not mem.any():
            continue
        Pv, Qv, Hv = x[mem, p][None], x[mem, q][None], x[mem, up]
        u = c * Pv + s * Qv            # float32, each operation rounded
        v = c * Qv - s * Pv
        ext = np.stack([u.min(1), u.max(1), v.min(1), v.max(1)], 1)
        out['extents'][o] = ext
        e = ext.astype(np.float64)
        du, dv = e[:, 1] - e[:, 0], e[:, 3] - e[:, 2]
        area = du * dv
        area[np.isnan(area)] = np.inf
        a = int(np.argmin(area))       # the first least area: the lowest a
        out['astar'][o] = a
        du, dv = du[a], dv[a]
        phi = np.pi * (a / (2.0 * A))
        if not du >= dv:
            phi += np.pi / 2
        hmin, hmax = np.float64(Hv.min()), np.float64(Hv.max())
        out['size'][o] = (max(du, dv), min(du, dv), hmax - hmin)
        cd, sd = np.float64(c[a, 0]), np.float64(s[a, 0])
        mu, mv = (e[a, 0] + e[a, 1]) * 0.5, (e[a, 2] + e[a, 3]) * 0.5
        cen = np.zeros(3, np.float32)
        cen[p], cen[q], cen[up] = cd * mu - sd * mv, sd * mu + cd * mv, (hmin + hmax) * 0.5
        out['center'][o] = cen
        cc = cen.astype(np.float64)
        Ro, to = np.asarray(R[o], np.float32).astype(np.float64), np.asarray(t[o], np.float32).astype(np.float64)
        y = np.array([((Ro[k, 0] * cc[0] + Ro[k, 1] * cc[1]) + Ro[k, 2] * cc[2]) + to[k] for k in range(3)])
        if use_ego:
            Re, te = np.asarray(ego[0], np.float32).astype(np.float64), np.asarray(ego[1], np.float32).astype(np.float64)
            w = y - te
            y = np.array([(Re[0, k] * w[0] + Re[1, k] * w[1]) + Re[2, k] * w[2] for k in range(3)])
        dd = y - cc
        out['displacement'][o] = dd
        if dd[p] * np.cos(phi) + dd[q] * np.sin(phi) < 0:
            phi += np.pi
        if phi > np.pi:
            phi -= 2 * np.pi
        out['phi'][o] = phi
        out['yaw'][o] = phi
        rot = np.zeros((3, 3))
        rot[p, 0], rot[q, 0], rot[p, 1], rot[q, 1], rot[up, 2] = np.cos(phi), np.sin(phi), -np.sin(phi), np.cos(phi), 1
        out['rotation'][o] = rot
    return out


def wrap(a):
    """An angle difference in (-pi, pi]."""
    return (a + np.pi) % (2 * np.pi) - np.pi


# ---- synthetic boxes -------------------------------------------------------------------------------------------------------
def box_points(rng, n, centre, size, yaw_deg, sides=(0, 1, 2, 3, 4)):
    """n points on the given faces of a box (0, 1: the faces at -x, +x of its own frame; 2, 3: -y, +y; 4: the top) standing
    at centre[2], turned by yaw_deg about z.  A LiDAR above a vehicle sees it from a corner as an L-shaped view: sides
    (0, 2, 4)."""
    face = rng.choice(np.asarray(sides), n)
    u, v = rng.random(n), rng.random(n)
    L, W, Hh = size
    loc = np.empty((n, 3))
    for f, (a, b, c, val) in enumerate(((1, 2, 0, 0.0), (1, 2, 0, 1.0), (0, 2, 1, 0.0), (0, 2, 1, 1.0), (0, 1, 2, 1.0))):
        sel = face == f
        loc[sel, a] = u[sel] * size[a]
        loc[sel, b] = v[sel] * size[b]
        loc[sel, c] = val * size[c]
    loc -= np.array([L / 2, W / 2, 0.0])
    return loc @ H.yaw(yaw_deg).T + np.asarray(centre)


# The accuracy the restatement reaches on these boxes (A = 90, 1 degree steps; 2000 points, no noise).  The least-area
# rectangle lies within half a step of the truth (23.7 and 137.4 degrees give a* = 24 and 47): a direction off by half a
# step widens the box by up to L sin(0.5 deg) = 4.0 cm and lengthens it by up to W sin(0.5 deg) = 1.7 cm, and the
# points sampled on the faces fall short of the corners by a few mm.  Seen: 3.2 cm on the size, 9 mm on the centre,
# 0.4 degrees.  An L-shaped view of two sides sees the top too, as a sensor above the box does.
SIZE_TOL, CENTRE_TOL, YAW_TOL = 0.045, 0.015, np.radians(0.5) + 1e-9
SIZE = np.array([4.6, 1.9, 1.5])


@pytest.mark.parametrize('yaw_deg', [23.7, 61.0, -37.2, 90.0, 0.0, 137.4])
@pytest.mark.parametrize('sides', [(0, 1, 2, 3, 4), (0, 2, 4), (1, 3, 4), (0, 3, 4)])
def test_restatement_recovers_boxes_off_the_angle_grid(yaw_deg, sides):
    rng = np.random.default_rng(int(abs(yaw_deg) * 10) + len(sides))
    centre = np.array([7.0, -3.0, -1.7])
    x = box_points(rng, 2000, centre, SIZE, yaw_deg, sides).astype(np.float32)
    out = boxes_ref(x, np.zeros(len(x), np.int64), np.eye(3)[None], np.zeros((1, 3)), 2, 90)
    assert out['count'][0] == 2000
    got = out['size'][0]
    assert np.abs(got - SIZE).max() < SIZE_TOL, (got, SIZE)
    assert np.abs(out['center'][0] - centre - np.array([0, 0, SIZE[2] / 2])).max() < CENTRE_TOL
    # a box that does not move keeps its length axis in [0, pi): the truth modulo pi
    assert 0 <= out['phi'][0] < np.pi
    assert abs(wrap(2 * (out['phi'][0] - np.radians(yaw_deg))) / 2) < YAW_TOL, (out['phi'][0], yaw_deg)
    assert np.allclose(out['displacement'][0], 0)


@pytest.mark.parametrize('yaw_deg', [23.7, -37.2])
def test_restatement_on_two_sides_alone_ties_with_the_hypotenuse(yaw_deg):
    """Two sides seen without the top have a right-triangle hull, and the rectangle on its hypotenuse has the same area L W
    as the true box: the least area is then either, as sampling and the grid decide (23.7 degrees gives the true box to a
    step, -37.2 the hypotenuse's).  The rule keeps this; a caller that sees such views needs the tracker's history."""
    rng = np.random.default_rng(int(abs(yaw_deg) * 10) + 2)
    x = box_points(rng, 2000, np.array([7.0, -3.0, -1.7]), SIZE, yaw_deg, (0, 2)).astype(np.float32)
    out = boxes_ref(x, np.zeros(len(x), np.int64), np.eye(3)[None], np.zeros((1, 3)), 2, 90)
    L, W = SIZE[:2]
    assert abs(out['size'][0][0] * out['size'][0][1] / (L * W) - 1) < 0.01
    hyp = np.radians(yaw_deg) + np.arctan2(W, L) * (1 if yaw_deg > 0 else -1)
    off = [abs(wrap(2 * (out['phi'][0] - a)) / 2) for a in (np.radians(yaw_deg), hyp, hyp + np.pi / 2)]
    assert min(off) < np.radians(1.0), np.degrees(off)


def test_restatement_takes_the_lowest_angle_on_ties_and_handles_degenerate_segments():
    x = np.array([[1, 2, 3], [1, 2, 3], [0, 0, 0], [3, 0, 0], [0, 0, 1], [np.nan, 0, 0], [5, 5, 5]], np.float32)
    labels = np.array([0, 0, 1, 1, 2, 3, -1])
    R, t = np.tile(np.eye(3), (5, 1, 1)), np.zeros((5, 3))
    out = boxes_ref(x, labels, R, t, 2, 8)
    assert list(out['count']) == [2, 2, 1, 0, 0]
    # one point (twice): every area is 0, so a* = 0 and the box is a point
    assert out['astar'][0] == 0 and np.all(out['size'][0] == 0) and np.all(out['center'][0] == [1, 2, 3])
    # a segment along x: width 0 at a = 0
    assert out['astar'][1] == 0 and np.allclose(out['size'][1], [3, 0, 0]) and np.allclose(out['center'][1], [1.5, 0, 0])
    # a segment whose only point is not finite, and an empty slot: zeros and the basis
    for o in (3, 4):
        assert np.all(out['size'][o] == 0) and np.all(out['rotation'][o] == np.eye(3))
        assert np.all(out['extents'][o] == [np.inf, -np.inf, np.inf, -np.inf])


def test_restatement_heading_follows_the_world_motion_with_ego_and_the_sensor_motion_without():
    """The two moving boxes of test_host_rigid_refine's scene, from their true fits: with the ego-motion the displacement is
    each box's own motion tb in the world (to a few mm: the centre found is off the true one by the noise, which tb's small
    rotation carries), and box 1, moving towards -x, faces -x (yaw near pi); relative to the sensor, which moves +0.9 m
    along x, box 1's centre moves towards +x, so its heading flips to near 0."""
    sc = H.scene(0)
    labels = sc['seg'] - 1
    fits = sc['motions'][1:]
    R, t = np.stack([f[0] for f in fits]), np.stack([f[1] for f in fits])
    Re, te = H.EGO
    world = boxes_ref(sc['xyz1'], labels, R, t, 2, 90, ego=(Re, te, False))
    sensor = boxes_ref(sc['xyz1'], labels, R, t, 2, 90)
    degenerate = boxes_ref(sc['xyz1'], labels, R, t, 2, 90, ego=(Re, te, True))
    for k in world:
        assert np.array_equal(degenerate[k], sensor[k]), k   # a degenerate ego is ignored
    for o, ((c, sz), (_, tb)) in enumerate(zip(H.BOXES, H.BOX_MOTIONS)):
        # 1 cm of noise per coordinate puts the extremes ~3 cm beyond the faces: 0.08 m on the size, 0.03 m on the centre
        assert np.abs(world['size'][o] - sz).max() < 0.08, (o, world['size'][o])
        assert np.abs(world['center'][o] - (c + [0, 0, sz[2] / 2])).max() < 0.03
        assert np.abs(world['displacement'][o] - tb).max() < 0.01, (o, world['displacement'][o], tb)
        assert np.array_equal(world['center'][o], sensor['center'][o]) and np.array_equal(world['size'][o], sensor['size'][o])
    # box 0 moves +x in both frames, box 1 -x in the world and +x relative to the sensor; the boxes' length is along x
    step = np.radians(1.0)
    assert abs(wrap(world['phi'][0])) <= step and abs(wrap(sensor['phi'][0])) <= step
    assert abs(wrap(world['phi'][1] - np.pi)) <= step, world['phi'][1]
    assert abs(wrap(sensor['phi'][1])) <= step, sensor['phi'][1]
    assert sensor['displacement'][1][0] > 0 > world['displacement'][1][0]
    # the rotation's first column is the heading
    for out in (world, sensor):
        for o in range(2):
            assert np.allclose(out['rotation'][o][:2, 0], [np.cos(out['phi'][o]), np.sin(out['phi'][o])], atol=1e-7)


# ---- the C ABI -----------------------------------------------------------------------------------------------------------
def test_header_declares_and_lib_binds_the_box_entry_points():
    from pvraft_b200 import _lib, build, ops
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    for name in NAMES:
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert name in _lib.EXPORTS
    assert [len(_lib._SIGNATURES[n][1]) for n in NAMES] == [22, 4]
    assert 'object_boxes.cu' in build.SOURCES
    params = _lib.FUNCTIONS['pvraft_object_boxes_fwd'][1]
    assert [d.name for d in params[7:12]] == ['B', 'N', 'O', 'up', 'A']
    assert [d.pointee for d in params[12:20]] == ['float'] * 5 + ['int32_t', 'float', 'float']
    assert ops.OBJECT_BOXES_MAX_ANGLES == 256


def test_box_workspace_size():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    b, n, o, a = 3, 1001, 5, 90
    g = b * o
    c = (n + 255) // 256
    s = (n + 1023) // 1024 + o
    grouping = r16(4 * b * n) + 2 * r16(4 * g) + 2 * r16(4 * b * c * o) + r16(4 * b * n) + r16(4 * b) + r16(4 * b * s) + r16(4 * b)
    assert lib.pvraft_object_boxes_workspace_bytes(b, n, o, a) == grouping + r16(16 * g * a) + r16(8 * g) + r16(4 * g)
    for bad in ((0, n, o, a), (b, 0, o, a), (b, n, 0, a), (b, n, 257, a), (b, n, o, 0), (b, n, o, 257), (1 << 16, 1 << 15, 1, a),
                (300, n, 256, a)):
        assert lib.pvraft_object_boxes_workspace_bytes(*bad) == 0, bad


def test_box_entry_point_refuses_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def fwd(x=P, lab=P, Ro=P, to=P, Re=None, te=None, de=None, B=2, N=64, O=4, up=2, A=90, ce=P, sz=P, yw=P, rot=P, dp=P, cn=P,
            ws=P):
        return lib.pvraft_object_boxes_fwd(x, lab, Ro, to, Re, te, de, B, N, O, up, A, ce, sz, yw, rot, dp, cn, None, None, ws, None)

    cases = (dict(B=0), dict(N=0), dict(B=1 << 16, N=1 << 15, O=1), dict(O=0), dict(O=257), dict(up=-1), dict(up=3), dict(A=0),
             dict(A=257), dict(Re=P), dict(Re=P, te=P), dict(te=P, de=P), dict(de=P))
    for kw in cases:
        assert fwd(**kw) == BAD, kw
        assert b'object_boxes_fwd' in lib.pvraft_last_error_string()
    for name in ('x', 'lab', 'Ro', 'to', 'ce', 'sz', 'yw', 'rot', 'dp', 'cn', 'ws'):
        assert fwd(**{name: None}) == BAD, name
    assert fwd(ws=P + 8) == BAD   # unaligned workspace
    assert fwd(B=300, O=256) == UNSUPPORTED
    assert fwd(B=65536, N=1, O=1) == UNSUPPORTED
    assert b'object_boxes_fwd' in lib.pvraft_last_error_string()


def test_public_function_refuses_bad_arguments():
    import pvraft_b200
    from pvraft_b200._lib import PvraftError
    b, n, o = 2, 50, 4
    x = torch.rand(b, n, 3)
    ego = pvraft_b200.RigidMotion(torch.eye(3).expand(b, 3, 3), torch.zeros(b, 3), torch.ones(b, n, dtype=torch.bool),
                                  torch.zeros(b, dtype=torch.int32), torch.zeros(b, dtype=torch.bool))
    obj = pvraft_b200.RigidObjects(torch.zeros(b, n, dtype=torch.int32), torch.ones(b, dtype=torch.int32), torch.eye(3).expand(b, o, 3, 3),
                                   torch.zeros(b, o, 3), torch.zeros(b, o, dtype=torch.int32), torch.zeros(b, o, dtype=torch.bool),
                                   torch.ones(b, n, dtype=torch.bool))
    calls = [dict(xyz1=x, objects=obj)]   # up missing
    calls += [dict(xyz1=x, objects=obj, up=v) for v in (None, -1, 3, 2.0, True, 'z')]
    calls += [dict(xyz1=x, objects=obj, up=2, angles=v) for v in (0, 257, 90.0, True, None, '90')]
    calls += [dict(xyz1=x[..., :2], objects=obj, up=2), dict(xyz1=x.long(), objects=obj, up=2), dict(xyz1=x[:, :0], objects=obj, up=2),
              dict(xyz1=x[:, :49], objects=obj, up=2), dict(xyz1=x[:1], objects=obj, up=2),
              dict(xyz1=x, objects=obj._replace(labels=obj.labels.long()), up=2),
              dict(xyz1=x, objects=obj._replace(translation=torch.zeros(b, o + 1, 3)), up=2),
              dict(xyz1=x, objects=obj._replace(rotation=torch.eye(3, dtype=torch.int32).expand(b, o, 3, 3)), up=2),
              dict(xyz1=x, objects=obj._replace(rotation=torch.eye(3).expand(b, 257, 3, 3),
                                                translation=torch.zeros(b, 257, 3)), up=2),
              dict(xyz1=x, objects=obj, up=2, ego=ego._replace(rotation=torch.eye(3).expand(b + 1, 3, 3))),
              dict(xyz1=x, objects=obj, up=2, ego=ego._replace(translation=torch.zeros(b, 4))),
              dict(xyz1=x, objects=obj, up=2, ego=ego._replace(degenerate=torch.zeros(b, dtype=torch.uint8)))]
    calls += [dict(xyz1=x, objects=v, up=2) for v in (None, ego, tuple(obj), obj._asdict())]
    calls += [dict(xyz1=x, objects=obj, up=2, ego=v) for v in (obj, (ego.rotation, ego.translation), ego.rotation)]
    for kw in calls:
        with pytest.raises(ValueError, match='object_boxes'):
            pvraft_b200.object_boxes(**kw)
    with pytest.raises(PvraftError):
        pvraft_b200.object_boxes(x, obj, up=2)
    with pytest.raises(PvraftError):
        pvraft_b200.object_boxes(x, obj, up=0, ego=ego, angles=256)
    assert pvraft_b200.ObjectBoxes._fields == ('center', 'size', 'yaw', 'rotation', 'displacement', 'count')
