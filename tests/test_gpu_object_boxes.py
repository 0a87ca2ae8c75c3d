"""The object boxes on the device (csrc/object_boxes.cu, pvraft_b200.object_boxes): bit for bit against the numpy
restatement of test_host_object_boxes run on the kernel's own directions -- including non-finite points, a one-point and a
collinear object and empty slots --, repeatability in both modes, batching, per-object equivalence, the cyclic symmetry
of `up`, the chain rigid_motion -> rigid_objects (-> rigid_refine) -> object_boxes with ObjectTracker's slots, and graph
capture."""
import numpy as np
import pytest
import torch

import test_host_object_boxes as HB
import test_host_rigid_refine as H
from test_gpu_rigid_motion import same_bits

pytestmark = pytest.mark.gpu

ROT_TOL = 1e-7   # rotation entries: the double cos / sin of the device and of numpy may round one fp32 ulp apart


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture(scope='module')
def sc():
    return H.scene(0)


def cloud(seed, n=3000, O=7):
    """A sample of O slots: boxes at random yaws, positions and sizes in objects 0 .. O - 5, then a one-point object, a
    collinear object (width 0), an object whose points are all non-finite and an empty slot; non-finite points and
    unlabelled points sprinkled in.  -> (x [n,3] f32, labels [n] int32, R [O,3,3], t [O,3] f32)."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-20, 20, (n, 3)).astype(np.float32)
    labels = np.full(n, -1, np.int32)
    nb = O - 4
    per = (n - 40) // nb
    for o in range(nb):
        size = rng.uniform([2, 1, 1], [6, 2.5, 2.5])
        pts = HB.box_points(rng, per, rng.uniform(-15, 15, 3), size, rng.uniform(-180, 180))
        x[o * per:(o + 1) * per] = pts
        labels[o * per:(o + 1) * per] = o
    k = nb * per
    x[k] = (1.5, -2.25, 0.75)
    labels[k] = nb                                   # one point
    x[k + 1:k + 11] = np.stack([np.linspace(-3, 4, 10), 0.5 * np.linspace(-3, 4, 10) + 1, np.full(10, 2.0)], 1)
    labels[k + 1:k + 11] = nb + 1                    # collinear in the plane: width 0 at its own direction only
    x[k + 11:k + 14, 1] = np.nan
    labels[k + 11:k + 14] = nb + 2                   # no finite point: an empty box
    bad = rng.choice(k, 25, replace=False)           # non-finite points inside the boxes, left out
    x[bad, rng.integers(0, 3, 25)] = rng.choice([np.nan, np.inf, -np.inf], 25)
    R = np.stack([H.yaw(rng.uniform(-10, 10)) for _ in range(O)]).astype(np.float32)
    t = rng.uniform(-2, 2, (O, 3)).astype(np.float32)
    return x, labels, R, t


def batch(seeds, dev, O=7):
    parts = [cloud(s, O=O) for s in seeds]
    return [torch.tensor(np.stack(p), device=dev) for p in zip(*parts)], parts


def ego_of(b, seed, dev, degenerate=()):
    rng = np.random.default_rng(seed)
    Re = np.stack([H.yaw(rng.uniform(-3, 3)) for _ in range(b)]).astype(np.float32)
    te = rng.uniform(-1, 1, (b, 3)).astype(np.float32)
    deg = np.array([i in degenerate for i in range(b)])
    return (torch.tensor(Re, device=dev), torch.tensor(te, device=dev), torch.tensor(deg, device=dev).view(torch.uint8)), (Re, te, deg)


def call(x, labels, R, t, ego, up, A, trace=True):
    from pvraft_b200 import ops
    return ops.object_boxes(x.contiguous(), labels.contiguous(), R.contiguous(), t.contiguous(), ego, up, A, want_trace=trace)


def astar_of(yaw, A):
    """a* from the yaw: phi is a* pi / (2 A) plus a multiple of pi / 2."""
    step = np.pi / (2 * A)
    return np.rint(np.mod(yaw.astype(np.float64), np.pi / 2) / step).astype(np.int64) % A


@pytest.mark.parametrize('A,up', [(90, 2), (256, 2), (7, 1), (1, 0)])
def test_boxes_match_the_restatement_bit_for_bit(A, up, dev):
    (x, labels, R, t), parts = batch((1, 2), dev)
    ego_t, (Re, te, deg) = ego_of(2, 3, dev, degenerate=(1,))
    center, size, yaw, rot, disp, count, extents, dirs = call(x, labels, R, t, ego_t, up, A)
    d = dirs.cpu().numpy()
    ref_d = HB.dirs_ref(A)
    assert np.abs(d.view(np.int32).astype(np.int64) - ref_d.view(np.int32)).max() <= 1   # 1 fp32 ulp (all >= 0)
    for b, (xb, lb, Rb, tb) in enumerate(parts):
        ref = HB.boxes_ref(xb, lb, Rb, tb, up, A, ego=(Re[b], te[b], deg[b]), dirs=d)
        assert np.array_equal(extents[b].cpu().numpy(), ref['extents'])
        assert np.array_equal(count[b].cpu().numpy(), ref['count'])
        for k, got in (('center', center), ('size', size), ('displacement', disp)):
            assert np.array_equal(got[b].cpu().numpy(), ref[k]), (b, k)
        y = yaw[b].cpu().numpy()
        assert np.abs(y - ref['yaw']).max() <= 1e-6
        assert np.abs(rot[b].cpu().numpy() - ref['rotation']).max() <= ROT_TOL
        full = ref['count'] > 0
        assert np.array_equal(astar_of(y, A)[full], ref['astar'][full])
        assert np.all((y > -np.pi - 1e-6) & (y <= np.pi + 1e-6))
    # the special slots: one point, collinear (width 0), no finite point, empty
    c = count.cpu().numpy()
    assert np.all(c[:, 3] == 1) and np.all(c[:, 4] == 10) and np.all(c[:, 5:] == 0)
    s = size.cpu().numpy()
    assert np.all(s[:, 3] == 0)
    if A == 90:   # the collinear object's direction, atan(0.5) = 26.57 degrees, is off this grid: only a thin box
        assert np.all(s[:, 4, 1] < 0.1) and np.all(s[:, 4, 2] == 0)
    for o in (5, 6):
        p, q = HB.axes(up)
        basis = np.zeros((3, 3), np.float32)
        basis[p, 0] = basis[q, 1] = basis[up, 2] = 1
        assert np.all(rot[:, o].cpu().numpy() == basis) and np.all(center[:, o].cpu().numpy() == 0)
        assert np.all(yaw[:, o].cpu().numpy() == 0) and np.all(disp[:, o].cpu().numpy() == 0) and np.all(s[:, o] == 0)


def test_collinear_object_on_the_grid_has_width_zero(dev):
    """Points along a grid direction (a = 1 of A = 4: 22.5 degrees) project to one v: width exactly 0 there."""
    A = 4
    d = HB.dirs_ref(A)[1].astype(np.float64)
    s = np.linspace(-2, 2, 9)
    x = np.stack([s * d[0], s * d[1], np.zeros(9)], 1).astype(np.float32)
    ref = HB.boxes_ref(x, np.zeros(9, np.int32), np.eye(3)[None], np.zeros((1, 3)), 2, A)
    xt = torch.tensor(x, device=dev)[None]
    out = call(xt, torch.zeros(1, 9, dtype=torch.int32, device=dev), torch.eye(3, device=dev).expand(1, 1, 3, 3),
               torch.zeros(1, 1, 3, device=dev), None, 2, A)
    assert np.array_equal(out[1][0].cpu().numpy(), ref['size'])
    assert np.array_equal(out[6][0].cpu().numpy(), ref['extents'])
    assert ref['size'][0][1] < 1e-6 and ref['astar'][0] == 1


def test_repeatable_deterministic_batched_and_per_object(dev):
    import pvraft_b200
    (x, labels, R, t), _ = batch((4, 5, 6), dev)
    ego_t, _ = ego_of(3, 7, dev)
    a = call(x, labels, R, t, ego_t, 2, 90)
    b = call(x, labels, R, t, ego_t, 2, 90)
    for u, v in zip(a, b):
        assert same_bits(u, v)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        c = call(x, labels, R, t, ego_t, 2, 90)
    finally:
        torch.use_deterministic_algorithms(was)
    for u, v in zip(a, c):
        assert same_bits(u, v)
    # a batched call equals per-sample calls
    for s in range(3):
        one = call(x[s:s + 1], labels[s:s + 1], R[s:s + 1], t[s:s + 1], tuple(e[s:s + 1] for e in ego_t), 2, 90)
        for u, v in zip(a[:7], one[:7]):
            assert same_bits(u[s:s + 1], v)
    # object o equals the same points labelled as the only object
    for o in (0, 2, 3, 4, 6):
        lo = torch.where(labels == o, 0, -1).int()
        one = call(x, lo, R[:, o:o + 1], t[:, o:o + 1], ego_t, 2, 90)
        for u, v in zip(a[:7], one[:7]):
            assert same_bits(u[:, o:o + 1], v)
    # the public function: the same bits, with the objects' labels and fits
    objs = pvraft_b200.RigidObjects(labels, torch.full((3,), 7, dtype=torch.int32, device=dev), R, t,
                                    torch.zeros(3, 7, dtype=torch.int32, device=dev), torch.zeros(3, 7, dtype=torch.bool, device=dev),
                                    labels >= 0)
    ego = pvraft_b200.RigidMotion(ego_t[0], ego_t[1], torch.ones(3, x.shape[1], dtype=torch.bool, device=dev),
                                  torch.zeros(3, dtype=torch.int32, device=dev), ego_t[2].bool())
    box = pvraft_b200.object_boxes(x, objs, up=2, ego=ego, angles=90)
    for u, v in zip(box, a[:6]):
        assert same_bits(u, v)


@pytest.mark.parametrize('up', [0, 1])
def test_cyclic_permutation_with_up_gives_the_same_boxes(up, dev):
    """x'_k = x_{(k + 2 - up) % 3}, so that x'_{p'}, x'_{q'}, x'_{up'} are x_p, x_q, x_up of up = 2: the same (P, Q, H),
    so the same bits.  The fits are rotation-free (R = I), so the displacement's sums are exact in any order."""
    (x, labels, _, t), _ = batch((8,), dev)
    R = torch.eye(3, device=dev).expand(1, 7, 3, 3).contiguous()
    perm = [(k + 2 - up) % 3 for k in range(3)]
    a = call(x, labels, R, t, None, 2, 90)
    b = call(x[..., perm], labels, R, t[..., perm], None, up, 90)
    for k in (0, 1, 4):   # center, size, displacement: size is (length, width, height) in both
        got = b[k] if k == 1 else b[k][..., [perm.index(j) for j in range(3)]]
        assert same_bits(got, a[k]), k
    for k in (2, 5, 6):   # yaw, count, extents
        assert same_bits(b[k], a[k]), k
    inv = [perm.index(j) for j in range(3)]
    assert same_bits(b[3][..., inv, :], a[3])


def _assert_scene_boxes(box, sc, ego_frame):
    """Both moving boxes of the scene are found, whatever their slots, within the host test's bounds."""
    centre = box.center[0].cpu().numpy()
    for o, ((c, sz), (_, tb)) in enumerate(zip(H.BOXES, H.BOX_MOTIONS)):
        want = c + [0, 0, sz[2] / 2]
        slot = int(np.argmin(np.linalg.norm(centre - want, axis=1)))
        assert int(box.count[0, slot]) > 1000
        assert np.abs(centre[slot] - want).max() < 0.03
        assert np.abs(box.size[0, slot].cpu().numpy() - sz).max() < 0.08
        yaw = float(box.yaw[0, slot])
        d = box.displacement[0, slot].cpu().numpy()
        if ego_frame:
            assert np.abs(d - tb).max() < 0.02, (o, d, tb)
        heading = np.pi if (ego_frame and o == 1) else 0.0   # box 1 moves towards -x in the world, +x relative to the sensor
        assert abs(HB.wrap(yaw - heading)) <= np.radians(1.0), (o, yaw)


def test_chain_recovers_the_scene_boxes_and_lines_up_with_the_tracker(sc, dev):
    import pvraft_b200
    x1 = torch.tensor(sc['xyz1'], device=dev)[None]
    x2 = torch.tensor(sc['xyz2'], device=dev)[None]
    flow = torch.tensor(sc['truth'], dtype=torch.float32, device=dev)[None]
    ego = pvraft_b200.rigid_motion(x1, flow)
    obj = pvraft_b200.rigid_objects(x1, flow, mask=~ego.inliers, flow_radius=0.3, max_objects=8)
    box = pvraft_b200.object_boxes(x1, obj, up=2, ego=ego)
    _assert_scene_boxes(box, sc, True)
    _assert_scene_boxes(pvraft_b200.object_boxes(x1, obj, up=2), sc, False)
    # a box counts every labelled point; its slot is the object's slot, so the tracker's ids name the boxes
    lab = obj.labels[0]
    for o in range(8):
        assert int(box.count[0, o]) == int((lab == o).sum())
    tracks = pvraft_b200.ObjectTracker().step(x1, flow, obj, ego)
    assert torch.equal(tracks.track_id >= 0, box.count > 0)
    # a refined fit gives the same extent, and a displacement as good
    ref = pvraft_b200.rigid_refine(x1, x2, obj)
    rbox = pvraft_b200.object_boxes(x1, ref.fit, up=2, ego=ego)
    assert same_bits(rbox.center, box.center) and same_bits(rbox.size, box.size) and torch.equal(rbox.count, box.count)
    _assert_scene_boxes(rbox, sc, True)


def test_graph_capture_replays_the_same_boxes(dev):
    import pvraft_b200
    (x, labels, R, t), _ = batch((9, 10), dev)
    objs = pvraft_b200.RigidObjects(labels, torch.full((2,), 7, dtype=torch.int32, device=dev), R, t,
                                    torch.zeros(2, 7, dtype=torch.int32, device=dev), torch.zeros(2, 7, dtype=torch.bool, device=dev),
                                    labels >= 0)
    eager = pvraft_b200.object_boxes(x, objs, up=2, angles=256)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pvraft_b200.object_boxes(x, objs, up=2, angles=256)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gout = pvraft_b200.object_boxes(x, objs, up=2, angles=256)
    g.replay()
    torch.cuda.synchronize()
    for u, v in zip(gout, eager):
        assert same_bits(u, v)
