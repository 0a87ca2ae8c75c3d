"""Cost of one ObjectTracker.step (the propagation search with k = 1, k_track_votes, k_track_assign and the ATen glue:
the per-point track ids and the rigid flow kept for the next step), without the flow, the ego-motion or the objects, which
are computed once beforehand.  CUDA-event median over `--steps` repetitions of the second step (each from the state the
first step left) after warm-up, at B in {1, 8}, N in
{8192, 32768, 131072} and O (the slot count, max_objects) in {64, 256}, on a synthetic scene: a static LiDAR-like scene and
O / 2 moving boxes holding a quarter of the points, re-sampled for the second scan.  Then, in a separate pass, each kernel's
device time from torch.profiler, grouped into the search, the two tracking kernels and the ATen glue.  Prints the card name
and power limit read in the same run.  `python tools/object_tracking_cost.py [--steps 20]`."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pvraft_b200  # noqa: E402
from pvraft_b200 import ops  # noqa: E402
from tools.bf16_train import _card, _median_ms  # noqa: E402


def scan(b, n, boxes, dev, g, offset=None):
    """xyz [b,n,3] and flow: 75 % static points over 120 x 120 x 6 m, and `boxes` 1.5 x 1 x 1 m boxes on a 6 m lattice,
    each translated by its own 1 to 2 m (offset: the boxes' motions, reused for the next scan), 1 cm flow noise."""
    k = n // 4 // boxes
    x = torch.rand(b, n, 3, generator=g) * torch.tensor([120.0, 120.0, 6.0]) - torch.tensor([60.0, 60.0, 2.0])
    f = torch.zeros(b, n, 3)
    if offset is None:
        offset = torch.randn(b, boxes, 3, generator=g)
        offset = offset / offset.norm(dim=-1, keepdim=True) * (1.0 + torch.rand(b, boxes, 1, generator=g))
    side = int(boxes ** 0.5 + 0.999)
    for o in range(boxes):
        sl = slice(o * k, (o + 1) * k)
        c = torch.tensor([-50.0 + 6.0 * (o % side), -50.0 + 6.0 * (o // side), 0.0])
        x[:, sl] = c + (torch.rand(b, k, 3, generator=g) - 0.5) * torch.tensor([1.5, 1.0, 1.0])
        f[:, sl] = offset[:, o:o + 1]
    f += torch.randn(b, n, 3, generator=g) * 0.01
    return x.to(dev), f.to(dev), offset


def inputs(b, n, objects, dev):
    """Two consecutive scans of the same boxes, each with its flow, ego-motion and objects."""
    g = torch.Generator().manual_seed(0)
    out, offset = [], None
    for s in range(2):
        x, f, offset = scan(b, n, objects // 2, dev, g, offset)
        if s == 1:   # the boxes have moved by their flow
            k = n // 4 // (objects // 2)
            x[:, :k * (objects // 2)] += offset.to(dev).repeat_interleave(k, dim=1)
        ego = pvraft_b200.rigid_motion(x, f)
        obj = pvraft_b200.rigid_objects(x, f, mask=~ego.inliers, max_objects=objects)
        out.append((x, f, obj, ego))
    return out


def kernel_ms(fn, steps):
    """Device time per step of every kernel fn launches, from torch.profiler, grouped -> {group: ms}."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_time_total <= 0:
            continue
        if 'k_track_votes' in e.key or 'k_track_assign' in e.key:
            group = 'k_track_votes' if 'votes' in e.key else 'k_track_assign'
        elif 'k_flow_propagate' in e.key or 'k_gi_' in e.key:
            group = 'search (k_flow_propagate*, grid index)'
        else:
            group = 'ATen glue (memsets, gather, rigid_flow, copies)'
        out[group] = out.get(group, 0.0) + e.device_time_total * 1e-3 / steps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('object_tracking_cost: needs a CUDA device')
    dev = torch.device('cuda:0')
    print(f'card: {_card()}')
    print(' B       N     O   search   step ms   sample 0')
    profiles = []
    for b in (1, 8):
        for n in (8192, 32768, 131072):
            for objects in (64, 256):
                (x0, f0, obj0, ego0), (x1, f1, obj1, ego1) = inputs(b, n, objects, dev)
                tr = pvraft_b200.ObjectTracker()
                tr.step(x0, f0, obj0, ego0)
                first = tr._prev   # every timed step is the step after scan 0 (the state is only reassigned, never changed)

                def step():
                    tr._prev = first
                    return tr.step(x1, f1, obj1, ego1)

                ms = _median_ms(step, a.steps, 5)
                matched = int((step().matched[0] >= 0).sum())
                form = 'grid' if ops.use_grid_search('flow_propagate', n) else 'brute'
                print(f'{b:2d} {n:7d} {objects:5d}   {form:6s} {ms:9.3f}   {int(obj1.num_objects[0])} objects, {matched} matched')
                if b == 1 or n == 131072:
                    profiles.append((b, n, objects, kernel_ms(step, a.steps)))
    for b, n, objects, ks in profiles:
        print(f'kernel device times, B = {b}, N = {n}, O = {objects} (ms per step):')
        for name, ms in sorted(ks.items(), key=lambda kv: -kv[1]):
            print(f'  {name:48s} {ms:8.4f}')


if __name__ == '__main__':
    main()
