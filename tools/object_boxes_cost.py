"""Cost of pvraft_b200.object_boxes (DESIGN.md §4.13): the call time over 20 calls for B in {1, 8}, N in {8192, 32768,
131072}, 64 objects and angles in {90, 256}, and the torch.profiler split of one call between the grouping, k_box_extents
and k_box_finalize, with the card's name and power limit from the same run.  For scale, the time of the rigid_objects
call that finds the same objects is measured beside it.
`python tools/object_boxes_cost.py [--out DIR]` (writes DIR/object_boxes_cost.json)."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pvraft_b200  # noqa: E402

OBJECTS = 64


def scene(b, n, seed, dev):
    """64 boxes of 1-5 m on an 80 x 80 m ground at random yaws, each moving by its own small motion; every point labelled
    with its box (the clustering's output), the fits their true motions."""
    g = torch.Generator(device='cpu').manual_seed(seed)
    o = torch.randint(0, OBJECTS, (b, n), generator=g)
    centre = torch.rand(b, OBJECTS, 3, generator=g) * torch.tensor([80.0, 80.0, 0.0]) - torch.tensor([40.0, 40.0, 0.0])
    size = torch.rand(b, OBJECTS, 3, generator=g) * 4 + 1
    yaw = torch.rand(b, OBJECTS, generator=g) * 2 * math.pi
    local = (torch.rand(b, n, 3, generator=g) - torch.tensor([0.5, 0.5, 0.0])) * torch.gather(size, 1, o[..., None].expand(-1, -1, 3))
    face = torch.randint(0, 2, (b, n), generator=g)   # the points on the box's -x or -y face: an L-shaped view
    local[..., 0] = torch.where(face == 0, -0.5 * torch.gather(size[..., 0], 1, o), local[..., 0])
    local[..., 1] = torch.where(face == 1, -0.5 * torch.gather(size[..., 1], 1, o), local[..., 1])
    c, s = torch.cos(torch.gather(yaw, 1, o)), torch.sin(torch.gather(yaw, 1, o))
    x = torch.stack([c * local[..., 0] - s * local[..., 1], s * local[..., 0] + c * local[..., 1], local[..., 2]], -1)
    x = x + torch.gather(centre, 1, o[..., None].expand(-1, -1, 3))
    a = (torch.rand(b, OBJECTS, generator=g) - 0.5) * 0.1
    R = torch.zeros(b, OBJECTS, 3, 3)
    R[..., 0, 0], R[..., 0, 1], R[..., 1, 0], R[..., 1, 1], R[..., 2, 2] = torch.cos(a), -torch.sin(a), torch.sin(a), torch.cos(a), 1
    t = torch.randn(b, OBJECTS, 3, generator=g) * torch.tensor([1.0, 1.0, 0.0])
    objs = pvraft_b200.RigidObjects(o.int().to(dev), torch.full((b,), OBJECTS, dtype=torch.int32, device=dev), R.to(dev), t.to(dev),
                                    torch.zeros(b, OBJECTS, dtype=torch.int32, device=dev), torch.zeros(b, OBJECTS, dtype=torch.bool, device=dev),
                                    torch.ones(b, n, dtype=torch.bool, device=dev))
    ego = pvraft_b200.RigidMotion(torch.eye(3, device=dev).expand(b, 3, 3).contiguous(), torch.tensor([[0.9, 0.1, 0.0]] * b, device=dev),
                                  torch.zeros(b, n, dtype=torch.bool, device=dev), torch.zeros(b, dtype=torch.int32, device=dev),
                                  torch.zeros(b, dtype=torch.bool, device=dev))
    return x.to(dev), objs, ego


def time_call(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def split(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    parts = {'grouping': 0.0, 'k_box_extents': 0.0, 'k_box_finalize': 0.0, 'other': 0.0}
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
        if us <= 0:
            continue
        k = ev.key
        key = ('grouping' if 'k_ro_group' in k else 'k_box_extents' if 'k_box_extents' in k else 'k_box_finalize' if 'k_box_finalize' in k
               else 'other')
        parts[key] += us / 1000
    return parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    rows = []
    for b in (1, 8):
        for n in (8192, 32768, 131072):
            x, objs, ego = scene(b, n, 0, dev)
            flow = torch.zeros_like(x)
            clusters_ms = time_call(lambda: pvraft_b200.rigid_objects(x, flow, max_objects=OBJECTS), 20)
            for angles in (90, 256):
                def fn():
                    return pvraft_b200.object_boxes(x, objs, up=2, ego=ego, angles=angles)
                ms = time_call(fn, 20)
                row = dict(B=b, N=n, objects=OBJECTS, angles=angles, ms=round(ms, 3), rigid_objects_ms=round(clusters_ms, 3),
                           split_ms={k: round(v, 3) for k, v in split(fn).items()})
                rows.append(row)
                print(json.dumps(row), flush=True)
    result = dict(card=card, rows=rows)
    print(json.dumps(dict(card=card)))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'object_boxes_cost.json'), 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
