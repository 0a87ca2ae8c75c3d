"""Cost of pvraft_b200.rigid_refine (DESIGN.md §4.12): the call time at iterations = 10 for B in {1, 8} and N = M in
{8192, 32768, 131072}, for one ego segment per sample and for 64 objects, and the torch.profiler split of one call between
the normals, the two index builds, k_icp_step and the rest, with the card's name and power limit from the same run.
`python tools/rigid_refine_cost.py [--out DIR]` (writes DIR/rigid_refine_cost.json)."""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pvraft_b200  # noqa: E402


def scan(b, n, seed, dev):
    """A LiDAR-like pair: a ground of 60 x 60 m with walls, and the same surfaces resampled after a small motion."""
    g = torch.Generator(device='cpu').manual_seed(seed)

    def surf(k):
        u = torch.rand(b, k, 3, generator=g) * torch.tensor([60.0, 60.0, 3.0]) - torch.tensor([30.0, 30.0, 0.0])
        kind = torch.randint(0, 3, (b, k, 1), generator=g)
        u[..., 2:] = torch.where(kind == 0, torch.zeros_like(u[..., 2:]), u[..., 2:])
        u[..., :1] = torch.where(kind == 1, torch.round(u[..., :1] / 10) * 10, u[..., :1])
        u[..., 1:2] = torch.where(kind == 2, torch.round(u[..., 1:2] / 10) * 10, u[..., 1:2])
        return u
    c, s = math.cos(0.02), math.sin(0.02)
    R = torch.tensor([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])
    t = torch.tensor([0.8, 0.1, 0.0])
    x1 = surf(n)
    x2 = surf(n) @ R.T + t
    return x1.to(dev), x2.to(dev), R.to(dev), t.to(dev)


def fit_for(x1, R, t, objects):
    b, n = x1.shape[:2]
    dev = x1.device
    if objects == 1:
        return pvraft_b200.RigidMotion(R.expand(b, 3, 3).contiguous(), (0.9 * t).expand(b, 3).contiguous(),
                                       torch.ones(b, n, dtype=torch.bool, device=dev), torch.full((b,), n, dtype=torch.int32, device=dev),
                                       torch.zeros(b, dtype=torch.bool, device=dev))
    # 64 objects: the points split by x into 64 strips
    labels = ((x1[..., 0] + 30) / 60 * objects).long().clamp(0, objects - 1).int()
    return pvraft_b200.RigidObjects(labels, torch.full((b,), objects, dtype=torch.int32, device=dev), R.expand(b, objects, 3, 3).contiguous(),
                                    (0.9 * t).expand(b, objects, 3).contiguous(), torch.zeros(b, objects, dtype=torch.int32, device=dev),
                                    torch.zeros(b, objects, dtype=torch.bool, device=dev), torch.ones(b, n, dtype=torch.bool, device=dev))


def time_call(x1, x2, fit, reps):
    for _ in range(3):
        pvraft_b200.rigid_refine(x1, x2, fit)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        pvraft_b200.rigid_refine(x1, x2, fit)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def split(x1, x2, fit):
    from torch.profiler import ProfilerActivity, profile
    pvraft_b200.rigid_refine(x1, x2, fit)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pvraft_b200.rigid_refine(x1, x2, fit)
        torch.cuda.synchronize()
    parts = {'normals': 0.0, 'index builds': 0.0, 'k_icp_step': 0.0, 'k_icp_solve': 0.0, 'other': 0.0}
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, 'device_time_total') else ev.cuda_time_total
        if us <= 0:
            continue
        k = ev.key
        key = ('normals' if 'k_rf_normals' in k else 'index builds' if 'k_gi_' in k else 'k_icp_step' if 'k_icp_step' in k
               else 'k_icp_solve' if 'k_icp_solve' in k else 'other')
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
            x1, x2, R, t = scan(b, n, 0, dev)
            for objects in (1, 64):
                fit = fit_for(x1, R, t, objects)
                ms = time_call(x1, x2, fit, 20)
                out = pvraft_b200.rigid_refine(x1, x2, fit)
                row = dict(B=b, N=n, objects=objects, ms=round(ms, 3), steps_max=int(out.steps.max()),
                           split_ms={k: round(v, 3) for k, v in split(x1, x2, fit).items()})
                rows.append(row)
                print(json.dumps(row), flush=True)
    result = dict(card=card, iterations=10, rows=rows)
    print(json.dumps(dict(card=card)))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'rigid_refine_cost.json'), 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
