"""Where the time of one RSF.forward goes, per kernel and per launch position of the RAFT iteration.

Runs the bench workload (B = 8, N = 8192, 32 iterations) eagerly (`use_cuda_graph = False`) after warm-up, records one
forward with torch.profiler (CUDA activity), and prints
  - the card name and power limit,
  - a per-kernel table of the whole forward (total us, launches, share of the forward's GPU span),
  - for each launch position of the iteration (position 1 = the correlation lookup), the median over iterations in us
    and its share of the forward (median x iterations / forward span).
Tracing slows the host, not the kernels; take end-to-end times from bench.py, not from here.

    python tools/profile_iteration.py [--batch 8] [--iters 32] [--dtype f32|bf16] [--refine] [--json OUT]
"""
import argparse
import collections
import json
import os
import re
import statistics
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvraft_b200 import RSF, RSF_refine  # noqa: E402


def short(name):
    name = re.sub(r'^void ', '', name)
    name = re.sub(r'\(.*$', '', name)
    return name.replace('pvraft::', '')


def card():
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or torch.cuda.get_device_name(0)
    except Exception:   # noqa: BLE001
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--iters', type=int, default=32)
    ap.add_argument('--dtype', choices=['f32', 'bf16'], default='f32')
    ap.add_argument('--refine', action='store_true')
    ap.add_argument('--warm', type=int, default=3)
    ap.add_argument('--json', default=None, help='also write the tables as JSON to this path')
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = (RSF_refine if a.refine else RSF)(bench.make_args()).to(dev).eval()
    if a.dtype == 'bf16':
        model.set_precision('bf16')
    model.use_cuda_graph = False   # per-launch positions need the eager launch sequence
    pc1, pc2 = [t.to(dev) for t in bench.synthetic_clouds(a.batch, bench.N_POINTS, 1234)]
    with torch.no_grad():
        for _ in range(a.warm):
            model([pc1, pc2], a.iters)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            model([pc1, pc2], a.iters)
            torch.cuda.synchronize()
    kernels = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_resource_id is not None:
            t0 = e.time_range.start
            kernels.append((t0, e.time_range.end - t0, short(e.name)))
    kernels.sort()
    span = kernels[-1][0] + kernels[-1][1] - kernels[0][0]

    print(f'card: {card()}')
    print(f'workload: B={a.batch} N={bench.N_POINTS} iters={a.iters} dtype={a.dtype} refine={a.refine}; '
          f'{len(kernels)} GPU activities, forward span {span / 1e3:.3f} ms (eager, traced)')
    per = collections.OrderedDict()
    for _, d, n in kernels:
        t = per.setdefault(n, [0.0, 0])
        t[0] += d
        t[1] += 1
    print(f'\n{"kernel":58s} {"total us":>10s} {"calls":>6s} {"share":>7s}')
    for n, (d, c) in sorted(per.items(), key=lambda kv: -kv[1][0]):
        print(f'{n[:58]:58s} {d:10.1f} {c:6d} {100 * d / span:6.1f}%')

    starts = [i for i, k in enumerate(kernels) if 'k_corr_lookup' in k[2]]
    if len(starts) != a.iters:
        print(f'\nexpected {a.iters} lookup launches, found {len(starts)}: no per-position table')
        return
    # iteration i = launches from lookup i up to lookup i + 1; the last one has the typical length
    length = statistics.mode(starts[i + 1] - starts[i] for i in range(len(starts) - 1))
    iters = [kernels[s:s + length] for s in starts]
    rows = []
    print(f'\nper launch position of the iteration ({length} launches), median over {len(iters)} iterations')
    print(f'{"pos":>3s} {"kernel":50s} {"median us":>10s} {"share":>7s}')
    for pos in range(length):
        names = {it[pos][2] for it in iters if pos < len(it)}
        med = statistics.median(it[pos][1] for it in iters if pos < len(it))
        name = names.pop() if len(names) == 1 else '/'.join(sorted(names))
        rows.append({'pos': pos + 1, 'kernel': name, 'median_us': med, 'share': med * a.iters / span})
        print(f'{pos + 1:3d} {name[:50]:50s} {med:10.1f} {100 * med * a.iters / span:6.1f}%')
    it_span = statistics.median(kernels[starts[i + 1]][0] - kernels[starts[i]][0] for i in range(len(starts) - 1))
    busy = sum(r['median_us'] for r in rows)
    print(f'iteration: median span {it_span:.1f} us, kernel time {busy:.1f} us; loop share of the forward '
          f'{100 * it_span * a.iters / span:.1f}%')
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        json.dump({'card': card(), 'span_us': span, 'kernels': per, 'positions': rows, 'iteration_span_us': it_span},
                  open(a.json, 'w'), indent=1)


if __name__ == '__main__':
    main()
