"""Cost of pairs of clouds of different sizes: a CUDA-graphed RSF forward at B = 1, K = 512, 32 iterations.

    python tools/unequal_clouds.py [--pairs 8192x8192 8192x12288 ...] [--iters 32] [--replays 30] [--out FILE.json]

For every (N1, N2), in one run:
  * the median CUDA-event time of --replays graph replays after the capture and a warm-up;
  * the peak of torch.cuda.max_memory_allocated from before the first call of that shape (capture pool included);
  * the lookup kernel's time per iteration, from torch.profiler over one eager forward (sum of k_corr_lookup durations / iters);
  * whether the lookup stages the gather table of the N2-point cloud in shared memory (ops.lookup_table_in_smem);
and the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pvraft_b200 import RSF, ops                 # noqa: E402

PAIRS = ['8192x8192', '8192x12288', '12288x8192', '8192x16384', '40000x60000']


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ', power limit unknown'


def clouds(n1, n2, seed):
    """pc1 = 10 U[0,1)^3 with N1 points; pc2 = a displaced copy of the same region with N2 points (the synthetic workload's
    scene, sampled twice)."""
    g = torch.Generator().manual_seed(seed)
    pc1 = 10.0 * torch.rand(1, n1, 3, generator=g)
    pc2 = 10.0 * torch.rand(1, n2, 3, generator=g) + 0.1 * torch.randn(1, n2, 3, generator=g)
    return pc1.cuda(), pc2.cuda()


def lookup_ms_per_iter(model, p, iters):
    model.use_cuda_graph = False
    with torch.no_grad():
        model(p, iters)                                  # warm (weight splits, derived constants)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            model(p, iters)
            torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if 'k_corr_lookup' in e.key)
    model.use_cuda_graph = True
    return us / 1e3 / iters


def measure(n1, n2, k, iters, replays):
    torch.manual_seed(0)
    model = RSF(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k)).cuda().eval()
    model.use_cuda_graph = True
    p = list(clouds(n1, n2, n1 + n2))
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        for _ in range(3):                               # capture + warm-up replays
            model(p, iters)
        torch.cuda.synchronize()
        times = []
        for _ in range(replays):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            model(p, iters)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b))
    peak = torch.cuda.max_memory_allocated() - base
    row = dict(n1=n1, n2=n2, k=k, iters=iters, replays=replays, median_ms=statistics.median(times), min_ms=min(times),
               max_ms=max(times), peak_mib=peak / 2 ** 20, table_in_smem=ops.lookup_table_in_smem(n2, k),
               lookup_ms_per_iter=lookup_ms_per_iter(model, p, iters))
    del model
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', nargs='+', default=PAIRS, help='N1xN2 pairs')
    ap.add_argument('--k', type=int, default=512)
    ap.add_argument('--iters', type=int, default=32)
    ap.add_argument('--replays', type=int, default=30)
    ap.add_argument('--out', default=None, help='also write the rows as JSON to this path')
    a = ap.parse_args()
    info = card()
    print(f'card: {info}')
    rows = []
    print(f'{"N1":>6} {"N2":>6} {"median ms":>10} {"min-max ms":>15} {"peak MiB":>9} {"lookup ms/iter":>15} {"table in smem":>14}')
    for pr in a.pairs:
        n1, n2 = (int(x) for x in pr.split('x'))
        r = measure(n1, n2, a.k, a.iters, a.replays)
        rows.append(r)
        print(f'{n1:>6} {n2:>6} {r["median_ms"]:>10.2f} {r["min_ms"]:>7.2f}-{r["max_ms"]:<7.2f} {r["peak_mib"]:>9.0f} '
              f'{r["lookup_ms_per_iter"]:>15.3f} {str(r["table_in_smem"]):>14}', flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == '__main__':
    main()
