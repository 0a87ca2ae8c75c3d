"""Time the correlation build and a whole forward on large clouds (B = 1), dense up to 49152 points, windowed beyond.

    python tools/large_clouds.py [--sizes 49152 65536 131072] [--iters 8] [--repeat 3] [--out FILE.json]

For every N: CorrBlock.init_module_pm on the feature maps of two synthetic clouds, and one RSF.forward (eager, `--iters`
iterations), each timed with CUDA events after a warm-up, the peak of torch.cuda.max_memory_allocated over the timed calls,
and the scratch bytes of the build's plan (ops.corr_plan: the dense matrix, or the slab + candidate lists of one row block).
The card's name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pvraft_oracle as O           # noqa: E402
from pvraft_b200 import RSF, ops                 # noqa: E402


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ', power limit unknown'


def timed(fn, repeat):
    fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for _ in range(repeat):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return sorted(times)[len(times) // 2], torch.cuda.max_memory_allocated()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', type=int, nargs='+', default=[49152, 65536, 131072])
    ap.add_argument('--iters', type=int, default=8)
    ap.add_argument('--k', type=int, default=512)
    ap.add_argument('--repeat', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    gpu = card()
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=a.k)
    torch.manual_seed(0)
    model = RSF(args).to(dev).eval()
    model.use_cuda_graph = False
    rows = []
    for n in a.sizes:
        pc1, pc2 = (p.to(dev) for p in O.synthetic_clouds(1, n, seed=n))
        plan = ops.corr_plan(1, n, n, 128, a.k)
        with torch.no_grad():
            fmap, _ = model.feature_extractor(torch.cat([pc1, pc2], 0), point_major=True)
            ms_build, mem_build = timed(lambda: model.corr_block.init_module_pm(fmap[:1], fmap[1:], pc2), a.repeat)
            ms_fwd, mem_fwd = timed(lambda: model([pc1, pc2], a.iters), a.repeat)
        row = dict(n=n, path='dense' if plan.dense else f'{len(plan.windows)} windows x {len(plan.row_blocks)} row blocks',
                   init_module_ms=round(ms_build, 2), init_module_peak_gib=round(mem_build / 2**30, 2),
                   forward_ms=round(ms_fwd, 2), forward_peak_gib=round(mem_fwd / 2**30, 2),
                   plan_scratch_gib=round(plan.slab_bytes / 2**30, 3), iters=a.iters, k=a.k, gpu=gpu)
        print(json.dumps(row), flush=True)
        rows.append(row)
        del fmap
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
