"""Cost of the nearest-neighbour searches, brute force against the uniform-grid index, at N = M in {8 192, 32 768, 131 072}:
`ops.chamfer` over S = 8 and 16 stacked predictions, `ops.laplacian` at k_int = 5 (S = 8), `ops.flow_propagate` at k = 3 and
`ops.knn` (a kNN graph of the cloud, B = 1) at k = 9 and 32.  Every time is the median of 20 launches timed with CUDA events
after 3 warm-up launches; the grid times include building the index.  Clouds are LiDAR-like (rings on a ground plane, dense
clusters, a sparse far range).  Then a captured self-supervised training step (bench.py --mode train shape: B = 2, N = M =
8192, K = 512, 8 iterations, w_laplacian = 0.3) with the grid forms at the module threshold against the same step with every
search forced to brute force, alternated `--runs` times.  Prints the card name and power limit read in the same run.
`python tools/grid_search_cost.py [--sizes 8192,32768,131072] [--runs 3]`."""
import argparse
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pvraft_b200 import ops  # noqa: E402
from tools.bf16_train import _card, _median_ms  # noqa: E402

CALLS, WARMUP = 20, 3


def lidar(b, n, g, dev):
    out = []
    for _ in range(b):
        n1, n2 = n // 2, n // 4
        n3 = n - n1 - n2
        ring = torch.randint(0, 64, (n1,), generator=g, device=dev).float()
        rad = 3 + ring * 1.2 + torch.rand(n1, generator=g, device=dev) * 0.05
        th = torch.rand(n1, generator=g, device=dev) * 2 * math.pi
        ground = torch.stack([rad * torch.cos(th), rad * torch.sin(th), -1.7 + torch.rand(n1, generator=g, device=dev) * 0.1], 1)
        ctr = (torch.rand(16, 3, generator=g, device=dev) * 40 - 20)[torch.randint(0, 16, (n2,), generator=g, device=dev)]
        clusters = ctr + torch.randn(n2, 3, generator=g, device=dev) * 0.5
        far = torch.cat([torch.rand(n3, 2, generator=g, device=dev) * 160 - 80, torch.rand(n3, 1, generator=g, device=dev) * 6 - 2], 1)
        out.append(torch.cat([ground, clusters, far])[torch.randperm(n, generator=g, device=dev)])
    return torch.stack(out).contiguous()


def both(fn):
    return _median_ms(lambda: fn(False), CALLS, WARMUP), _median_ms(lambda: fn(True), CALLS, WARMUP)


def searches(n, dev):
    g = torch.Generator(device=dev).manual_seed(n)
    rows = []
    p1, p2 = lidar(1, n, g, dev), lidar(1, n, g, dev)
    for s in (8, 16):
        w = (p1.repeat(s, 1, 1) + torch.randn(s, n, 3, generator=g, device=dev) * 0.1).contiguous()
        rows.append((f'chamfer S={s}', both(lambda grid: ops.chamfer(w, p2, use_grid=grid))))
    w = (p1.repeat(8, 1, 1) + torch.randn(8, n, 3, generator=g, device=dev) * 0.1).contiguous()
    g1, g2 = ops.knn(p1, p1, 10, mode=0), ops.knn(p2, p2, 10, mode=0)
    l2 = ops.cloud_laplacian(p2, g2)
    rows.append(('laplacian S=8 k_int=5', both(lambda grid: ops.laplacian(w, p2, l2, g1, 5, use_grid=grid))))
    flow = (torch.randn(1, n, 3, generator=g, device=dev) * 0.1).contiguous()
    rows.append(('flow_propagate k=3', both(lambda grid: ops.flow_propagate(p1, flow, p2, 3, use_grid=grid))))
    for k in (9, 32):
        # use_sweep: the grid search (the shared-memory sort up to 16 384 points, the counting sort beyond)
        rows.append((f'knn graph k={k}', both(lambda grid: ops.knn(p1, p1, k, mode=0, use_sweep=grid))))
    return rows


def train_step(runs):
    import bench
    from tools.self_supervised_cost import TrainStep
    from pvraft_b200 import RSF
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    state = RSF(bench.make_args()).state_dict()
    pc1, pc2 = (t.to(dev) for t in bench.synthetic_clouds(2, bench.N_POINTS, 1234))
    thresholds = dict(ops.GRID_SEARCH_MIN_POINTS)
    steps = {}
    for name, t in (('brute force', {k: 1 << 40 for k in thresholds}), ('grid', thresholds)):
        ops.GRID_SEARCH_MIN_POINTS.update(t)   # read while the step is captured
        steps[name] = TrainStep(state, dev, pc1, pc2, 'laplacian').capture()
    ops.GRID_SEARCH_MIN_POINTS.update(thresholds)
    times = {k: [] for k in steps}
    for _ in range(runs):
        for name, step in steps.items():
            times[name].append(_median_ms(step, 10, 5))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='8192,32768,131072')
    ap.add_argument('--runs', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('grid_search_cost.py measures on a CUDA device; none is available')
    dev = torch.device('cuda:0')
    print(f'card: {_card()}')
    print(f'GRID_SEARCH_MIN_POINTS = {ops.GRID_SEARCH_MIN_POINTS}')
    print(f'median of {CALLS} launches, ms (brute force | grid, index build included)')
    for n in (int(x) for x in a.sizes.split(',')):
        for name, (brute, grid) in searches(n, dev):
            print(f'  N=M={n:6}  {name:24} brute {brute:9.3f}  grid {grid:8.3f}  {brute / grid:7.1f}x')
    times = train_step(a.runs)
    print('captured self-supervised step B=2 N=M=8192 K=512 iters=8 w_laplacian=0.3, median of 10 steps, ms:')
    for name, t in times.items():
        print(f'  {name:12} ' + '  '.join(f'{x:7.2f}' for x in t) + f'   median {sorted(t)[len(t) // 2]:7.2f}')


if __name__ == '__main__':
    main()
