"""Standalone time of the SetConv edge kernel (ops.setconv_edge) at the shapes a forward launches it at, with CUDA events.
python tools/bench_edge.py [--launches 50] [--det]

Inputs are the real ones: the 32-NN graph from ops.knn and the Morton processing order from ops.point_order over the bench
clouds.  Shapes (bench default, B = 8, N = 8192):
  loop      B = 8,  C = 64, cin = 64  (flow-head SetConv, 32 launches per forward)
  feat1..3  B = 16, C = 16 / 48 / 96, cin = 3 / 32 / 64  (feature encoder over both clouds)
  ctx1..3   B = 8,  same channels  (context encoder over pc1)
Each shape is timed with the Morton order and with order = None (index order), each from its graph's gather plan
(ops.edge_plan, built once per graph and not counted in the launch); the plan build itself is timed once per graph."""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvraft_b200 import ops, Graph  # noqa: E402


def card_line():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the timing below does not depend on it
        return f'(nvidia-smi unavailable: {e})'


def time_launches(run, launches, det=False):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        for _ in range(5):
            run()
        torch.cuda.synchronize()
        times = []
        for _ in range(5):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(launches):
                run()
            e.record()
            torch.cuda.synchronize()
            times.append(s.elapsed_time(e) * 1e3 / launches)
    finally:
        torch.use_deterministic_algorithms(prev)
    return sorted(times)[len(times) // 2], min(times), max(times)


def time_edge(p, g, w, cin, order, plan, launches, det):
    b = p.shape[0]
    st = torch.zeros(b, 8, 2, dtype=torch.float64, device=p.device)
    ymax, ymin = torch.empty_like(p), torch.empty_like(p)
    return time_launches(lambda: ops.setconv_edge(p, g.nbr, g._rel, w, cin, st, ymax, ymin, order=order, plan=plan), launches, det)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=50, help='launches per timed window (5 windows, median reported)')
    ap.add_argument('--det', action='store_true', help='also time the deterministic form')
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    print('card:', card_line())
    b, n = 8, 8192
    pc1, pc2 = [t.to(dev) for t in bench.synthetic_clouds(b, n, 1234)]
    both = torch.cat([pc1, pc2], 0).contiguous()
    g8, g16 = Graph.construct_graph(pc1, 32), Graph.construct_graph(both, 32)
    plans = {}
    for gname, g in (('B=8 ', g8), ('B=16', g16)):
        for oname, order in (('morton', g.order), ('index ', None)):
            plans[id(g), oname] = ops.edge_plan(g.nbr, order)
            med, lo, hi = time_launches(lambda: ops.edge_plan(g.nbr, order), a.launches)
            print(f'edge_plan {gname} {oname}: {med:8.1f} us  (min {lo:.1f}, max {hi:.1f})', flush=True)
    shapes = [('loop ', g8, 64, 64)] + [(f'feat{i + 1}', g16, c, cin) for i, (c, cin) in enumerate([(16, 3), (48, 32), (96, 64)])] \
        + [(f'ctx{i + 1} ', g8, c, cin) for i, (c, cin) in enumerate([(16, 3), (48, 32), (96, 64)])]
    torch.manual_seed(0)
    for label, g, c, cin in shapes:
        bb = g.nbr.shape[0]
        p = torch.randn(bb, n, c, device=dev)
        w = torch.randn(c, cin + 3, device=dev)
        for det in ([False, True] if a.det else [False]):
            for oname, order in (('morton', g.order), ('index ', None)):
                med, lo, hi = time_edge(p, g, w, cin, order, plans[id(g), oname], a.launches, det)
                gathers = bb * n * 32 * c * 4 / 1e9   # neighbour-row bytes the gathers read per launch
                print(f'{label} B={bb:2d} C={c:3d} {"DET " if det else ""}{oname}: {med:8.1f} us  (min {lo:.1f}, max {hi:.1f}; '
                      f'{gathers * 1e3:.0f} MB of neighbour rows, {gathers / (med * 1e-6) / 1e3:.2f} TB/s)', flush=True)


if __name__ == '__main__':
    main()
