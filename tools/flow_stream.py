"""Cost of estimating scene flow along a scan sequence: `SceneFlowStream.step` (every scan encoded once; cold, and warm-started
from the previous pair's flow) against one `model(p)` call per pair, at B = 1 and 2, N = 8192 points per scan, K = 512, 8 and 32
iterations, all with CUDA-graph replay (the default at B <= 2).  The arms alternate `--runs` times; every time is the median
of per-scan CUDA-event times over `--steps` scans after `--warmup` scans.  Then CUDA events time pvraft_flow_propagate_fwd
alone (k = 3) at N = M = 8192, N = M = 32768 and one unequal pair, with its rate in point pairs (B N M) per second.  Prints
the card name and power limit read in the same run.

The scans are seeded synthetic: each samples a 40 m x 40 m x 4 m scene anew (points do not correspond between scans), the
scene moves rigidly (a turn about z and a translation per scan), a box in it moves on its own, with 2 cm of noise.
`python tools/flow_stream.py [--runs 3] [--steps 10] [--warmup 3]`."""
import argparse
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvraft_b200 import RSF, SceneFlowStream, ops  # noqa: E402
from tools.bf16_train import _card, _median_ms  # noqa: E402

N = 8192
ARMS = ('pairs', 'stream cold', 'stream warm')


def scan_sequence(b, n, count, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    scans = []
    for t in range(count):
        pts = torch.rand(b, n, 3, device=dev, generator=g) * torch.tensor([40.0, 40.0, 4.0], device=dev) - torch.tensor(
            [20.0, 20.0, 0.0], device=dev)
        in_box = ((pts[..., 0] - 5).abs() < 3) & ((pts[..., 1] + 5).abs() < 2)
        a = 0.01 * t
        rot = torch.tensor([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]], device=dev)
        pts = pts @ rot.T + torch.tensor([0.8, 0.1, 0.0], device=dev) * t + in_box.unsqueeze(-1) * torch.tensor([0.0, 0.5, 0.0], device=dev) * t
        scans.append((pts + 0.02 * torch.randn(b, n, 3, device=dev, generator=g)).contiguous())
    return scans


class Arm:
    """One scan per call: the next pair through model(p), or the next scan through a stream."""

    def __init__(self, model, scans, iters, arm):
        self.model, self.scans, self.iters, self.arm, self.t = model, scans, iters, arm, 0
        self.stream = None if arm == 'pairs' else SceneFlowStream(model, iters, warm_start=arm == 'stream warm')
        if self.stream is not None:
            self.stream.step(scans[0])

    def __call__(self):
        self.t += 1
        if self.t >= len(self.scans):   # start the sequence over (the stream from a new first scan)
            self.t = 1
            if self.stream is not None:
                self.stream.reset()
                self.stream.step(self.scans[0])
        with torch.no_grad():
            if self.stream is None:
                return self.model([self.scans[self.t - 1], self.scans[self.t]], self.iters)
            return self.stream.step(self.scans[self.t])


def propagate_time(dev, n, m, k=3, calls=20):
    g = torch.Generator(device=dev).manual_seed(n + m)
    xyz_prev = torch.rand(1, m, 3, device=dev, generator=g) * 40 - 20
    flow_prev = torch.randn(1, m, 3, device=dev, generator=g) * 0.5
    xyz = torch.rand(1, n, 3, device=dev, generator=g) * 40 - 20
    return _median_ms(lambda: ops.flow_propagate(xyz_prev, flow_prev, xyz, k), calls, 3), n * m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('flow_stream.py measures on a CUDA device; none is available')
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = RSF(bench.make_args()).to(dev).eval()
    print(f'card: {_card()}')
    print(f'per-scan time, N={N} K={bench.make_args().truncate_k}, CUDA-graph replay; median of {a.steps} scans after {a.warmup} '
          f'warm-up scans, ms')
    for b in (1, 2):
        scans = scan_sequence(b, N, a.steps + a.warmup + 2, dev)
        for iters in (8, 32):
            arms = {k: Arm(model, scans, iters, k) for k in ARMS}
            rows = {k: [] for k in ARMS}
            for _ in range(a.runs):
                for k in ARMS:
                    rows[k].append(_median_ms(arms[k], a.steps, a.warmup))
            med = {k: sorted(rows[k])[a.runs // 2] for k in ARMS}
            runs = '  '.join(f"{k} [{', '.join(f'{v:.2f}' for v in rows[k])}]" for k in ARMS)
            print(f'B={b} iters={iters:2}  ' + '  '.join(f'{k} {med[k]:7.2f}' for k in ARMS) +
                  f"  stream/pairs {med['stream cold'] / med['pairs']:.3f}x  runs: {runs}")
            del arms
            model.reset_graphs()
    print('pvraft_flow_propagate_fwd alone (B=1, k=3), median of 20 launches:')
    for n, m in ((8192, 8192), (32768, 32768), (12000, 8192)):
        ms, pairs = propagate_time(dev, n, m)
        print(f'  N={n:6} M={m:6}  {ms * 1e3:9.1f} us  {pairs:.3e} pairs  {pairs / ms / 1e9:.3f} Tpairs/s')


if __name__ == '__main__':
    main()
