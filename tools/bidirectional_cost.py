"""Cost of the flow in both directions.  A graphed `model(p, n, bidirectional=True)` against `model(p, n)` followed by
`model([xyz2, xyz1], n)`, the two arms alternating, at B in {1, 2}, N1 = N2 = 8192 and one unequal pair 8192 / 12288, K = 512,
8 and 32 iterations; CUDA-event times of the consistency kernels alone (brute force and grid, forward and backward, k = 3,
S = 8 stacked predictions at B = 1); and the captured self-supervised training step of tools/self_supervised_cost.py with a
bidirectional forward and w_consistency = 0.3 against the one-direction step.  Every time is a median of per-call CUDA-event
times; repeated runs print median and min-max.  Prints the card name and power limit read in the same run.
`python tools/bidirectional_cost.py [--runs 5] [--calls 10]`."""
import argparse
import functools
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvraft_b200 import RSF, ops  # noqa: E402
from pvraft_b200.loss import sequence_self_supervised_loss  # noqa: E402
from tools.bf16_train import _card, _median_ms  # noqa: E402
from tools.self_supervised_cost import TrainStep  # noqa: E402


def spread(xs):
    xs = sorted(xs)
    return f'{xs[len(xs) // 2]:7.2f} ({xs[0]:.2f}-{xs[-1]:.2f})'


def forward_rows(model, dev, runs, calls):
    print('graphed forward, ms: both directions in one call | two one-direction calls; median (min-max) over runs of the '
          f'median of {calls} calls')
    for b, n1, n2 in ((1, 8192, 8192), (2, 8192, 8192), (1, 8192, 12288)):
        x1, _ = (t.to(dev) for t in bench.synthetic_clouds(b, n1, 1234))
        x2, _ = (t.to(dev) for t in bench.synthetic_clouds(b, n2, 4321))
        for iters in (8, 32):
            with torch.no_grad():
                both = functools.partial(model, [x1, x2], iters, bidirectional=True)

                def two():
                    model([x1, x2], iters)
                    model([x2, x1], iters)

                a, t = [], []
                for _ in range(runs):
                    a.append(_median_ms(both, calls, 3))
                    t.append(_median_ms(two, calls, 3))
            print(f'  B={b} N1={n1} N2={n2} iters={iters:2d}: one call {spread(a)}  two calls {spread(t)}  '
                  f'ratio {sorted(a)[runs // 2] / sorted(t)[runs // 2]:.3f}')


def kernel_rows(dev, calls):
    print(f'consistency kernels alone (S = 8 predictions, B = 1, k = 3), median of {calls} launches, ms:')
    for n in (8192, 32768, 131072):
        g = torch.Generator(device=dev).manual_seed(n)
        p1 = torch.rand(1, n, 3, device=dev, generator=g) * 40 - 20
        p2 = torch.rand(1, n, 3, device=dev, generator=g) * 40 - 20
        f12 = torch.randn(8, n, 3, device=dev, generator=g) * 0.1
        f21 = torch.randn(8, n, 3, device=dev, generator=g) * 0.1
        w = (p1 + f12).contiguous()
        row = []
        for grid in (False, True):
            fwd = functools.partial(ops.flow_consistency, w, f12, p2, f21, 3, 0.01, 0.0025, use_grid=grid)
            _, nn_idx, res, _ = fwd()
            gs = torch.ones(8, device=dev)
            row.append((_median_ms(fwd, calls, 3), _median_ms(lambda: ops.flow_consistency_bwd(w, p2, f21, nn_idx, res, gs), calls, 3)))
        print(f'  N = M = {n:6d}: brute force fwd {row[0][0]:8.3f} bwd {row[0][1]:6.3f}   grid fwd {row[1][0]:8.3f} bwd {row[1][1]:6.3f}')


class BiStep(TrainStep):
    def _step(self):
        self.opt.zero_grad(set_to_none=True)
        flows = self.model([self.pc1, self.pc2], num_iters=8, bidirectional=True)
        self.loss = sequence_self_supervised_loss(flows, self.batch, w_laplacian=0.3, w_consistency=0.3)
        self.loss.backward()
        self.opt.step()


def train_rows(dev, runs, calls):
    torch.manual_seed(0)
    state = RSF(bench.make_args()).state_dict()
    pc1, pc2 = (t.to(dev) for t in bench.synthetic_clouds(2, bench.N_POINTS, 1234))
    one = TrainStep(state, dev, pc1, pc2, 'laplacian').capture()
    bi = BiStep(state, dev, pc1, pc2, 'laplacian').capture()
    a, t = [], []
    for _ in range(runs):
        t.append(_median_ms(one, calls, 3))
        a.append(_median_ms(bi, calls, 3))
    print(f'captured training step B=2 N=M={bench.N_POINTS} 8 iterations, ms: one direction (Chamfer + smoothness + Laplacian) '
          f'{spread(t)}  both directions + consistency 0.3 {spread(a)}  ratio {sorted(a)[runs // 2] / sorted(t)[runs // 2]:.3f}')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=5)
    ap.add_argument('--calls', type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bidirectional_cost.py measures on a CUDA device; none is available')
    dev = torch.device('cuda:0')
    print(f'card: {_card()}')
    torch.manual_seed(0)
    model = RSF(bench.make_args()).to(dev).eval()
    model.use_cuda_graph = True
    forward_rows(model, dev, a.runs, a.calls)
    kernel_rows(dev, 20)
    train_rows(dev, a.runs, a.calls)


if __name__ == '__main__':
    main()
