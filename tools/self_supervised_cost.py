"""Cost of training without ground truth: the stage-1 step of `bench.py --mode train` (B=2, N=M=8192, K=512, 8 iterations,
forward + loss + backward + Adam) with the supervised `sequence_loss` against `sequence_self_supervised_loss`, eager and captured
as one CUDA graph with a capturable Adam.  The two losses alternate, `--runs` times each; every time is the median of per-step
CUDA-event times after `--warmup` steps.  Then torch.profiler lists the loss kernels of one eager self-supervised step (a run
of its own), and CUDA events time the brute-force search alone (`ops.chamfer` on the 8 stacked predictions) at B=2, N=M=8192
and B=1, N=M=32768, with its rate in pair evaluations (2 S N M per launch) per second.  Prints the card name and power limit
read in the same run.
`python tools/self_supervised_cost.py [--runs 3] [--steps 10] [--warmup 5]`."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvraft_b200 import RSF, ops  # noqa: E402
from pvraft_b200.loss import sequence_loss, sequence_self_supervised_loss  # noqa: E402
from tools.bf16_train import _card, _median_ms, _profile  # noqa: E402

B, ITERS = 2, 8   # bench.py --mode train defaults
LOSSES = ('supervised', 'self-supervised')
LOSS_KERNELS = ('k_chamfer_nn', 'k_chamfer_bwd', 'k_flow_smooth_fwd', 'k_flow_smooth_bwd', 'k_fx_flush')


class TrainStep:
    """bench.py's training step on a fresh copy of fixed weights with one of the two losses; capture() turns it into bench's
    whole-step CUDA graph."""

    def __init__(self, state, dev, pc1, pc2, loss):
        self.model = RSF(bench.make_args())
        self.model.load_state_dict(state)
        self.model = self.model.to(dev).train()
        self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3)
        self.dev, self.pc1, self.pc2 = dev, pc1, pc2
        self.batch = {'sequence': [pc1, pc2], 'ground_truth': [torch.ones_like(pc1[..., :1]), pc2 - pc1]}
        self.loss_fn = sequence_loss if loss == 'supervised' else sequence_self_supervised_loss
        self.graph = None
        self.loss = None

    def _step(self):
        self.opt.zero_grad(set_to_none=True)
        flows = self.model([self.pc1, self.pc2], num_iters=ITERS)
        self.loss = self.loss_fn(flows, self.batch)
        self.loss.backward()
        self.opt.step()

    def __call__(self):
        if self.graph is None:
            self._step()
        else:
            self.graph.replay()

    def capture(self):
        self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3, capturable=True)
        side = torch.cuda.Stream(device=self.dev)
        side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(side):
            for _ in range(3):
                self._step()
        torch.cuda.current_stream(self.dev).wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._step()
        return self


def search_time(dev, b, n, m, preds=ITERS, calls=20):
    """Median ms of one ops.chamfer launch over `preds` stacked predictions of a batch of b, and its pair evaluations."""
    g = torch.Generator(device=dev).manual_seed(n)
    w = torch.rand(preds * b, n, 3, device=dev, generator=g) * 40 - 20
    p2 = torch.rand(b, m, 3, device=dev, generator=g) * 40 - 20
    return _median_ms(lambda: ops.chamfer(w, p2), calls, 3), 2 * preds * b * n * m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('self_supervised_cost.py measures on a CUDA device; none is available')
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    state = RSF(bench.make_args()).state_dict()
    pc1, pc2 = (t.to(dev) for t in bench.synthetic_clouds(B, bench.N_POINTS, 1234))

    eager = {k: TrainStep(state, dev, pc1, pc2, k) for k in LOSSES}
    captured = {k: TrainStep(state, dev, pc1, pc2, k).capture() for k in LOSSES}
    rows = {k: [] for k in LOSSES}
    for _ in range(a.runs):
        for k in LOSSES:
            rows[k].append((_median_ms(eager[k], a.steps, a.warmup), _median_ms(captured[k], a.steps, a.warmup)))

    print(f'card: {_card()}')
    print(f'train step B={B} N=M={bench.N_POINTS} K={bench.make_args().truncate_k} iters={ITERS} (eager | captured as bench.py '
          f'--graph 1); median of {a.steps} steps after {a.warmup} warm-up steps, ms')
    for i in range(a.runs):
        for k in LOSSES:
            e, c = rows[k][i]
            print(f'run {i + 1} {k:16}  step eager {e:7.2f}  step captured {c:7.2f}')
    med = {k: [sorted(r[j] for r in rows[k])[a.runs // 2] for j in range(2)] for k in LOSSES}
    for k in LOSSES:
        print(f'median {k:16}  step eager {med[k][0]:7.2f}  step captured {med[k][1]:7.2f}')
    s, u = med['self-supervised'], med['supervised']
    print(f'self-supervised / supervised: eager {s[0] / u[0]:.3f}x, captured {s[1] / u[1]:.3f}x')

    print('kernel time of one eager step (torch.profiler), ms (launches):')
    prof = {k: _profile(eager[k]) for k in LOSSES}
    for name in LOSS_KERNELS + ('k_flow_metrics', 'k_flow_l1_bwd', 'k_knn_brute', 'k_knn_grid'):
        if any(name in prof[k][0] for k in LOSSES):
            print(f'  {name:18} ' + '  '.join(f'{k} {prof[k][0].get(name, 0.0):7.3f} ({prof[k][1].get(name, 0):3d})' for k in LOSSES))
    print('  total              ' + '  '.join(f'{k} {sum(prof[k][0].values()):7.3f}' for k in LOSSES))
    knn_sites = sorted(n for n in prof['self-supervised'][0] if 'knn' in n.lower())
    print(f"  kNN sites of the self-supervised step: {', '.join(knn_sites)}")

    print(f'brute-force search alone (ops.chamfer over {ITERS} stacked predictions, both directions), median of 20 launches:')
    for b, n in ((2, 8192), (1, 32768)):
        ms, pairs = search_time(dev, b, n, n)
        print(f'  B={b} N=M={n:6}  {ms:8.3f} ms  {pairs:.3e} pairs  {pairs / ms / 1e9:.3f} Tpairs/s')


if __name__ == '__main__':
    main()
