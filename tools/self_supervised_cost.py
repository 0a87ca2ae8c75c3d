"""Cost of training without ground truth: the stage-1 step of `bench.py --mode train` (B=2, N=M=8192, K=512, 8 iterations,
forward + loss + backward + Adam) with the supervised `sequence_loss`, `sequence_self_supervised_loss` (Chamfer + smoothness)
and the same loss with its Laplacian term (`w_laplacian=0.3`), eager and captured as one CUDA graph with a capturable Adam.
The three losses alternate, `--runs` times each; every time is the median of per-step CUDA-event times after `--warmup`
steps.  Then torch.profiler lists the loss kernels of one eager step of each loss (a run of its own), and CUDA events time
the brute-force searches alone on the 8 stacked predictions -- `ops.chamfer` at B=2, N=M=8192 and B=1, N=M=32768, with its
rate in pair evaluations (2 S N M per launch) per second, and the Laplacian term's k_int = 5 search (`ops.laplacian`, S N M
pairs) at B=2, N=M=8192.  Prints the card name and power limit read in the same run.
`python tools/self_supervised_cost.py [--runs 3] [--steps 10] [--warmup 5]`."""
import argparse
import functools
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvraft_b200 import RSF, ops  # noqa: E402
from pvraft_b200.loss import sequence_loss, sequence_self_supervised_loss  # noqa: E402
from tools.bf16_train import _card, _median_ms, _profile  # noqa: E402

B, ITERS = 2, 8   # bench.py --mode train defaults
LOSSES = ('supervised', 'self-supervised', 'laplacian')
LOSS_KERNELS = ('k_chamfer_nn', 'k_chamfer_bwd', 'k_flow_smooth_fwd', 'k_flow_smooth_bwd', 'k_laplacian_fwd', 'k_laplacian_bwd',
                'k_cloud_laplacian', 'k_cloud_laplacian_bwd', 'k_fx_flush')
W_LAPLACIAN, K_LAP, K_INT = 0.3, 10, 5


class TrainStep:
    """bench.py's training step on a fresh copy of fixed weights with one of the three losses; capture() turns it into bench's
    whole-step CUDA graph."""

    def __init__(self, state, dev, pc1, pc2, loss):
        self.model = RSF(bench.make_args())
        self.model.load_state_dict(state)
        self.model = self.model.to(dev).train()
        self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3)
        self.dev, self.pc1, self.pc2 = dev, pc1, pc2
        self.batch = {'sequence': [pc1, pc2], 'ground_truth': [torch.ones_like(pc1[..., :1]), pc2 - pc1]}
        self.loss_fn = {'supervised': sequence_loss, 'self-supervised': sequence_self_supervised_loss,
                        'laplacian': functools.partial(sequence_self_supervised_loss, w_laplacian=W_LAPLACIAN, k_lap=K_LAP, k_int=K_INT)}[loss]
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


def laplacian_search_time(dev, b, n, m, preds=ITERS, calls=20):
    """Median ms of one ops.laplacian launch (the k_int-nearest search, interpolation and residual) over `preds` stacked
    predictions of a batch of b, and its pair evaluations."""
    g = torch.Generator(device=dev).manual_seed(n + 1)
    p1 = torch.rand(b, n, 3, device=dev, generator=g) * 40 - 20
    w = (p1 + torch.randn(preds, b, n, 3, device=dev, generator=g) * 0.1).reshape(preds * b, n, 3).contiguous()
    p2 = torch.rand(b, m, 3, device=dev, generator=g) * 40 - 20
    g1, g2 = ops.knn(p1, p1, K_LAP, mode=0), ops.knn(p2, p2, K_LAP, mode=0)
    l2 = ops.cloud_laplacian(p2, g2)
    return _median_ms(lambda: ops.laplacian(w, p2, l2, g1, K_INT), calls, 3), preds * b * n * m


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
    s, u, lp = med['self-supervised'], med['supervised'], med['laplacian']
    print(f'self-supervised / supervised: eager {s[0] / u[0]:.3f}x, captured {s[1] / u[1]:.3f}x')
    print(f'laplacian / self-supervised: eager {lp[0] / s[0]:.3f}x, captured {lp[1] / s[1]:.3f}x')

    print('kernel time of one eager step (torch.profiler), ms (launches):')
    prof = {k: _profile(eager[k]) for k in LOSSES}
    for name in LOSS_KERNELS + ('k_flow_metrics', 'k_flow_l1_bwd', 'k_knn_brute', 'k_knn_grid'):
        if any(name in prof[k][0] for k in LOSSES):
            print(f'  {name:18} ' + '  '.join(f'{k} {prof[k][0].get(name, 0.0):7.3f} ({prof[k][1].get(name, 0):3d})' for k in LOSSES))
    print('  total              ' + '  '.join(f'{k} {sum(prof[k][0].values()):7.3f}' for k in LOSSES))
    knn_sites = sorted(n for n in prof['self-supervised'][0] if 'knn' in n.lower())
    print(f"  kNN sites of the self-supervised step: {', '.join(knn_sites)}")
    print(f"  kNN launches: {'  '.join(f'{k} {sum(c for n, c in prof[k][1].items() if "knn" in n.lower())}' for k in LOSSES)}")

    print(f'brute-force search alone (ops.chamfer over {ITERS} stacked predictions, both directions), median of 20 launches:')
    for b, n in ((2, 8192), (1, 32768)):
        ms, pairs = search_time(dev, b, n, n)
        print(f'  B={b} N=M={n:6}  {ms:8.3f} ms  {pairs:.3e} pairs  {pairs / ms / 1e9:.3f} Tpairs/s')
    print(f'Laplacian term alone (ops.laplacian over {ITERS} stacked predictions, k_lap={K_LAP}, k_int={K_INT}), median of 20 launches:')
    ms, pairs = laplacian_search_time(dev, B, bench.N_POINTS, bench.N_POINTS)
    print(f'  B={B} N=M={bench.N_POINTS:6}  {ms:8.3f} ms  {pairs:.3e} pairs  {pairs / ms / 1e9:.3f} Tpairs/s')


if __name__ == '__main__':
    main()
