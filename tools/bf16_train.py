"""Cost of the 'bf16-mixed' training mode on the stage-1 step of `bench.py --mode train` (BASELINE.json configs[3] per GPU:
B=2, N=8192, K=512, 8 iterations, forward + loss + backward + Adam), eager and captured as one CUDA graph with a capturable
Adam as `bench.py --mode train --graph 1` captures it.  'fp32' and 'bf16-mixed' alternate, `--runs` times each; every time is
the median of per-step CUDA-event times after `--warmup` steps.  Then torch.profiler times the kernels of one eager step in
each mode (a run of its own) and lists the weight-gradient kernels (k_linear_wgrad, k_tc_wgrad), k_tc_linear and the total.
Prints the card name and power limit read in the same run.
`python tools/bf16_train.py [--runs 3] [--steps 10] [--warmup 5]`."""
import argparse
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvraft_b200 import RSF  # noqa: E402

B, ITERS = 2, 8   # bench.py --mode train defaults
MODES = ('fp32', 'bf16-mixed')


def _card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def _median_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return sorted(times)[len(times) // 2]


class TrainStep:
    """bench.py's training step on a fresh copy of fixed weights in one precision mode; capture() turns it into bench's
    whole-step CUDA graph."""

    def __init__(self, state, dev, pc1, pc2, mode):
        self.model = RSF(bench.make_args())
        self.model.load_state_dict(state)
        self.model = self.model.to(dev).train().set_precision(mode)
        self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3)
        self.dev, self.pc1, self.pc2 = dev, pc1, pc2
        self.graph = None
        self.loss = None

    def _step(self):
        self.opt.zero_grad(set_to_none=True)
        flows = self.model([self.pc1, self.pc2], num_iters=ITERS)
        gt, n = self.pc2 - self.pc1, len(flows)
        self.loss = sum(0.8 ** (n - i - 1) * (flows[i] - gt).abs().sum(-1).mean() for i in range(n))   # bench.py's loss_fn
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


def _site(name):
    """Kernel name -> its site (template arguments dropped)."""
    name = re.sub(r'<.*', '', name.replace('void ', ''))
    return re.sub(r'\(.*', '', name).replace('pvraft::', '')


def _profile(step):
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    per, calls = {}, {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = _site(ev.key)
            per[k] = per.get(k, 0.0) + ev.device_time_total / 1e3
            calls[k] = calls.get(k, 0) + ev.count
    return per, calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=5)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    state = RSF(bench.make_args()).state_dict()
    pc1, pc2 = (t.to(dev) for t in bench.synthetic_clouds(B, bench.N_POINTS, 1234))

    eager = {m: TrainStep(state, dev, pc1, pc2, m) for m in MODES}
    captured = {m: TrainStep(state, dev, pc1, pc2, m).capture() for m in MODES}
    rows = {m: [] for m in MODES}
    for _ in range(a.runs):
        for m in MODES:
            rows[m].append((_median_ms(eager[m], a.steps, a.warmup), _median_ms(captured[m], a.steps, a.warmup)))

    print(f'card: {_card()}')
    print(f'train step B={B} N={bench.N_POINTS} K={bench.make_args().truncate_k} iters={ITERS} (eager | captured as bench.py '
          f'--graph 1); median of {a.steps} steps after {a.warmup} warm-up steps, ms')
    for i in range(a.runs):
        for m in MODES:
            e, c = rows[m][i]
            print(f'run {i + 1} {m:10}  step eager {e:7.2f}  step captured {c:7.2f}')
    med = {m: [sorted(r[j] for r in rows[m])[a.runs // 2] for j in range(2)] for m in MODES}
    for m in MODES:
        print(f'median {m:10}  step eager {med[m][0]:7.2f}  step captured {med[m][1]:7.2f}')
    print(f"bf16-mixed / fp32: eager {med['bf16-mixed'][0] / med['fp32'][0]:.3f}x, captured {med['bf16-mixed'][1] / med['fp32'][1]:.3f}x")
    print(f"loss after the timed steps: fp32 {float(eager['fp32'].loss.detach()):.4f}, bf16-mixed {float(eager['bf16-mixed'].loss.detach()):.4f}")

    print('kernel time of one eager step (torch.profiler), ms (launches):')
    prof = {m: _profile(eager[m]) for m in MODES}
    for k in ('k_linear_wgrad', 'k_tc_wgrad', 'k_tc_linear', 'k_linear'):
        print(f'  {k:16} ' + '  '.join(f'{m} {prof[m][0].get(k, 0.0):7.3f} ({prof[m][1].get(k, 0):4d})' for m in MODES))
    print('  total            ' + '  '.join(f'{m} {sum(prof[m][0].values()):7.3f}' for m in MODES))


if __name__ == '__main__':
    main()
