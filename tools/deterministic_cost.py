"""Cost of deterministic mode (torch.use_deterministic_algorithms(True)) on bench.py's workloads:
  - the stage-1 training step of `bench.py --mode train` (B=2, N=8192, 8 iterations, forward + loss + backward + Adam), eager,
    and captured as one CUDA graph with a capturable Adam as `bench.py --mode train --graph 1` captures it;
  - the default inference forward of `bench.py` (RSF.forward, batch 8, N=8192, 32 iterations, CUDA-graph replay).
The two settings alternate, `--runs` times each; every time is the median of per-step CUDA-event times after `--warmup`
steps.  Then, in each setting, two steps from identical state (eager, and captured) are compared: the largest |delta param|.
With `--profile`, the kernels of one eager step are timed with torch.profiler in each setting and the per-kernel difference
is listed, largest first (the deterministic instantiations share the default kernels' names up to their template argument).
Prints the card name and power limit read in the same run.
`python tools/deterministic_cost.py [--runs 3] [--steps 10] [--warmup 5] [--profile]`."""
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
    """bench.py's training step on a fresh copy of fixed weights; capture() turns it into bench's whole-step CUDA graph."""

    def __init__(self, state, dev, pc1, pc2):
        self.model = RSF(bench.make_args())
        self.model.load_state_dict(state)
        self.model = self.model.to(dev).train()
        self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3)
        self.dev, self.pc1, self.pc2 = dev, pc1, pc2
        self.graph = None

    def _step(self):
        self.opt.zero_grad(set_to_none=True)
        flows = self.model([self.pc1, self.pc2], num_iters=ITERS)
        gt, n = self.pc2 - self.pc1, len(flows)
        loss = sum(0.8 ** (n - i - 1) * (flows[i] - gt).abs().sum(-1).mean() for i in range(n))   # bench.py's loss_fn
        loss.backward()
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

    def params(self):
        return [p.detach().clone() for p in self.model.parameters()]


def _max_delta(a, b):
    return max(float((x - y).abs().max()) for x, y in zip(a, b))


def _site(name):
    """Kernel name -> the site it belongs to (template arguments, which carry the deterministic flag, dropped)."""
    name = re.sub(r'<.*', '', name.replace('void ', ''))
    return re.sub(r'\(.*', '', name)


def _profile(step):
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[_site(ev.key)] = per.get(_site(ev.key), 0.0) + ev.device_time_total / 1e3
    return per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--profile', action='store_true')
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    state = RSF(bench.make_args()).state_dict()
    pc1, pc2 = (t.to(dev) for t in bench.synthetic_clouds(B, bench.N_POINTS, 1234))

    inf = RSF(bench.make_args())
    inf.load_state_dict(state)
    inf = inf.to(dev).eval()
    inf.use_cuda_graph = True
    q1, q2 = (t.to(dev) for t in bench.synthetic_clouds(8, bench.N_POINTS, 99))

    def forward():
        with torch.no_grad():
            inf([q1, q2], num_iters=bench.ITERS)

    eager, captured = {}, {}
    for flag in (False, True):   # one model per setting; a captured graph belongs to the setting it was captured in
        torch.use_deterministic_algorithms(flag)
        eager[flag] = TrainStep(state, dev, pc1, pc2)
        captured[flag] = TrainStep(state, dev, pc1, pc2).capture()
    rows = {False: [], True: []}
    for _ in range(a.runs):
        for flag in (False, True):
            torch.use_deterministic_algorithms(flag)
            rows[flag].append((_median_ms(eager[flag], a.steps, a.warmup), _median_ms(captured[flag], a.steps, a.warmup),
                               _median_ms(forward, a.steps, a.warmup)))
    delta = {}
    for flag in (False, True):
        torch.use_deterministic_algorithms(flag)
        d = []
        for make in (lambda: TrainStep(state, dev, pc1, pc2), lambda: TrainStep(state, dev, pc1, pc2).capture()):
            after = []
            for _ in range(2):
                s = make()
                s()
                torch.cuda.synchronize()
                after.append(s.params())
            d.append(_max_delta(*after))
        delta[flag] = d
    torch.use_deterministic_algorithms(False)

    print(f'card: {_card()}')
    print(f'train step B={B} N={bench.N_POINTS} iters={ITERS} (eager | captured as bench.py --graph 1); forward B=8 iters={bench.ITERS} '
          f'(graph replay); median of {a.steps} steps after {a.warmup} warm-up steps, ms')
    for i in range(a.runs):
        for flag in (False, True):
            e, c, f = rows[flag][i]
            print(f'run {i + 1} deterministic={flag!s:5}  step eager {e:7.2f}  step captured {c:7.2f}  forward {f:6.2f}')
    for flag in (False, True):
        print(f'deterministic={flag!s:5}  max |dparam| between two steps from identical state: eager {delta[flag][0]:.3g}, '
              f'captured {delta[flag][1]:.3g}')
    med = lambda flag, j: sorted(r[j] for r in rows[flag])[a.runs // 2]
    print('ratio deterministic/default (medians over runs): ' +
          ', '.join(f'{name} {med(True, j) / med(False, j):.3f}x' for j, name in enumerate(('step eager', 'step captured', 'forward'))))

    if a.profile:
        per = {}
        for flag in (False, True):
            torch.use_deterministic_algorithms(flag)
            per[flag] = _profile(eager[flag])
        torch.use_deterministic_algorithms(False)
        diff = sorted(((per[True].get(k, 0.0) - per[False].get(k, 0.0), k) for k in set(per[True]) | set(per[False])), reverse=True)
        print(f'kernel time of one eager step (torch.profiler): default {sum(per[False].values()):.2f} ms, '
              f'deterministic {sum(per[True].values()):.2f} ms; largest increases:')
        for d, k in diff[:10]:
            print(f'  {d:+8.3f} ms  {k}  ({per[False].get(k, 0.0):.3f} -> {per[True].get(k, 0.0):.3f})')


if __name__ == '__main__':
    main()
