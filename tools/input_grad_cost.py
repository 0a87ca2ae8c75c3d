"""Cost of gradients into the input clouds on the workload of `bench.py --mode train` (B=2, N=8192, K=512, 8 iterations), eager,
with torch.use_deterministic_algorithms off and on:
  - plain:  a training step (forward + loss + backward + Adam) whose clouds do not require grad;
  - inputs: the same step with xyz1 and xyz2 requiring grad;
  - attack: frozen weights (model.requires_grad_(False)), forward + loss + backward into the clouds only.
The settings alternate, `--runs` times each; every time is the median of per-step CUDA-event times after `--warmup` steps.
Then torch.profiler times one eager step of `plain` and of `inputs` in each setting and reports the kernels the input
gradients add: k_lookup_xyz_bwd (the lookup's table gradient, one launch per iteration) and the C = 3 k_edge_bwd calls (the
graphs' edge features: the difference of k_edge_bwd between the two steps), with the deterministic flushes.
Prints the card name and power limit read in the same run.
`python tools/input_grad_cost.py [--runs 3] [--steps 10] [--warmup 3]`."""
import argparse
import os
import re
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvraft_b200 import RSF  # noqa: E402
from tools.deterministic_cost import _card, _median_ms  # noqa: E402

B, ITERS = 2, 8   # bench.py --mode train defaults


def _loss(flows, gt):
    n = len(flows)
    return sum(0.8 ** (n - i - 1) * (flows[i] - gt).abs().sum(-1).mean() for i in range(n))   # bench.py's loss_fn


class Step:
    def __init__(self, state, dev, pc1, pc2, kind):
        self.model = RSF(bench.make_args())
        self.model.load_state_dict(state)
        self.model = self.model.to(dev).train()
        self.kind = kind
        if kind == 'attack':
            self.model.requires_grad_(False)
        else:
            self.opt = torch.optim.Adam(self.model.parameters(), lr=1e-3)
        self.pc1, self.pc2 = pc1, pc2

    def __call__(self):
        x1, x2 = self.pc1, self.pc2
        if self.kind != 'plain':
            x1, x2 = x1.detach().requires_grad_(), x2.detach().requires_grad_()
        if self.kind != 'attack':
            self.opt.zero_grad(set_to_none=True)
        _loss(self.model([x1, x2], num_iters=ITERS), self.pc2 - self.pc1).backward()
        if self.kind != 'attack':
            self.opt.step()


def _kernels(step):
    """Device time (ms) per kernel name (template arguments dropped) of one step."""
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            name = re.sub(r'\(.*', '', re.sub(r'<.*', '', ev.key.replace('void ', '')))
            per[name] = per.get(name, 0.0) + ev.device_time_total / 1e3
    return per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    state = RSF(bench.make_args()).state_dict()
    pc1, pc2 = (t.to(dev) for t in bench.synthetic_clouds(B, bench.N_POINTS, 1234))
    kinds = ('plain', 'inputs', 'attack')
    steps = {k: Step(state, dev, pc1, pc2, k) for k in kinds}
    rows = {(flag, k): [] for flag in (False, True) for k in kinds}
    for _ in range(a.runs):
        for flag in (False, True):
            torch.use_deterministic_algorithms(flag)
            for k in kinds:
                rows[flag, k].append(_median_ms(steps[k], a.steps, a.warmup))
    per = {}
    for flag in (False, True):
        torch.use_deterministic_algorithms(flag)
        per[flag] = {k: _kernels(steps[k]) for k in ('plain', 'inputs')}
    torch.use_deterministic_algorithms(False)

    print(f'card: {_card()}')
    print(f'B={B} N={bench.N_POINTS} K={bench.make_args().truncate_k} iters={ITERS}, eager; median of {a.steps} steps after '
          f'{a.warmup} warm-up steps, ms')
    med = lambda flag, k: sorted(rows[flag, k])[a.runs // 2]
    for flag in (False, True):
        for i in range(a.runs):
            print(f'run {i + 1} deterministic={flag!s:5}  ' + '  '.join(f'{k} {rows[flag, k][i]:7.2f}' for k in kinds))
        print(f'deterministic={flag!s:5} medians: ' + ', '.join(f'{k} {med(flag, k):.2f}' for k in kinds) +
              f'; inputs/plain {med(flag, "inputs") / med(flag, "plain"):.3f}x')
    for flag in (False, True):
        p, q = per[flag]['plain'], per[flag]['inputs']
        added = sorted(((q.get(k, 0.0) - p.get(k, 0.0), k) for k in set(p) | set(q)), reverse=True)
        print(f'deterministic={flag!s:5} kernel time of one step (torch.profiler): plain {sum(p.values()):.2f} ms, inputs '
              f'{sum(q.values()):.2f} ms; k_lookup_xyz_bwd {q.get("pvraft::k_lookup_xyz_bwd", 0.0):.3f} ms, '
              f'C = 3 k_edge_bwd {q.get("pvraft::k_edge_bwd", 0.0) - p.get("pvraft::k_edge_bwd", 0.0):.3f} ms; largest increases:')
        for d, k in added[:6]:
            print(f'  {d:+8.3f} ms  {k}  ({p.get(k, 0.0):.3f} -> {q.get(k, 0.0):.3f})')


if __name__ == '__main__':
    main()
