"""What the 'bf16-compute' precision mode buys: BASELINE configs[2] (RSF_refine, B=8, N=8192, K=512, 32 iterations) and the
bench default (RSF, same sizes), each in the modes fp32 / bf16 (state) / bf16-compute, one model per mode with the same
weights and clouds, CUDA-graph replay:
  - the median forward time of `--steps` replays after `--warmup`, the modes alternating, `--runs` times each;
  - the kernel time per RAFT iteration of k_tc_linear and k_update_chain, and of the whole forward, from torch.profiler
    over one eager forward of each mode (a run of its own, after the timing);
  - the final flow's deviation from the fp32 mode, mean-abs / mean|flow|.
Prints the card name and power limit read in the same run.
`python tools/bf16_compute.py [--runs 3] [--steps 10] [--warmup 3]`."""
import argparse
import os
import re
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvraft_b200 import RSF, RSF_refine  # noqa: E402
from tools.deterministic_cost import _card, _median_ms  # noqa: E402

B, ITERS = 8, bench.ITERS
MODES = ('fp32', 'bf16', 'bf16-compute')
LAYERS = ('pvraft::k_tc_linear', 'pvraft::k_update_chain')


def _kernels(fn):
    """Device time (ms) per kernel name (template arguments dropped) of one call of fn."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            name = re.sub(r'\(.*', '', re.sub(r'<.*', '', ev.key.replace('void ', '')))
            per[name] = per.get(name, 0.0) + ev.device_time_total / 1e3
    return per


def workload(refine, dev, a):
    cls = RSF_refine if refine else RSF
    torch.manual_seed(0)
    state = cls(bench.make_args()).state_dict()
    pc1, pc2 = (t.to(dev) for t in bench.synthetic_clouds(B, bench.N_POINTS, 1234))
    models = {}
    for mode in MODES:
        m = cls(bench.make_args())
        m.load_state_dict(state)
        m = m.to(dev).eval().set_precision(mode)
        m.use_cuda_graph = True
        models[mode] = m
    final = lambda out: out if torch.is_tensor(out) else out[-1]   # noqa: E731
    times = {mode: [] for mode in MODES}
    flows = {}
    with torch.no_grad():
        for mode in MODES:
            flows[mode] = final(models[mode]([pc1, pc2], ITERS)).clone()
        for _ in range(a.runs):
            for mode in MODES:
                times[mode].append(_median_ms(lambda: models[mode]([pc1, pc2], ITERS), a.steps, a.warmup))
        per = {}
        for mode in MODES:
            models[mode].use_cuda_graph = False
            per[mode] = _kernels(lambda: models[mode]([pc1, pc2], ITERS))
    ref = flows['fp32']
    name = 'configs[2] RSF_refine' if refine else 'bench default RSF'
    print(f'{name}: B={B} N={bench.N_POINTS} K={bench.TRUNC_K} iters={ITERS}, CUDA-graph replay; median of {a.steps} replays '
          f'after {a.warmup}, ms')
    for i in range(a.runs):
        print(f'  run {i + 1}: ' + '  '.join(f'{mode} {times[mode][i]:7.2f}' for mode in MODES))
    med = {mode: sorted(times[mode])[a.runs // 2] for mode in MODES}
    for mode in MODES:
        p = per[mode]
        dev_rel = float((flows[mode] - ref).abs().mean() / ref.abs().mean())
        layers = '  '.join(f'{k.split("::")[1]} {p.get(k, 0.0) / ITERS:.3f}' for k in LAYERS)
        print(f'  {mode:13s} median {med[mode]:7.2f} ms ({med[mode] / med["fp32"]:.3f}x fp32, {med[mode] / med["bf16"]:.3f}x bf16); '
              f'kernel ms per iteration: {layers}, sum {sum(p.get(k, 0.0) for k in LAYERS) / ITERS:.3f}; whole eager forward '
              f'{sum(p.values()):.2f} ms of kernels; flow vs fp32 {dev_rel:.2e}')
    del models
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bf16_compute.py measures on the GPU: no CUDA device')
    dev = torch.device('cuda:0')
    print(f'card: {_card()}')
    for refine in (True, False):
        workload(refine, dev, a)


if __name__ == '__main__':
    main()
