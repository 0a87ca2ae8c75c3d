"""Cost of the rigid-motion fit (pvraft_b200.rigid_motion): CUDA-event times of the forward, of the forward with a mask that
allows 9 points in 10, and of forward + backward at B in {1, 8}, N in {8192, 32768, 131072}, H in {256, 1024} hypotheses,
rounds = 2, on LiDAR-like scenes (ego-motion, two moving objects, 1 cm noise, threshold 0.05), and the score kernel's own time from torch.profiler in a separate pass, as
point-hypothesis tests per second (B N H over its time).  Every time is a median over `--calls` calls.  Prints the card name
and power limit read in the same run.  `python tools/rigid_motion_cost.py [--calls 20]`."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pvraft_b200  # noqa: E402
from tools.bf16_train import _card, _median_ms  # noqa: E402


def scene(b, n, dev, seed=0):
    """xyz1, flow [b,n,3]: a rotation of a few degrees and a translation of about a metre for 80 % of the points, two
    objects moving 1 m further, 1 cm noise."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(b, n, 3, generator=g) * torch.tensor([120.0, 120.0, 6.0]) - torch.tensor([60.0, 60.0, 2.0])
    c, s = torch.cos(torch.tensor(0.05)), torch.sin(torch.tensor(0.05))
    R = torch.tensor([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
    y = x @ R.T + torch.tensor([1.0, 0.2, 0.0])
    y[:, : n // 10] += torch.tensor([1.0, 0.0, 0.0])
    y[:, n // 10: n // 5] += torch.tensor([0.0, -1.0, 0.0])
    y += torch.randn(b, n, 3, generator=g) * 0.01
    return x.to(dev), (y - x).to(dev)


def score_seconds(x, f, h, calls):
    """Device time of k_rigid_score per call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            pvraft_b200.rigid_motion(x, f, threshold=0.05, hypotheses=h, rounds=2)
        torch.cuda.synchronize()
    total = sum(e.device_time_total for e in prof.key_averages() if 'k_rigid_score' in e.key)
    return total * 1e-6 / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('rigid_motion_cost: needs a CUDA device')
    dev = torch.device('cuda:0')
    print(f'card: {_card()}')
    rows = []
    for b in (1, 8):
        for n in (8192, 32768, 131072):
            x, f = scene(b, n, dev)
            xg, fg = x.clone().requires_grad_(True), f.clone().requires_grad_(True)
            gR, gt = torch.randn(b, 3, 3, device=dev), torch.randn(b, 3, device=dev)
            mask = (torch.arange(n, device=dev) % 10 != 0).expand(b, n).contiguous()
            for h in (256, 1024):
                def fwd():
                    pvraft_b200.rigid_motion(x, f, threshold=0.05, hypotheses=h, rounds=2)

                def fwd_masked():
                    pvraft_b200.rigid_motion(x, f, mask=mask, threshold=0.05, hypotheses=h, rounds=2)

                def fwd_bwd():
                    out = pvraft_b200.rigid_motion(xg, fg, threshold=0.05, hypotheses=h, rounds=2)
                    torch.autograd.grad((out.rotation * gR).sum() + (out.translation * gt).sum(), (xg, fg))

                t_f = _median_ms(fwd, a.calls, 5)
                t_m = _median_ms(fwd_masked, a.calls, 5)
                t_fb = _median_ms(fwd_bwd, a.calls, 5)
                rows.append((b, n, h, t_f, t_m, t_fb, x, f))
    print(' B       N     H   forward ms   masked fwd ms   fwd+bwd ms   score kernel ms   tests/s')
    for b, n, h, t_f, t_m, t_fb, x, f in rows:
        sc = score_seconds(x, f, h, a.calls)
        print(f'{b:2d} {n:7d} {h:5d} {t_f:12.3f} {t_m:15.3f} {t_fb:12.3f} {sc * 1e3:17.4f} {b * n * h / sc:9.3e}')


if __name__ == '__main__':
    main()
