"""How far from zero-mean are the inputs of this model's GroupNorms?  python tools/gn_conditioning.py [--n 8192] [--b 2]

Every GroupNorm of the library takes var = sum x^2 / n - mean^2 from raw sums, which cancels when a group's mean is r times
its standard deviation (DESIGN.md section 5, "GroupNorm statistics at large mean-to-std ratios").  This prints, for every
GroupNorm of RSF and RSF_refine, the largest r = |mean| / std over samples, groups and calls (a GroupNorm of the RAFT loop
runs once per iteration), measured in float64 on the fp32 oracle's inputs to that GroupNorm:
  default   the seeded default-init weights
  trained   the same weights after --steps Adam steps (lr 1e-3) of the library's own training path (self-supervised loss,
            2 RAFT iterations) on one synthetic rigid-motion pair: P2 = P1 rotated by 5 degrees about z, moved by
            (0.1, -0.05, 0.08), plus 5 mm of noise.  Only RSF trains; RSF_refine reuses its weights with a default refine block.
The flow is evaluated with 8 RAFT iterations on --b synthetic pairs of --n points (the bench clouds, scaled by 0.4)."""
import argparse
import math
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import pvraft_oracle as O  # noqa: E402


def record_ratios(run, W):
    """Run `run()` with the oracle's group_norm instrumented -> {GroupNorm name: largest |mean| / std of its input}."""
    names = {id(v): k[:-len('.weight')] for k, v in W.items() if k.endswith('.weight')}
    worst = {}
    real = O.group_norm

    def rec(x, gamma, beta, groups=O.GN_GROUPS):
        xg = x.detach().double().reshape(x.shape[0], groups, -1)
        r = float((xg.mean(-1).abs() / xg.std(-1, unbiased=False).clamp_min(1e-30)).max())
        name = names.get(id(gamma), '?')
        worst[name] = max(worst.get(name, 0.0), r)
        return real(x, gamma, beta, groups)

    O.group_norm = rec
    try:
        with torch.no_grad():
            run()
    finally:
        O.group_norm = real
    return worst


def rigid_pair(n, seed, dev):
    gen = torch.Generator().manual_seed(seed)
    pc1 = O.synthetic_clouds(1, n, seed=seed)[0] * 0.4
    t = torch.tensor(5.0 * math.pi / 180)
    rot = torch.tensor([[torch.cos(t), -torch.sin(t), 0.0], [torch.sin(t), torch.cos(t), 0.0], [0.0, 0.0, 1.0]])
    pc2 = pc1 @ rot.T + torch.tensor([0.1, -0.05, 0.08]) + torch.randn(pc1.shape, generator=gen) * 0.005
    return pc1.to(dev), pc2.to(dev)


def train(args, W, steps, dev):
    from pvraft_b200 import RSF
    from pvraft_b200.loss import sequence_self_supervised_loss
    m = RSF(args)
    m.load_state_dict(W)
    m = m.to(dev).train()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    pc1, pc2 = rigid_pair(1024, 23, dev)
    batch = {'sequence': [pc1, pc2]}
    first = last = None
    for _ in range(steps):
        opt.zero_grad()
        loss = sequence_self_supervised_loss(m([pc1, pc2], num_iters=2), batch)
        loss.backward()
        opt.step()
        last = float(loss.detach())
        first = last if first is None else first
    print(f'# trained: {steps} Adam steps, self-supervised loss {first:.5f} -> {last:.5f}')
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=8192)
    ap.add_argument('--b', type=int, default=2)
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--iters', type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('gn_conditioning: needs a CUDA device')
    dev = torch.device('cuda:0')
    from pvraft_b200 import RSF_refine
    args = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=512)
    torch.manual_seed(0)
    Wd = {k: v.detach().clone() for k, v in RSF_refine(args).state_dict().items()}
    Wt = dict(Wd)
    Wt.update(train(args, {k: v for k, v in Wd.items() if not k.startswith('refine_block.')}, a.steps, dev))
    pc1, pc2 = (t.to(dev) * 0.4 for t in O.synthetic_clouds(a.b, a.n, seed=1234))
    table = {}
    for tag, W in (('default', Wd), ('trained', Wt)):
        Wg = {k: v.to(dev).float() for k, v in W.items()}
        for model, fwd in (('RSF', O.rsf_forward), ('RSF_refine', O.rsf_refine_forward)):
            r = record_ratios(lambda: fwd(Wg, pc1, pc2, a.iters, 3, 0.25, args.truncate_k), Wg)
            for name, v in r.items():
                table.setdefault((model, name), {})[tag] = v
    print(f'# largest group |mean| / std of each GroupNorm input, B={a.b}, N={a.n}, {a.iters} RAFT iterations')
    print(f'{"model":<11} {"GroupNorm":<48} {"default":>9} {"trained":>9}')
    for (model, name), v in sorted(table.items()):
        if model == 'RSF_refine' and not name.startswith('refine_block.'):
            continue   # (the RAFT part of RSF_refine is RSF's)
        print(f'{model:<11} {name:<48} {v.get("default", float("nan")):9.3g} {v.get("trained", float("nan")):9.3g}')


if __name__ == '__main__':
    main()
