"""Micro-benchmark of the wgmma fused layer: python tools/bench_tc.py"""
import os, sys, json
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pvraft_b200 import ops
dev = torch.device('cuda:0')
b, n = int(os.environ.get('TC_B', '8')), 8192
def run(cin, cout, stats, reps=30, srcs=1):
    xs = [torch.randn(b, n, cin // srcs, device=dev) for _ in range(srcs)]
    w = torch.randn(cout, cin, device=dev) / cin ** 0.5
    tw = ops.tc_weights(w)
    st = torch.zeros(b, 8, 2, dtype=torch.float64, device=dev) if stats else None
    out = torch.empty(b, n, cout, device=dev)
    for _ in range(3):
        ops.tc_linear(xs, tw, out=out, out_stats=st)
    torch.cuda.synchronize()
    # queue the launches behind a long kernel so that the GPU runs them back to back (the python launch path costs
    # ~20 us per call and would otherwise be what is measured)
    big = torch.randn(8192, 8192, device=dev)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3): big @ big
    s.record()
    for _ in range(reps):
        ops.tc_linear(xs, tw, out=out, out_stats=st)
    e.record()
    torch.cuda.synchronize()
    t = s.elapsed_time(e) * 1e3 / reps
    byt = b * n * (cin + cout) * 4
    print(json.dumps(dict(cin=cin, cout=cout, stats=stats, srcs=srcs, us=round(t, 1), GBps=round(byt / t / 1e3), TFLOPs=round(2 * b * n * cin * cout * 3 / t / 1e6, 1))))
for cin, cout, stats, srcs in [(32, 64, False, 1), (64, 64, False, 1), (64, 64, True, 1), (128, 64, False, 1), (192, 64, False, 3), (192, 128, False, 3),
                               (96, 128, True, 1), (64, 32, False, 1), (64, 128, False, 1), (256, 64, False, 1)]:
    run(cin, cout, stats, srcs=srcs)
