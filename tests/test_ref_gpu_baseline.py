"""Not a parity test: times the REFERENCE FORMULATION (the oracle's torch op sequence = the reference's own
ATen op sequence, model/corr.py + model/update.py + model/flot/*) on the GPU itself, fp32, TF32 off --
"the reference GPU build" that BASELINE.json's >=10x target refers to.  Prints the timings as one JSON line (run with -s)."""
import json
import os

import pytest
import torch

from conftest import default_weights
from oracle import pvraft_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(os.environ.get('PVRAFT_REF_GPU', '0') != '1', reason='baseline timing run: set PVRAFT_REF_GPU=1')
def test_time_reference_formulation_on_gpu():
    dev = torch.device('cuda:0')
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    W = {k: v.to(dev) for k, v in default_weights().items()}
    out = {}
    for name, b, iters in (('config2_B2_iters8', 2, 8), ('bench_B8_iters32', 8, 32)):
        pc1, pc2 = [t.to(dev) for t in O.synthetic_clouds(b, 8192, 1234)]
        with torch.no_grad():
            for _ in range(2):                                   # warm-up
                O.rsf_forward(W, pc1, pc2, 2, 3, 0.25, 512)
            torch.cuda.synchronize()
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            li = O.prepare(W, pc1, pc2, 512)
            e[1].record()
            O.raft_loop(W, li, pc1, iters, 3, 0.25)
            e[2].record()
            torch.cuda.synchronize()
        t_prep, t_loop = e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])
        out[name] = {'B': b, 'N': 8192, 'iters': iters, 'prepare_ms': t_prep, 'loop_ms': t_loop,
                     'sample_iters_per_s_end_to_end': b * iters / ((t_prep + t_loop) * 1e-3),
                     'sample_iters_per_s_loop_only': b * iters / (t_loop * 1e-3)}
        del li
        torch.cuda.empty_cache()
    print(json.dumps(out))
