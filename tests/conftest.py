import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """-> (arrays dict of torch tensors / numpy scalars, weights dict keyed like state_dict)."""
    z = np.load(os.path.join(GOLDEN, name), allow_pickle=False)
    arrays, weights = {}, {}
    for k in z.files:
        v = z[k]
        if k.startswith('w/'):
            weights[k[2:]] = torch.from_numpy(v.copy())
        elif v.dtype.kind in 'fiub' and v.ndim > 0:
            arrays[k] = torch.from_numpy(v.copy())
        else:
            arrays[k] = v
    return arrays, weights


def default_weights(refine=False, seed=0, args=None):
    """Seeded default-init weights with the reference's construction order (RSF.__init__,
    model/RAFTSceneFlow.py:10-20): built from the product modules, which are asserted elsewhere to
    consume the RNG identically to the reference."""
    import types
    from pvraft_b200 import RSF, RSF_refine
    args = args or types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=512)
    torch.manual_seed(seed)
    m = (RSF_refine if refine else RSF)(args)
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def rel_err(a, b):
    a = a.double()
    b = b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.fixture(autouse=True)
def _poison_uninitialised(monkeypatch):
    """PVRAFT_POISON=1: every torch.empty/empty_like/new_empty allocation is filled with NaN (floats) or a huge
    value (ints), so that any kernel reading memory it was supposed to have been given initialised shows up as a
    hard failure instead of a once-in-a-while mismatch."""
    if os.environ.get('PVRAFT_POISON') != '1':
        yield
        return
    real_empty, real_like = torch.empty, torch.empty_like

    def fill(t):
        if t.is_floating_point():
            t.fill_(float('nan'))
        elif t.dtype != torch.bool:
            t.fill_(torch.iinfo(t.dtype).max // 2)
        return t

    monkeypatch.setattr(torch, 'empty', lambda *a, **k: fill(real_empty(*a, **k)))
    monkeypatch.setattr(torch, 'empty_like', lambda *a, **k: fill(real_like(*a, **k)))
    real_new = torch.Tensor.new_empty
    monkeypatch.setattr(torch.Tensor, 'new_empty', lambda self, *a, **k: fill(real_new(self, *a, **k)))
    yield
