"""The forward-backward consistency term and the bidirectional forward without a GPU: the C entry points are declared, bound,
size their workspaces and refuse bad arguments before any launch; the wrappers, the loss and the model refuse bad k_cons,
w_consistency with a single flow, a warm-started bidirectional forward, truncate_k beyond N1 and CPU tensors first."""
import os
import re
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ('pvraft_flow_consistency_fwd', 'pvraft_flow_consistency_grid_fwd', 'pvraft_flow_consistency_bwd')
P = 256   # never dereferenced: every call below fails its argument check
BAD = -1


def test_header_declares_and_lib_binds_the_entry_points():
    from pvraft_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    for name in NAMES + ('pvraft_flow_consistency_fwd_det_workspace_bytes', 'pvraft_flow_consistency_bwd_det_workspace_bytes'):
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert name in _lib.EXPORTS
    assert [len(_lib._SIGNATURES[n][1]) for n in NAMES] == [17, 18, 17]


def test_workspace_sizes():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    assert lib.pvraft_flow_consistency_fwd_det_workspace_bytes(6) == 6 * 24
    assert lib.pvraft_flow_consistency_bwd_det_workspace_bytes(6, 2, 70) == (2 * 70 * 3 + 6 * 70 * 3) * 24
    assert lib.pvraft_flow_consistency_fwd_det_workspace_bytes(0) == 0
    assert lib.pvraft_flow_consistency_bwd_det_workspace_bytes(6, 2, 0) == 0
    assert lib.pvraft_flow_consistency_bwd_det_workspace_bytes(6, 0, 70) == 0


CASES = (dict(S=3), dict(S=0), dict(B=0), dict(N=0), dict(M=0), dict(k=0), dict(k=9), dict(M=3, k=4))


def test_entry_points_refuse_bad_arguments():
    """Null pointers, S % B, k outside 1..min(8, M), and alpha or beta negative or not finite: PVRAFT_ERR_BAD_ARG."""
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def fwd(w=P, f12=P, p2=P, f21=P, S=4, B=2, N=64, M=70, k=3, alpha=0.01, beta=0.0025, nn=P, res=P, ok=P, acc=P):
        return lib.pvraft_flow_consistency_fwd(w, f12, p2, f21, S, B, N, M, k, alpha, beta, nn, res, ok, acc, None, None)

    def grid(ws=P, **kw):
        a = dict(w=P, f12=P, p2=P, f21=P, S=4, B=2, N=64, M=70, k=3, alpha=0.01, beta=0.0025, nn=P, res=P, ok=P, acc=P)
        a.update(kw)
        return lib.pvraft_flow_consistency_grid_fwd(*a.values(), ws, None, None)

    def bwd(w=P, p2=P, f21=P, nn=P, res=P, g=P, S=4, B=2, N=64, M=70, k=3, d_w=P, d_f12=P, d_p2=P, d_f21=P):
        return lib.pvraft_flow_consistency_bwd(w, p2, f21, nn, res, g, S, B, N, M, k, d_w, d_f12, d_p2, d_f21, None, None)

    for kw in CASES:
        for fn, what in ((fwd, b'flow_consistency_fwd'), (grid, b'flow_consistency_grid_fwd'), (bwd, b'flow_consistency_bwd')):
            assert fn(**kw) == BAD, (what, kw)
            assert what in lib.pvraft_last_error_string()
    for kw in (dict(alpha=-1e-3), dict(beta=-1.0), dict(alpha=float('nan')), dict(beta=float('inf')), dict(alpha=float('inf'))):
        assert fwd(**kw) == BAD, kw
        assert grid(**kw) == BAD, kw
    for name in ('w', 'f12', 'p2', 'f21', 'nn', 'res', 'ok', 'acc'):
        assert fwd(**{name: None}) == BAD, name
        assert grid(**{name: None}) == BAD, name
    assert grid(ws=None) == BAD
    for name in ('w', 'p2', 'f21', 'nn', 'res', 'g', 'd_w', 'd_f12', 'd_f21'):
        assert bwd(**{name: None}) == BAD, name


def test_wrappers_refuse_bad_k_and_cpu_tensors():
    from pvraft_b200 import ops
    from pvraft_b200._lib import PvraftError
    w, p2 = torch.rand(4, 50, 3), torch.rand(2, 40, 3)
    f21 = torch.rand(4, 40, 3)
    for k in (0, 9, 2.0, True):
        with pytest.raises(ValueError):
            ops.flow_consistency(w, w, p2, f21, k, 0.01, 0.0)
    with pytest.raises(ValueError):
        ops.flow_consistency(w, w, p2, torch.rand(2, 40, 3), 3, 0.01, 0.0)   # f21 per prediction
    with pytest.raises(ValueError):
        ops.flow_consistency(w, w, p2, f21, 3, -0.5, 0.0)
    with pytest.raises(PvraftError):
        ops.flow_consistency(w, w, p2, f21, 3, 0.01, 0.0)
    import pvraft_b200
    with pytest.raises(PvraftError):
        pvraft_b200.flow_consistency(p2, p2, p2, p2)


def _batch(n1=64, n2=64):
    return {'sequence': [torch.rand(2, n1, 3), torch.rand(2, n2, 3)]}


def test_loss_refuses_bad_k_cons_and_single_flow_consistency():
    from pvraft_b200.loss import self_supervised_loss, sequence_self_supervised_loss
    batch = _batch()
    f = torch.rand(2, 64, 3)
    for k_cons in (0, 9, 3.0, False):
        with pytest.raises(ValueError, match='k_cons'):
            self_supervised_loss((f, f), batch, w_consistency=0.3, k_cons=k_cons)
        with pytest.raises(ValueError, match='k_cons'):
            sequence_self_supervised_loss(([f], [f]), batch, w_consistency=0.3, k_cons=k_cons)
        with pytest.raises(ValueError, match='k_cons'):
            self_supervised_loss(f, batch, k_cons=k_cons)
    with pytest.raises(ValueError, match='w_consistency'):
        self_supervised_loss(f, batch, w_consistency=0.3)
    with pytest.raises(ValueError, match='w_consistency'):
        sequence_self_supervised_loss([f, f], batch, w_consistency=0.3)


def _model(refine=False, k=64):
    from pvraft_b200 import RSF, RSF_refine
    return (RSF_refine if refine else RSF)(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k))


@pytest.mark.parametrize('refine', [False, True])
def test_model_refuses_flow_init_and_truncate_k_beyond_n1(refine):
    from pvraft_b200._lib import PvraftError
    m = _model(refine, k=64)
    p = [torch.rand(1, 48, 3), torch.rand(1, 96, 3)]
    with pytest.raises(ValueError, match='flow_init'):
        m(p, 2, flow_init=torch.zeros(1, 48, 3), bidirectional=True)
    with pytest.raises(ValueError, match='truncate_k'):
        m(p, 2, bidirectional=True)              # truncate_k = 64 <= N2 = 96 but > N1 = 48
    with torch.no_grad(), pytest.raises(ValueError, match='truncate_k'):
        m(p, 2, bidirectional=True)
    m.set_precision('bf16')
    with pytest.raises(ValueError, match='65536'):
        m([torch.rand(1, 96, 3), torch.rand(1, 70000, 3)], 2, bidirectional=True)
    with pytest.raises(PvraftError):
        m([torch.rand(1, 96, 3), torch.rand(1, 96, 3)], 2, bidirectional=True)   # CPU tensors
