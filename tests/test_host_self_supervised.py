"""The self-supervised losses without a GPU: the C entry points are declared, bound, and refuse bad arguments before any
launch; the Python wrappers refuse CPU tensors, a bad neighbour count and mismatched batches before launching anything."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ('pvraft_chamfer_fwd', 'pvraft_chamfer_bwd', 'pvraft_flow_smooth_fwd', 'pvraft_flow_smooth_bwd')


def test_header_declares_and_lib_binds_the_entry_points():
    from pvraft_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    for name in NAMES + tuple(n + '_det_workspace_bytes' for n in NAMES):
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert name in _lib.EXPORTS
    assert [len(_lib._SIGNATURES[n][1]) for n in NAMES] == [11, 13, 9, 10]


def test_workspace_sizes():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    assert lib.pvraft_chamfer_fwd_det_workspace_bytes(6) == 6 * 2 * 24
    assert lib.pvraft_chamfer_bwd_det_workspace_bytes(6, 2, 100, 70) == (6 * 100 * 3 + 2 * 70 * 3) * 24
    assert lib.pvraft_flow_smooth_fwd_det_workspace_bytes(6) == 6 * 24
    assert lib.pvraft_flow_smooth_bwd_det_workspace_bytes(6, 100) == 6 * 100 * 3 * 24


def test_entry_points_refuse_bad_arguments():
    """Null pointers, S % B != 0, N or M < 1 and k outside 1..32 return PVRAFT_ERR_BAD_ARG (-1) before any launch."""
    from pvraft_b200 import _lib
    lib = _lib.lib()
    p = 256   # never dereferenced: every call below fails its argument check
    bad = -1

    def fwd(a=p, b=p, S=4, B=2, N=64, M=64, nn_ab=p, nn_ba=p, acc=p):
        return lib.pvraft_chamfer_fwd(a, b, S, B, N, M, nn_ab, nn_ba, acc, None, None)

    for kw in (dict(a=None), dict(b=None), dict(nn_ab=None), dict(nn_ba=None), dict(acc=None), dict(S=3), dict(S=0), dict(B=0),
               dict(N=0), dict(M=0), dict(N=-5)):
        assert fwd(**kw) == bad, kw
        assert b'chamfer_fwd' in lib.pvraft_last_error_string()

    def bwd(a=p, b=p, nn_ab=p, nn_ba=p, g=p, S=4, B=2, N=64, M=64, d_a=p):
        return lib.pvraft_chamfer_bwd(a, b, nn_ab, nn_ba, g, S, B, N, M, d_a, None, None, None)

    for kw in (dict(a=None), dict(b=None), dict(nn_ab=None), dict(nn_ba=None), dict(g=None), dict(d_a=None), dict(S=5), dict(B=0),
               dict(N=0), dict(M=0)):
        assert bwd(**kw) == bad, kw
        assert b'chamfer_bwd' in lib.pvraft_last_error_string()

    def sfwd(f=p, nbr=p, S=4, B=2, N=64, k=9, acc=p):
        return lib.pvraft_flow_smooth_fwd(f, nbr, S, B, N, k, acc, None, None)

    def sbwd(f=p, nbr=p, g=p, S=4, B=2, N=64, k=9, d_f=p):
        return lib.pvraft_flow_smooth_bwd(f, nbr, g, S, B, N, k, d_f, None, None)

    for kw in (dict(f=None), dict(nbr=None), dict(S=3), dict(B=0), dict(N=0), dict(k=0), dict(k=33), dict(k=-1)):
        assert sfwd(**kw) == bad, kw
        assert sbwd(**kw) == bad, kw
    assert sfwd(acc=None) == bad and sbwd(g=None) == bad and sbwd(d_f=None) == bad


def test_cpu_tensors_raise():
    from pvraft_b200 import ops
    from pvraft_b200._lib import PvraftError
    from pvraft_b200.loss import self_supervised_loss, sequence_self_supervised_loss
    p1, p2 = torch.rand(2, 64, 3), torch.rand(2, 80, 3)
    f = torch.zeros(2, 64, 3)
    batch = {'sequence': [p1, p2]}
    with pytest.raises(PvraftError):
        self_supervised_loss(f, batch)
    with pytest.raises(PvraftError):
        sequence_self_supervised_loss([f, f], batch)
    with pytest.raises(PvraftError):
        ops.chamfer(p1, p2)
    with pytest.raises(PvraftError):
        ops.flow_smooth(f, torch.zeros(2, 64, 9, dtype=torch.int32))


@pytest.mark.parametrize('k', [0, 33, -1])
def test_bad_k_raises_before_any_launch(k):
    from pvraft_b200 import ops
    from pvraft_b200.loss import sequence_self_supervised_loss
    n0 = ops.launch_count
    batch = {'sequence': [torch.rand(2, 64, 3), torch.rand(2, 64, 3)]}
    with pytest.raises(ValueError):
        sequence_self_supervised_loss([torch.zeros(2, 64, 3)], batch, k=k)
    with pytest.raises(ValueError):
        ops.flow_smooth(torch.zeros(2, 64, 3), torch.zeros(2, 64, max(k, 0), dtype=torch.int32))
    assert ops.launch_count == n0


@pytest.mark.parametrize('case', ['clouds', 'flow', 'samples'])
def test_mismatched_batches_raise_before_any_launch(case):
    from pvraft_b200 import ops
    from pvraft_b200.loss import self_supervised_loss
    n0 = ops.launch_count
    p1, p2, f = torch.rand(2, 64, 3), torch.rand(2, 70, 3), torch.zeros(2, 64, 3)
    with pytest.raises(ValueError):
        if case == 'clouds':
            self_supervised_loss(f, {'sequence': [p1, p2[:1]]})
        elif case == 'flow':
            self_supervised_loss(f[:, :60], {'sequence': [p1, p2]})
        else:
            ops.chamfer(torch.rand(3, 64, 3), p2)
    with pytest.raises(ValueError):
        ops.flow_smooth(torch.zeros(3, 64, 3), torch.zeros(2, 64, 9, dtype=torch.int32))
    assert ops.launch_count == n0
