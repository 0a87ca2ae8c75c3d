"""The Laplacian term of the self-supervised loss without a GPU: the C entry points are declared, bound, and refuse bad
arguments before any launch; the Python wrappers and the loss refuse bad k_lap and k_int, CPU tensors and mismatched batches
before launching anything."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ('pvraft_cloud_laplacian_fwd', 'pvraft_cloud_laplacian_bwd', 'pvraft_laplacian_fwd', 'pvraft_laplacian_bwd')
REDUCING = ('pvraft_cloud_laplacian_bwd', 'pvraft_laplacian_fwd', 'pvraft_laplacian_bwd')
P = 256   # never dereferenced: every call below fails its argument check
BAD = -1


def test_header_declares_and_lib_binds_the_entry_points():
    from pvraft_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    for name in NAMES + tuple(n + '_det_workspace_bytes' for n in REDUCING):
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert name in _lib.EXPORTS
    assert 'pvraft_cloud_laplacian_fwd_det_workspace_bytes' not in _lib.EXPORTS   # writes every output once
    assert [len(_lib._SIGNATURES[n][1]) for n in NAMES] == [7, 8, 15, 18]


def test_workspace_sizes():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    assert lib.pvraft_cloud_laplacian_bwd_det_workspace_bytes(2, 70) == 2 * 70 * 3 * 24
    assert lib.pvraft_laplacian_fwd_det_workspace_bytes(6) == 6 * 24
    assert lib.pvraft_laplacian_bwd_det_workspace_bytes(6, 2, 100, 70) == (6 * 100 * 3 + 2 * 2 * 70 * 3) * 24
    assert lib.pvraft_laplacian_fwd_det_workspace_bytes(0) == 0
    assert lib.pvraft_laplacian_bwd_det_workspace_bytes(6, 2, 100, 0) == 0


def test_cloud_laplacian_entry_points_refuse_bad_arguments():
    """Null pointers, B or N < 1 and k outside 2..min(32, N) return PVRAFT_ERR_BAD_ARG."""
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def fwd(x=P, nbr=P, B=2, N=64, k=10, out=P):
        return lib.pvraft_cloud_laplacian_fwd(x, nbr, B, N, k, out, None)

    def bwd(g_l=P, nbr=P, B=2, N=64, k=10, d_x=P):
        return lib.pvraft_cloud_laplacian_bwd(g_l, nbr, B, N, k, d_x, None, None)

    for kw in (dict(nbr=None), dict(B=0), dict(B=-1), dict(N=0), dict(k=1), dict(k=0), dict(k=33), dict(N=8, k=9)):
        assert fwd(**kw) == BAD, kw
        assert b'cloud_laplacian_fwd' in lib.pvraft_last_error_string()
        assert bwd(**kw) == BAD, kw
        assert b'cloud_laplacian_bwd' in lib.pvraft_last_error_string()
    assert fwd(x=None) == BAD and fwd(out=None) == BAD
    assert bwd(g_l=None) == BAD and bwd(d_x=None) == BAD


TERM_CASES = (dict(S=3), dict(S=0), dict(B=0), dict(N=0), dict(M=0), dict(M=-4), dict(k_lap=1), dict(k_lap=33), dict(N=8, k_lap=9),
              dict(k_int=0), dict(k_int=9), dict(M=3, k_int=4))


def test_laplacian_fwd_refuses_bad_arguments():
    """Null pointers, S % B != 0, N or M < 1, k_lap outside 2..min(32, N) and k_int outside 1..min(8, M)."""
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def fwd(w=P, p2=P, l2=P, g1=P, S=4, B=2, N=64, M=64, k_lap=10, k_int=5, nn_idx=P, res=P, acc=P):
        return lib.pvraft_laplacian_fwd(w, p2, l2, g1, S, B, N, M, k_lap, k_int, nn_idx, res, acc, None, None)

    for kw in TERM_CASES + (dict(w=None), dict(p2=None), dict(l2=None), dict(g1=None), dict(nn_idx=None), dict(res=None), dict(acc=None)):
        assert fwd(**kw) == BAD, kw
        assert b'laplacian_fwd' in lib.pvraft_last_error_string()


def test_laplacian_bwd_refuses_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def bwd(w=P, p2=P, l2=P, g1=P, nn_idx=P, res=P, g=P, S=4, B=2, N=64, M=64, k_lap=10, k_int=5, d_w=P):
        return lib.pvraft_laplacian_bwd(w, p2, l2, g1, nn_idx, res, g, S, B, N, M, k_lap, k_int, d_w, None, None, None, None)

    for kw in TERM_CASES + (dict(w=None), dict(p2=None), dict(l2=None), dict(g1=None), dict(nn_idx=None), dict(res=None), dict(g=None),
                            dict(d_w=None)):
        assert bwd(**kw) == BAD, kw
        assert b'laplacian_bwd' in lib.pvraft_last_error_string()


def _batch(b=2, n=64, m=70):
    return {'sequence': [torch.rand(b, n, 3), torch.rand(b, m, 3)]}


@pytest.mark.parametrize('kw', [dict(k_lap=1), dict(k_lap=33), dict(k_lap=2.0), dict(k_lap=True), dict(k_int=0), dict(k_int=9),
                                dict(k_int=None), dict(k_lap=65), dict(k_int=5, k_lap=20)])
def test_bad_k_raises_before_any_launch(kw):
    from pvraft_b200 import ops
    from pvraft_b200.loss import self_supervised_loss, sequence_self_supervised_loss
    n0 = ops.launch_count
    batch = _batch(n=16, m=18) if kw.get('k_lap') == 20 else _batch()
    f = torch.zeros_like(batch['sequence'][0])
    with pytest.raises(ValueError):
        sequence_self_supervised_loss([f, f], batch, w_laplacian=0.3, **kw)
    with pytest.raises(ValueError):
        self_supervised_loss(f, batch, w_laplacian=0.3, **kw)
    assert ops.launch_count == n0


def test_graph_larger_than_a_cloud_raises_only_when_the_term_is_on():
    """k_lap and k_int beyond a cloud's size are refused for the third term; with w_laplacian = 0 they are never used."""
    from pvraft_b200 import ops
    from pvraft_b200._lib import PvraftError
    from pvraft_b200.loss import self_supervised_loss
    n0 = ops.launch_count
    for b in (_batch(n=64, m=9), _batch(n=9, m=64), _batch(n=64, m=4)):
        f = torch.zeros_like(b['sequence'][0])
        with pytest.raises(ValueError):
            self_supervised_loss(f, b, w_laplacian=0.3)
        with pytest.raises(PvraftError):   # accepted, then refused for the CPU tensors at the first launch
            self_supervised_loss(f, b, w_laplacian=0.0)
    assert ops.launch_count == n0


def test_cpu_tensors_raise():
    from pvraft_b200 import ops
    from pvraft_b200._lib import PvraftError
    from pvraft_b200.loss import LaplacianFn, self_supervised_loss
    n0 = ops.launch_count
    batch = _batch()
    p1, p2 = batch['sequence']
    nbr1, nbr2 = torch.zeros(2, 64, 10, dtype=torch.int32), torch.zeros(2, 70, 10, dtype=torch.int32)
    with pytest.raises(PvraftError):
        self_supervised_loss(torch.zeros_like(p1), batch, w_laplacian=0.3)
    with pytest.raises(PvraftError):
        ops.cloud_laplacian(p2, nbr2)
    with pytest.raises(PvraftError):
        ops.cloud_laplacian_bwd(p2, nbr2, torch.zeros_like(p2))
    with pytest.raises(PvraftError):
        ops.laplacian(p1, p2, p2, nbr1, 5)
    with pytest.raises(PvraftError):
        ops.laplacian_bwd(p1, p2, p2, nbr1, torch.zeros(2, 64, 5, dtype=torch.int32), p1, torch.ones(2))
    with pytest.raises(PvraftError):
        LaplacianFn.apply(p1, p2, nbr1, nbr2, 5)
    assert ops.launch_count == n0


@pytest.mark.parametrize('case', ['clouds', 'samples', 'graph', 'l2', 'k_int', 'nn_idx', 'g'])
def test_mismatched_shapes_raise_before_any_launch(case):
    from pvraft_b200 import ops
    from pvraft_b200.loss import self_supervised_loss
    n0 = ops.launch_count
    p1, p2 = torch.rand(2, 64, 3), torch.rand(2, 70, 3)
    nbr1 = torch.zeros(2, 64, 10, dtype=torch.int32)
    with pytest.raises(ValueError):
        if case == 'clouds':
            self_supervised_loss(torch.zeros_like(p1), {'sequence': [p1, p2[:1]]}, w_laplacian=0.3)
        elif case == 'samples':
            ops.laplacian(torch.rand(3, 64, 3), p2, p2, nbr1, 5)
        elif case == 'graph':
            ops.laplacian(p1, p2, p2, nbr1[:, :60], 5)
        elif case == 'l2':
            ops.laplacian(p1, p2, p2[:, :60], nbr1, 5)
        elif case == 'k_int':
            ops.laplacian(p1, p2, p2, nbr1, 9)
        elif case == 'nn_idx':
            ops.laplacian_bwd(p1, p2, p2, nbr1, torch.zeros(2, 60, 5, dtype=torch.int32), p1, torch.ones(2))
        else:
            ops.laplacian_bwd(p1, p2, p2, nbr1, torch.zeros(2, 64, 5, dtype=torch.int32), p1, torch.ones(3))
    with pytest.raises(ValueError):
        ops.cloud_laplacian(p2, torch.zeros(2, 70, 1, dtype=torch.int32))
    assert ops.launch_count == n0
