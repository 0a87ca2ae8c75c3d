"""Scan sequences without a GPU: the propagation entry point is declared, bound, and refuses bad arguments before any launch;
ops.flow_propagate, forward(..., flow_init=) and SceneFlowStream refuse bad shapes, a bad k and CPU tensors before launching
anything."""
import os
import re
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def model(refine=False):
    from pvraft_b200 import RSF, RSF_refine
    return (RSF_refine if refine else RSF)(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=64))


def test_header_declares_and_lib_binds_the_entry_point():
    from pvraft_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    assert re.search(r'PVRAFT_API int pvraft_flow_propagate_fwd\(', header)
    assert 'pvraft_flow_propagate_fwd_det_workspace_bytes' not in header     # nothing to make deterministic
    assert 'pvraft_flow_propagate_fwd' in _lib.EXPORTS
    assert len(_lib._SIGNATURES['pvraft_flow_propagate_fwd'][1]) == 10


def test_entry_point_refuses_bad_arguments():
    """Null pointers, B, M or N < 1 and k outside 1..min(8, M) return PVRAFT_ERR_BAD_ARG (-1) before any launch."""
    from pvraft_b200 import _lib
    lib = _lib.lib()
    p = 256   # never dereferenced: every call below fails its argument check

    def fwd(xyz_prev=p, flow_prev=p, xyz=p, B=2, M=64, N=64, k=3, flow_out=p, idx_out=None):
        return lib.pvraft_flow_propagate_fwd(xyz_prev, flow_prev, xyz, B, M, N, k, flow_out, idx_out, None)

    for kw in (dict(xyz_prev=None), dict(flow_prev=None), dict(xyz=None), dict(flow_out=None), dict(B=0), dict(B=-1), dict(M=0),
               dict(N=0), dict(N=-3), dict(k=0), dict(k=9), dict(k=-1), dict(M=4, k=5), dict(M=1, k=2), dict(idx_out=p, k=0)):
        assert fwd(**kw) == -1, kw
        assert b'flow_propagate_fwd' in lib.pvraft_last_error_string()


@pytest.mark.parametrize('case', ['dims', 'channels', 'flow_shape', 'batch', 'empty', 'dtype'])
def test_flow_propagate_bad_shapes_raise_before_any_launch(case):
    from pvraft_b200 import ops
    a, f, q = torch.rand(2, 50, 3), torch.rand(2, 50, 3), torch.rand(2, 70, 3)
    if case == 'dims':
        a = a[0]
    elif case == 'channels':
        q = torch.rand(2, 70, 4)
    elif case == 'flow_shape':
        f = f[:, :49]
    elif case == 'batch':
        q = q[:1]
    elif case == 'empty':
        a, f = a[:, :0], f[:, :0]
    else:
        f = f.double()
    n0 = ops.launch_count
    with pytest.raises(ValueError):
        ops.flow_propagate(a, f, q)
    assert ops.launch_count == n0


@pytest.mark.parametrize('k', [0, 9, -1, 1.5, True, 51])
def test_flow_propagate_bad_k_raises(k):
    from pvraft_b200 import ops
    n0 = ops.launch_count
    with pytest.raises(ValueError):
        ops.flow_propagate(torch.rand(2, 50, 3), torch.rand(2, 50, 3), torch.rand(2, 70, 3), k=k)
    assert ops.launch_count == n0


def test_cpu_tensors_raise():
    from pvraft_b200 import SceneFlowStream, ops
    from pvraft_b200._lib import PvraftError
    with pytest.raises(PvraftError):
        ops.flow_propagate(torch.rand(2, 50, 3), torch.rand(2, 50, 3), torch.rand(2, 70, 3))
    m = model()
    p = [torch.rand(2, 64, 3), torch.rand(2, 80, 3)]
    with pytest.raises(PvraftError):
        m(p, 2, flow_init=torch.zeros(2, 64, 3))
    with pytest.raises(PvraftError):
        SceneFlowStream(m, 2).step(p[0])


@pytest.mark.parametrize('refine', [False, True])
@pytest.mark.parametrize('shape', [(2, 80, 3), (1, 64, 3), (2, 64, 2), (2, 64), (128, 3)])
def test_bad_flow_init_shape_raises(refine, shape):
    """flow_init must be shaped like the first cloud [B,N1,3]."""
    from pvraft_b200 import ops
    m = model(refine)
    p = [torch.rand(2, 64, 3), torch.rand(2, 80, 3)]
    n0 = ops.launch_count
    with pytest.raises(ValueError):
        m(p, 2, flow_init=torch.zeros(shape))
    with pytest.raises(ValueError):
        m(p, 2, flow_init=torch.zeros(2, 64, 3, dtype=torch.int32))
    with pytest.raises(ValueError):
        m(p, 2, flow_init=[[0.0, 0.0, 0.0]])
    assert ops.launch_count == n0


def test_stream_arguments():
    from pvraft_b200 import SceneFlowStream
    m = model()
    for k in (0, 9, -1, 2.0, True):
        with pytest.raises(ValueError):
            SceneFlowStream(m, 4, k=k)
    for iters in (0, -2, 1.5):
        with pytest.raises(ValueError):
            SceneFlowStream(m, iters)
    with pytest.raises(TypeError):
        SceneFlowStream(torch.nn.DataParallel(m), 4)
    with pytest.raises(TypeError):
        SceneFlowStream(torch.nn.Linear(3, 3), 4)
    st = SceneFlowStream(m, 4, warm_start=False, k=8)
    assert (st.num_iters, st.warm_start, st.k) == (4, False, 8)
    for bad in (torch.rand(64, 3), torch.rand(2, 64, 4), torch.rand(2, 31, 3)):
        with pytest.raises(ValueError):
            st.step(bad)
    assert st._scan is None
