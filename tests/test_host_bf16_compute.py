"""The 'bf16-compute' precision mode without a GPU: the mode switch, the scope that carries it into the RAFT loop, and the
C ABI's rule that a tensor-core layer gets its weights in exactly one operand format."""
import ctypes
import types

import pytest
import torch


def model(refine=False):
    from pvraft_b200 import RSF, RSF_refine
    return (RSF_refine if refine else RSF)(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=64))


@pytest.mark.parametrize('refine', [False, True], ids=['RSF', 'RSF_refine'])
def test_set_precision_accepts_bf16_compute_and_rejects_unknown_modes(refine):
    m = model(refine)
    assert not m.bf16_compute and m.corr_block.state_dtype == torch.float32
    assert m.set_precision('bf16-compute') is m
    assert m.bf16_compute and m.corr_block.state_dtype == torch.bfloat16
    assert 'bf16_compute' in m.__dict__                  # nn.DataParallel replicas copy __dict__
    m.set_precision('bf16')
    assert not m.bf16_compute and m.corr_block.state_dtype == torch.bfloat16
    m.set_precision('bf16-compute').set_precision('fp32')
    assert not m.bf16_compute and m.corr_block.state_dtype == torch.float32
    for bad in ('fp16', 'bf16_compute', 'BF16', None):
        with pytest.raises(ValueError):
            m.set_precision(bad)
    assert not m.bf16_compute and m.corr_block.state_dtype == torch.float32


def test_set_precision_resets_the_graphs():
    m = model()
    m.__dict__['_graphs'] = {'k': None}
    m.set_precision('bf16-compute')
    assert '_graphs' not in m.__dict__


def test_bf16_compute_scope_nests_and_restores():
    from pvraft_b200 import ops
    state = lambda: bool(getattr(ops._TLS, 'bf16', False))   # noqa: E731
    assert not state()
    with ops.bf16_compute():
        assert state()
        with ops.bf16_compute(False):
            assert not state()
        assert state()
    assert not state()


def test_one_weight_format_per_launch():
    """w_bf16 together with w_hi / w_lo, or a chain whose layers mix the formats, is rejected before any launch."""
    from pvraft_b200 import _lib, ops
    lib = _lib.lib()
    a = ops.pack.TcLinearArgs(in_=[16], in_channels=[32], out=16, n_pad=16, cout=16, B=1, N=128, w_hi=16, w_lo=16, w_bf16=16)
    assert lib.pvraft_tc_linear_fwd(ctypes.byref(a), None, None) == -1
    assert b'w_bf16' in lib.pvraft_last_error_string()
    c = ops.pack.UpdateChainArgs(**{f: 16 for f in ('y1', 'y1_stats', 'gn_gamma', 'gn_beta', 'kfeat', 'cflow', 'flow', 'net', 'inp',
                                                        'b_cc', 'b_m', 'b_z', 'b_r', 'b_q', 'p_out')},
                 net_out=32, B=1, N=128, hidden=64, context=64, y1_channels=128, w_bf16=[16] * 5)
    c.w_hi[3], c.w_lo[3] = 16, 16
    assert lib.pvraft_update_chain_fwd(ctypes.byref(c), None) == -1
    assert b'layer 3' in lib.pvraft_last_error_string()
    c.w_hi[3] = c.w_lo[3] = None
    c.w_bf16[4] = None
    assert lib.pvraft_update_chain_fwd(ctypes.byref(c), None) == -1
    assert b'layer 4' in lib.pvraft_last_error_string()
