"""The 'bf16-mixed' training mode without a GPU: the mode switch, the rule that picks which loop layers run on bf16 wgmma,
and the C entry points of the tensor-core weight gradient (declared, bound, and refusing bad arguments before any launch)."""
import os
import re
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def model(refine=False):
    from pvraft_b200 import RSF, RSF_refine
    return (RSF_refine if refine else RSF)(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=64))


@pytest.mark.parametrize('refine', [False, True], ids=['RSF', 'RSF_refine'])
def test_set_precision_bf16_mixed(refine):
    m = model(refine)
    m.__dict__['_graphs'] = {'k': None}
    assert m.set_precision('bf16-mixed') is m
    assert m.bf16_compute and m.corr_block.state_dtype == torch.float32
    assert 'bf16_compute' in m.__dict__                  # nn.DataParallel replicas copy __dict__
    assert '_graphs' not in m.__dict__                   # switching modes resets the graphs
    m.set_precision('bf16-compute')
    assert m.bf16_compute and m.corr_block.state_dtype == torch.bfloat16
    m.set_precision('bf16-mixed').set_precision('fp32')
    assert not m.bf16_compute and m.corr_block.state_dtype == torch.float32
    with pytest.raises(ValueError):
        m.set_precision('bf16_mixed')


# (n_points, cin, cout, want_stats) -> (forward, dx, dW) on bf16 wgmma: the layers of one RAFT iteration at N = 8192, then the
# rule's edges
LAYERS = {
    'corr out_conv[0] (81 -> 128, stats)': ((8192, 81, 128, True), (False, False, False)),
    'corr out_conv[3] (128 -> 64)': ((8192, 128, 64, False), (True, True, True)),
    'knn_out (64 -> 64)': ((8192, 64, 64, False), (True, True, True)),
    'conv_corr (64 -> 64)': ((8192, 64, 64, False), (True, True, True)),
    'conv_flow (3 -> 64)': ((8192, 3, 64, False), (False, False, False)),
    'motion conv (128 -> 61)': ((8192, 128, 61, False), (True, False, False)),
    'GRU [z|r] (192 -> 128)': ((8192, 192, 128, False), (True, True, True)),
    'GRU q (192 -> 64)': ((8192, 192, 64, False), (True, True, True)),
    'flow head conv1 (64 -> 64)': ((8192, 64, 64, False), (True, True, True)),
    'SetConv fc1 point term (64 -> 64)': ((8192, 64, 64, False), (True, True, True)),
    'SetConv fc2 / fc3 (64 -> 64, stats)': ((8192, 64, 64, True), (True, True, True)),
    'flow head out_conv[0] (128 -> 64)': ((8192, 128, 64, False), (True, True, True)),
    'flow head out_conv[2] (64 -> 3)': ((8192, 64, 3, False), (True, False, False)),
    'knn_conv, edge level (4 -> 64, stats)': ((8192 * 32, 4, 64, True), (False, False, False)),
    'N % 128 != 0': ((1000, 64, 64, False), (False, False, False)),
    'cout > 128': ((8192, 64, 192, False), (False, False, False)),
    'stats with cout % 32 != 0': ((8192, 64, 48, True), (False, False, False)),
    'cout = 48 without stats': ((8192, 64, 48, False), (True, False, False)),
    'cin = 256': ((8192, 256, 64, False), (True, True, False)),
}


@pytest.mark.parametrize('name', list(LAYERS))
def test_layer_plan(name):
    from pvraft_b200 import train as T
    shape, want = LAYERS[name]
    assert T.bf16_layer_plan(*shape) == want


def test_header_declares_and_lib_binds_the_weight_gradient():
    from pvraft_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    for name in ('pvraft_tc_wgrad_bf16', 'pvraft_tc_wgrad_bf16_det_workspace_bytes'):
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert name in _lib.EXPORTS
    assert len(_lib._SIGNATURES['pvraft_tc_wgrad_bf16'][1]) == 10


def test_weight_gradient_refuses_bad_arguments():
    """Shapes outside the kernel and null pointers return a status before any launch (no device needed)."""
    from pvraft_b200 import _lib
    lib = _lib.lib()
    assert lib.pvraft_tc_wgrad_bf16_det_workspace_bytes(192, 128) == lib.pvraft_linear_wgrad_det_workspace_bytes(192, 128)
    p = 256
    for cin, cout in ((16, 64), (48, 64), (224, 64), (64, 16), (64, 48), (64, 160)):
        assert lib.pvraft_tc_wgrad_bf16(p, p, 1024, cin, cout, p, 0, None, None, None) == -2, (cin, cout)
        assert b'tc_wgrad_bf16' in lib.pvraft_last_error_string()
    assert lib.pvraft_tc_wgrad_bf16(None, p, 1024, 64, 64, p, 0, None, None, None) == -1
    assert lib.pvraft_tc_wgrad_bf16(p, p, 0, 64, 64, p, 0, None, None, None) == -1
    assert lib.pvraft_tc_wgrad_bf16(p, p, 1024, 64, 64, p, 32, None, None, None) == -1   # dw_ld < cin
