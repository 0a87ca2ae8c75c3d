"""The uniform-grid searches without a GPU: the C entry points are declared and bound, report their workspace sizes, and
refuse bad arguments before any launch; the Python wrappers refuse CPU tensors and bad K before launching anything, and pick
the grid form from the size of the searched cloud."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = {'pvraft_grid_index_workspace_bytes': 2, 'pvraft_grid_index_fwd': 6, 'pvraft_chamfer_grid_workspace_bytes': 4,
         'pvraft_chamfer_grid_fwd': 12, 'pvraft_laplacian_grid_fwd': 16, 'pvraft_flow_propagate_grid_fwd': 11}
P = 256   # never dereferenced: every call below fails its argument check
BAD, UNSUPPORTED = -1, -2


def test_header_declares_and_lib_binds_the_entry_points():
    from pvraft_b200 import _lib
    with open(os.path.join(ROOT, 'include', 'pvraft_b200.h')) as f:
        header = f.read()
    for name, nargs in NAMES.items():
        assert re.search(r'PVRAFT_API int(64_t)? ' + name + r'\(', header), name
        assert len(_lib._SIGNATURES[name][1]) == nargs, name
    assert _lib.PvraftError   # the status codes below are the header's
    assert re.search(r'PVRAFT_ERR_BAD_ARG\s*=\s*-1', header) and re.search(r'PVRAFT_ERR_UNSUPPORTED\s*=\s*-2', header)


def index_bytes(s, n):
    """The documented layout: pts, ids, key, rank, cell_start (max(32768, n) + 1 per sample), grid parameters (56 B) and two
    16-byte scratch rows per sample, every block rounded up to 16 bytes."""
    def a16(x):
        return (x + 15) // 16 * 16
    cells = max(32768, n)
    return a16(16 * s * n) + 3 * a16(4 * s * n) + a16(4 * s * (cells + 1)) + a16(56 * s) + 2 * a16(16 * s)


def test_workspace_sizes():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    for s, n in ((1, 1), (2, 1000), (3, 16385), (8, 131072), (1, 1000000)):
        assert lib.pvraft_grid_index_workspace_bytes(s, n) == index_bytes(s, n), (s, n)
    assert lib.pvraft_chamfer_grid_workspace_bytes(6, 2, 20000, 5000) == index_bytes(2, 5000) + index_bytes(6, 20000)
    for bad in ((0, 10), (2, 0), (-1, 5)):
        assert lib.pvraft_grid_index_workspace_bytes(*bad) == 0
    assert lib.pvraft_chamfer_grid_workspace_bytes(0, 1, 10, 10) == 0 and lib.pvraft_chamfer_grid_workspace_bytes(2, 2, 10, 0) == 0
    # the kNN graph keeps its shared-memory layout up to 16 384 points and uses the counting-sort index beyond
    assert lib.pvraft_knn_workspace_bytes(2, 16385) == index_bytes(2, 16385)
    assert lib.pvraft_knn_workspace_bytes(2, 16384) == 2 * 16384 * 24 + 2 * 32769 * 4 + 2 * 56 + 512
    assert lib.pvraft_knn_workspace_bytes(0, 20000) == 0


def test_grid_index_refuses_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()
    for kw, code in ((dict(xyz=None), BAD), (dict(ws=None), BAD), (dict(S=0), BAD), (dict(N=0), BAD), (dict(ws=P + 8), BAD),
                     (dict(S=65536), UNSUPPORTED)):
        a = dict(xyz=P, S=2, N=100, ws=P) | kw
        assert lib.pvraft_grid_index_fwd(a['xyz'], None, a['S'], a['N'], a['ws'], None) == code, kw
        assert b'grid_index' in lib.pvraft_last_error_string()


def test_chamfer_grid_refuses_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def call(a=P, b=P, S=4, B=2, N=100, M=70, ab=P, ba=P, acc=P, ws=P):
        return lib.pvraft_chamfer_grid_fwd(a, b, S, B, N, M, ab, ba, acc, ws, None, None)

    for kw in (dict(a=None), dict(b=None), dict(ab=None), dict(ba=None), dict(acc=None), dict(ws=None), dict(S=3), dict(S=0),
               dict(B=0), dict(N=0), dict(M=0)):
        assert call(**kw) == BAD, kw
        assert b'chamfer_grid_fwd' in lib.pvraft_last_error_string()
    assert call(S=65536, B=1) == UNSUPPORTED


def test_laplacian_grid_refuses_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def call(w=P, p2=P, l2=P, g1=P, S=4, B=2, N=100, M=70, k_lap=10, k_int=5, idx=P, res=P, acc=P, ws=P):
        return lib.pvraft_laplacian_grid_fwd(w, p2, l2, g1, S, B, N, M, k_lap, k_int, idx, res, acc, ws, None, None)

    for kw in (dict(w=None), dict(p2=None), dict(l2=None), dict(g1=None), dict(idx=None), dict(res=None), dict(acc=None),
               dict(ws=None), dict(S=3), dict(S=0), dict(B=0), dict(N=0), dict(M=0), dict(k_lap=1), dict(k_lap=33), dict(N=8, k_lap=9),
               dict(k_int=0), dict(k_int=9), dict(M=3, k_int=4)):
        assert call(**kw) == BAD, kw
        assert b'laplacian_grid_fwd' in lib.pvraft_last_error_string()
    assert call(S=65536, B=1) == UNSUPPORTED


def test_flow_propagate_grid_refuses_bad_arguments():
    from pvraft_b200 import _lib
    lib = _lib.lib()

    def call(xp=P, fp=P, x=P, B=2, M=70, N=100, k=3, out=P, ws=P):
        return lib.pvraft_flow_propagate_grid_fwd(xp, fp, x, B, M, N, k, out, None, ws, None)

    for kw in (dict(xp=None), dict(fp=None), dict(x=None), dict(out=None), dict(ws=None), dict(B=0), dict(M=0), dict(N=0),
               dict(k=0), dict(k=9), dict(M=2, k=3)):
        assert call(**kw) == BAD, kw
        assert b'flow_propagate_grid_fwd' in lib.pvraft_last_error_string()
    assert call(B=65536) == UNSUPPORTED


def test_threshold_choice():
    from pvraft_b200 import ops
    assert set(ops.GRID_SEARCH_MIN_POINTS) == {'chamfer', 'laplacian', 'flow_propagate'}
    for op, t in ops.GRID_SEARCH_MIN_POINTS.items():
        assert isinstance(t, int) and t >= 1
        assert ops.use_grid_search(op, t) and not ops.use_grid_search(op, t - 1)
        assert ops.use_grid_search(op, 1, True) and not ops.use_grid_search(op, 10 ** 7, False)
    with pytest.raises(KeyError):
        ops.use_grid_search('knn', 10 ** 6)


@pytest.mark.parametrize('op', ['chamfer', 'laplacian', 'flow_propagate'])
def test_each_op_searches_on_the_grid_from_the_threshold(op, monkeypatch):
    """Which entry point each op calls, on either side of the threshold and under the forcing keyword: recorded by a stand-in
    library that launches nothing (CPU tensors pass the device check of this stand-in only)."""
    from pvraft_b200 import ops
    calls = []

    class Lib:
        def __getattr__(self, name):
            def fn(*args):
                calls.append(name)
                return 64 if name.endswith('_bytes') else 0
            return fn

    monkeypatch.setattr(ops, 'lib', lambda: Lib())
    monkeypatch.setattr(ops, '_p', lambda t, dtype=None: None)
    monkeypatch.setattr(ops, '_stream', lambda: None)
    monkeypatch.setattr(ops, 'GRID_SEARCH_MIN_POINTS', {'chamfer': 100, 'laplacian': 100, 'flow_propagate': 100})
    monkeypatch.setattr(torch.Tensor, 'is_cuda', property(lambda self: True))

    def run(n, m, use_grid=None):
        calls.clear()
        a, b = torch.zeros(2, n, 3), torch.zeros(2, m, 3)
        if op == 'chamfer':
            ops.chamfer(a, b, use_grid=use_grid)
        elif op == 'laplacian':
            ops.laplacian(a, b, torch.zeros(2, m, 3), torch.zeros(2, n, 10, dtype=torch.int32), 5, use_grid=use_grid)
        else:
            ops.flow_propagate(b, torch.zeros(2, m, 3), a, 3, use_grid=use_grid)
        return [c for c in calls if c.endswith('_fwd')]

    grid, brute = f'pvraft_{op}_grid_fwd', f'pvraft_{op}_fwd'
    assert run(150, 100) == [grid] and run(150, 99) == ([grid] if op == 'chamfer' else [brute])
    assert run(50, 99) == [brute]
    assert run(50, 60, use_grid=True) == [grid] and run(500, 600, use_grid=False) == [brute]


def test_wrappers_refuse_cpu_tensors_and_bad_k():
    from pvraft_b200 import _lib, ops
    a, b = torch.zeros(2, 100, 3), torch.zeros(2, 70, 3)
    with pytest.raises(_lib.PvraftError):
        ops.chamfer(a, b, use_grid=True)
    with pytest.raises(_lib.PvraftError):
        ops.flow_propagate(b, b, a, 3, use_grid=True)
    with pytest.raises(_lib.PvraftError):
        ops.laplacian(a, b, b, torch.zeros(2, 100, 10, dtype=torch.int32), 5, use_grid=True)
    for k in (0, 9, 2.0, True):
        with pytest.raises(ValueError):
            ops.flow_propagate(b, b, a, k, use_grid=True)
        with pytest.raises(ValueError):
            ops.laplacian(a, b, b, torch.zeros(2, 100, 10, dtype=torch.int32), k, use_grid=True)
