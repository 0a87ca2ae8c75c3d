"""CPU-only checks of the table gradient of the correlation lookup (pvraft_corr_lookup_xyz_bwd): argument errors are reported
before anything is launched, and the deterministic workspace has the documented size, B * M * 3 fixed-point slots."""
import pytest


@pytest.fixture(scope='module')
def lib():
    from pvraft_b200 import _lib
    return _lib.lib()


def test_null_pointers_and_bad_shapes_are_rejected(lib):
    p = 16   # any non-null address: the checks run before a launch, so it is never dereferenced
    for ptrs in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
        idx, slot, g, d = ptrs
        assert lib.pvraft_corr_lookup_xyz_bwd(idx, slot, g, 2, 64, 96, 64, d, None, None) == -1
        assert b'null pointer' in lib.pvraft_last_error_string()
    for b, n, m, k in ((0, 64, 96, 64), (2, 0, 96, 64), (2, 64, 0, 64), (2, 64, 96, 31), (2, 64, 96, 97), (-1, 64, 96, 64)):
        assert lib.pvraft_corr_lookup_xyz_bwd(p, p, p, b, n, m, k, p, None, None) == -1, (b, n, m, k)
        assert b'bad shape' in lib.pvraft_last_error_string()
        assert lib.pvraft_corr_lookup_xyz_bwd(p, p, p, b, n, m, k, p, p, None) == -1   # the deterministic form checks the same


def test_workspace_size_formula(lib):
    for b, m in ((1, 32), (2, 8192), (3, 12345), (8, 65536)):
        assert lib.pvraft_corr_lookup_xyz_bwd_det_workspace_bytes(b, m) == b * m * 3 * 24
