"""CPU tests of ops.corr_plan: how the truncated correlation is built for a cloud size (one dense matrix up to 49152 points,
column windows and row blocks beyond)."""
import pytest

from pvraft_b200 import ops


def check_plan(plan, n, k, window=ops.CORR_ROW_MAX):
    pos = 0
    for c0, w in plan.windows:                    # the windows tile [0, N) in order, 128-aligned, each in [K, window]
        assert c0 == pos and c0 % 128 == 0
        assert k <= w <= window and w <= plan.ld
        pos += w
    assert pos == n
    assert plan.ld % 128 == 0
    pos = 0
    rows = max(r for _, r in plan.row_blocks)
    assert rows % 128 == 0 or len(plan.row_blocks) == 1
    for r0, r in plan.row_blocks:                 # the row blocks tile [0, N) in order, 128-aligned
        assert r0 == pos and r0 % 128 == 0 and 0 < r <= rows
        pos += r
    assert pos == n


@pytest.mark.parametrize('b', [1, 8])
@pytest.mark.parametrize('k', [32, 512, 1024])
@pytest.mark.parametrize('n', [49153, 65536, 100000, 131072, 262143, 500000, 1000000])
def test_windowed_plan_tiles_the_cloud_and_keeps_the_byte_cap(b, n, k):
    plan = ops.corr_plan(b, n, n, 128, k)
    assert not plan.dense
    assert len(plan.windows) == -(-n // ops.CORR_ROW_MAX)
    check_plan(plan, n, k)
    rows = max(r for _, r in plan.row_blocks)
    assert plan.slab_bytes == rows * (4 * plan.ld + 8 * len(plan.windows) * k)
    assert plan.slab_bytes <= ops.CORR_SLAB_CAP
    assert rows >= 1024                           # GEMM launches of many tiles, not a sliver per launch


@pytest.mark.parametrize('n', [128, 1000, 8192, 20000, 49152])
def test_up_to_49152_points_the_plan_is_the_dense_build(n):
    plan = ops.corr_plan(2, n, n, 128, 64)
    assert plan.dense
    assert plan.windows == ((0, n),) and plan.row_blocks == ((0, n),)
    assert plan.slab_bytes == 4 * 2 * plan.ld * plan.ld      # the [B,N,N] matrix of 128-padded rows


@pytest.mark.parametrize('n, k, window', [(8192, 512, 3072), (20000, 512, 8192), (20001, 64, 1024), (49152, 512, 16384),
                                          (49152, 512, 2048), (1000, 32, 128)])
def test_forced_small_windows(n, k, window):
    """The window widths the GPU tests force: several windows, a ragged last one where N allows it."""
    plan = ops.corr_plan(2, n, n, 128, k, window=window, cap=64 << 20)
    assert not plan.dense and len(plan.windows) >= 3
    check_plan(plan, n, k, window)
    assert plan.slab_bytes <= 64 << 20


def test_too_many_candidates_per_row_are_refused():
    limit = ops.CORR_ROW_MAX // 1024 * ops.CORR_ROW_MAX       # 48 windows x 1024 candidates = 49152
    plan = ops.corr_plan(1, limit, limit, 128, 1024)
    assert len(plan.windows) * 1024 == ops.CORR_ROW_MAX
    with pytest.raises(ValueError, match='candidates per row'):
        ops.corr_plan(1, limit + 1, limit + 1, 128, 1024)
    with pytest.raises(ValueError, match='candidates per row'):
        ops.corr_plan(1, 4 * limit, 4 * limit, 128, 512)
    assert not ops.corr_plan(1, 2 * limit, 2 * limit, 128, 512).dense


def test_bad_arguments_are_refused():
    with pytest.raises(ValueError):
        ops.corr_plan(1, 65536, 65536, 128, 0)
    with pytest.raises(ValueError):
        ops.corr_plan(1, 1000, 1000, 128, 64, window=1000)       # not a multiple of 128
    with pytest.raises(ValueError):
        ops.corr_plan(1, 200000, 200000, 128, 64, window=65536)  # wider than a row the top-K kernels stage
    with pytest.raises(ValueError, match='truncate_k'):
        ops.corr_plan(1, 1000, 1000, 128, 2000, window=512)
