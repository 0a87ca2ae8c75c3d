"""Shape rules of pairs of clouds of different sizes, checked on the host before any kernel runs (CPU only)."""
import types

import pytest
import torch


def model(k=64, refine=False):
    from pvraft_b200 import RSF, RSF_refine
    return (RSF_refine if refine else RSF)(types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=k))


def clouds(b1, n1, b2, n2):
    return torch.rand(b1, n1, 3), torch.rand(b2, n2, 3)


@pytest.mark.parametrize('refine', [False, True])
def test_mismatched_batch_sizes_raise(refine):
    from pvraft_b200 import train
    m = model(refine=refine)
    p = clouds(2, 256, 1, 256)
    with pytest.raises(ValueError, match='batch size'):
        m._encode(list(p))
    with pytest.raises(ValueError, match='batch size'):
        train.rsf_forward(m, list(p), 2)


@pytest.mark.parametrize('n1, n2', [(31, 256), (256, 31), (8, 8)])
def test_clouds_below_32_points_raise(n1, n2):
    from pvraft_b200 import train
    m = model(k=8)
    p = list(clouds(1, n1, 1, n2))
    with pytest.raises(ValueError, match='at least 32 points'):
        m._encode(p)
    with pytest.raises(ValueError, match='at least 32 points'):
        train.rsf_forward(m, p, 2)


def test_truncate_k_above_the_second_cloud_raises():
    from pvraft_b200 import ops, train
    m = model(k=128)
    p = list(clouds(2, 512, 2, 100))       # N1 >= K does not help: candidates are rows of xyz2
    with pytest.raises(ValueError, match='truncate_k=128 exceeds the number of points 100'):
        m._encode(p)
    with pytest.raises(ValueError, match='truncate_k=128 exceeds'):
        train.rsf_forward(m, p, 2)
    ops.check_pair(torch.rand(2, 100, 3), torch.rand(2, 512, 3), 128)   # N1 < K <= N2 is fine


def test_bad_ranks_raise():
    from pvraft_b200 import ops
    with pytest.raises(ValueError, match=r'xyz1 \[B,N1,3\], xyz2 \[B,N2,3\]'):
        ops.check_pair(torch.rand(2, 64, 3), torch.rand(2, 64, 4), 32)
    with pytest.raises(ValueError, match=r'xyz1 \[B,N1,3\]'):
        ops.check_pair(torch.rand(64, 3), torch.rand(2, 64, 3), 32)


@pytest.mark.parametrize('n, m', [(1000, 3000), (3000, 1000), (49152, 49153), (60000, 200000), (300, 100000)])
def test_corr_plan_with_unequal_sizes(n, m):
    from pvraft_b200 import ops
    b, c, k = 2, 128, 512
    plan = ops.corr_plan(b, n, m, c, k)
    rows = [r for _, r in plan.row_blocks]
    assert plan.row_blocks[0][0] == 0 and sum(rows) == n                      # the rows tile fmap1's N
    assert all(r0 % 128 == 0 for r0, _ in plan.row_blocks)
    assert plan.windows[0][0] == 0 and sum(w for _, w in plan.windows) == m   # the columns tile fmap2's M
    assert all(c0 % 128 == 0 and w <= ops.CORR_ROW_MAX for c0, w in plan.windows)
    if m <= ops.CORR_ROW_MAX:
        assert plan.dense and plan.slab_bytes == 4 * b * ops._pad128(n) * ops._pad128(m)
    else:
        assert not plan.dense and len(plan.windows) == -(-m // ops.CORR_ROW_MAX) and plan.windows[-1][1] >= k
        assert plan.slab_bytes <= ops.CORR_SLAB_CAP + 128 * (4 * plan.ld + 8 * len(plan.windows) * k)


def test_corr_plan_limits_apply_to_the_second_cloud():
    from pvraft_b200 import ops
    k = 1024
    limit = ops.CORR_ROW_MAX // k * ops.CORR_ROW_MAX          # the windows' W*K candidates must fit one merge row
    ops.corr_plan(1, 1000, limit, 128, k)
    with pytest.raises(ValueError, match='candidates per row'):
        ops.corr_plan(1, 1000, limit + 1, 128, k)
    ops.corr_plan(1, limit + 1, 1000, 128, k)                 # a long first cloud needs no windows at all
    with pytest.raises(ValueError, match='truncate_k'):
        ops.corr_plan(1, 100000, 50000, 128, 50001)


def test_graph_key_depends_on_the_second_cloud():
    m = model()
    a, b = torch.rand(1, 8192, 3), torch.rand(1, 12288, 3)
    c = torch.rand(1, 16384, 3)
    assert m._graph_key(a, b, 8) != m._graph_key(a, c, 8)
    assert m._graph_key(a, b, 8) == m._graph_key(a, b.clone(), 8)
    assert m._graph_key(a, a, 8) != m._graph_key(a, b, 8)


def test_bf16_state_limit_is_on_the_second_cloud():
    from pvraft_b200 import ops
    with pytest.raises(ValueError, match='65536'):
        # checked before anything runs on the device: the state's rows (N1) do not matter, the ids address N2 rows
        ops.corr_state_pack_bf16(torch.zeros(1, 100, 32), torch.zeros(1, 100, 32, dtype=torch.int32), 70000)
