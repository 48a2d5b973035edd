"""Host side of tests/test_gpu_front_sweep.py: its fused-front shapes reach every branch of launch_front_fwd's plan.
Runs without a GPU."""
from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)

from test_gpu_front_sweep import FRONT_SHAPES, MAX_FIELDS, front_branch, next_pow2_log2, reachable_branches


def test_plan_restatement():
    from fuxictr_b200._lib import B2_MAX_FIELDS
    assert MAX_FIELDS == B2_MAX_FIELDS
    assert [next_pow2_log2(v) for v in (1, 2, 3, 4, 5, 8, 9, 32)] == [0, 1, 2, 2, 3, 3, 4, 5]
    assert front_branch(4, 1) == (1, 2, False)            # 32 rows per pass
    assert front_branch(128, 9) == (32, 8, True)          # one row per pass, 9 passes: two chunks
    assert front_branch(40, 26) == (16, 8, True)          # dim/4 = 10 lanes of 16 on, 13 passes
    assert front_branch(8, 128) == (2, 8, False)          # 16 rows per pass, 8 passes


def test_front_shapes_reach_every_branch():
    """Every (LPR, MAX_PASSES, chunk loop) that a dim in 4..128 (% 4) and 1..B2_MAX_FIELDS fields can select is
    run by the sweep; at LPR = 1 (32 rows per pass) MAX_PASSES = 8 is out of reach, at LPR = 2 the chunk loop."""
    reach = reachable_branches()
    assert len(reach) == 4 * 4 + 3 + 2
    assert (1, 8, False) not in reach and (2, 8, True) not in reach
    swept = {front_branch(dim, F) for dim, F in FRONT_SHAPES}
    assert swept == reach, sorted(reach - swept)
    assert all(dim % 4 == 0 and 4 <= dim <= 128 and 1 <= F <= MAX_FIELDS for dim, F in FRONT_SHAPES)
    # lanes left idle in their row group: dim / 4 not a power of two, at LPR 4, 8, 16 and 32
    idle = {front_branch(dim, F)[0] for dim, F in FRONT_SHAPES if (dim // 4) & (dim // 4 - 1)}
    assert {4, 8, 16, 32} <= idle
