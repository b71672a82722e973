"""compute-sanitizer target for the rank pass and the worst-worlds select (rank_kernels.cu behind
b200_sixdof_outcome_[group_]ranks, topk_kernels.cu behind b200_sixdof_outcome_[group_]top_worlds):

    compute-sanitizer --tool memcheck python scripts/sanitizer_rank_topk.py

The index arithmetic an out-of-bounds access would come from, on small versions of the cases of
tests/test_rank_topk_shapes.py: a level that holds its most ranges (R = n / 8193, the size of rg0 / rg1 and of the
histograms), a rank task that refines through all 5 levels (kCap + 1 signed zeros over the key span of +-DBL_MAX), a
rank call of two scratch slices whose boundary falls between one group's planes, and a top-worlds task that switches to
world indices (phase 1) beside worlds on the small routes.  The ranks and records are checked against scipy and the
numpy order, so a wrong index also shows as a wrong value.  Small sizes: the tool slows every kernel by 10-50x."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from tests.test_outcome_rank_correlation import _only_values, ref_ranks, same
from tests.test_outcome_top_worlds import ref_top
from tests.test_rank_topk_shapes import KCAP, KEY_ONE, from_keys, rank_slices, rank_task_bytes

rng = np.random.default_rng(5)


def ranks(values, sizes, planes):
    with _only_values(values, "exact", groups=sizes) as ex:
        got = ex.outcome_group_ranks(planes) if sizes else ex.outcome_ranks(planes)
        assert same(got, ref_ranks(values[:, planes], sizes)), sizes
        return ex.rank_reads()


# R = 2 ranges at level 2: two clusters of kCap + 1 keys in two level-1 bins
cl = np.concatenate([(c * 9000 << 20) + np.arange(KCAP + 1) for c in range(2)])
assert ranks(from_keys(rng.permutation(cl), KEY_ONE)[:, None], None, [0]) == 4.0
# 5 levels: kCap + 1 signed zeros, subnormals and +-DBL_MAX, with a second plane and NaN dropping worlds
M = 9000
v = np.empty((M, 2))
v[:, 0] = rng.normal(0, 1, M)
v[:KCAP + 1, 0] = np.where(np.arange(KCAP + 1) % 2, 0.0, -0.0)
v[KCAP + 1:KCAP + 5, 0] = [5e-324, -1e-310, -np.finfo(np.float64).max, np.finfo(np.float64).max]
v[:, 1] = rng.uniform(-1, 1, M)
v[KCAP + 10:KCAP + 40, 1] = np.nan
v = v[rng.permutation(M)]
assert ranks(v, None, [0]) == 7.0
ranks(v, [100, M - 100], [1, 0])
# two slices, the boundary between the planes of one group: tasks of about 140 MB each
n = 3_300_000
assert rank_slices([n, n]) == [(0, 1, 256 + 40 + rank_task_bytes(n)), (1, 1, 256 + 40 + rank_task_bytes(n))]
big = rng.uniform(1.0, 2.0, (n + 300, 2))
ranks(big, [300, n], [0, 1])
# phase 1 of the select after 2 phase-0 levels, beside the warp and block routes
x = np.full(9000, np.nan)
x[:KCAP + 1], x[KCAP + 1:KCAP + 3] = 1.0, from_keys([KEY_ONE - (1 << 26), KEY_ONE + (1 << 26)])
x = np.concatenate([rng.normal(0, 1, 300), x, rng.normal(0, 1, 40)])[:, None]
sizes = [300, 9000, 40]
with _only_values(x, "exact", groups=sizes) as ex:
    for k, largest in ((2, True), (1024, False)):
        got = ex.outcome_group_top_worlds([0], k, largest)
        o = 0
        for g, m in enumerate(sizes):
            assert same(got[g, 0], ref_top(x[o:o + m, 0], k, largest, o)), (g, k)
            o += m
print("done")
