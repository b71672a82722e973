"""compute-sanitizer target for the grouped ensemble entries (world_stats_chunk_kernel / world_stats_merge_kernel and
hist_kernel driven by a world-group table; the quantile kernels and cov_chunk_kernel / cov_merge_kernel driven by the
quantiles' route order and the covariance group table):

    compute-sanitizer --tool memcheck python scripts/sanitizer_group_kernels.py

Every grouped entry (state / trajectory statistics and histograms) and its ungrouped twin, on small batches with empty
leading, middle and trailing groups, groups of one and of several chunks (the merge launch), and a ring whose partials
run in two slices of planes (E = 300, a 512-world group of 64 chunks, 16 samples of 25 planes).  The group index
arithmetic an out-of-bounds access would come from: the binary search over the table, the empty groups (one empty
statistics chunk, no histogram chunk), the group table placed after the edges in the staging buffer and the per-slice
scratch offsets.  Each case also checks what a wrong index would change: group counts against numpy, and the sum of the
grouped histograms against the ungrouped table.  The grouped quantiles and covariance: empty leading, middle and
trailing groups in a call that takes the warp, block and radix routes at once; a radix call whose (group, plane) rows
run in two slices (E = 30, 45 rows a slice); and a covariance call whose groups run in two slices of partials (100
groups of 528 chunks at p = 25).  The quantiles are checked against np.quantile per group, the covariance counts
against the complete worlds of each group.  Small sizes: the tool slows every kernel by 10-50x."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import elodin_b200 as el

SPECS = [(0, 4, 16, -3.0, 3.0), (1, (4, 5), (8, 8), (-3.0, -3.0), (3.0, 3.0))]


def run(sizes, E, samples):
    M = sum(sizes)
    rng = np.random.default_rng(M + E)
    x = rng.normal(size=(M, E, 25))
    x[rng.random(x.shape) < 0.02] = np.nan
    ine = np.broadcast_to(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 7))
    with el.B200Exec(E, M, 0.01, None, [], "rk4", "exact", trajectory_every=1, trajectory_capacity=samples,
                     trajectory_full=True) as ex:
        ex.set_state(x[..., :7], x[..., 7:13], ine, accel=x[..., 13:19], force=x[..., 19:25])
        ex.step(samples)
        ex.set_world_groups(sizes)
        specs = [s for s in SPECS if s[0] < E]
        st, tr = ex.state_group_stats(), ex.trajectory_group_stats()
        sh, th = ex.state_group_histograms(specs), ex.trajectory_group_histograms(specs)
        assert np.array_equal(sh.sum(0), ex.state_histograms(specs)) and np.array_equal(th.sum(1), ex.trajectory_histograms(specs))
        traj = ex.trajectory()
        now = np.concatenate([ex.download(c) for c in ("world_pos", "world_vel", "world_accel", "force")], -1)
    o = np.concatenate([[0], np.cumsum(sizes)])
    for g in range(len(sizes)):
        assert np.array_equal(st[g, ..., 0], np.isfinite(now[o[g]:o[g + 1]]).sum(0)), g
        assert np.array_equal(tr[:, g, ..., 0], np.isfinite(traj[:, o[g]:o[g + 1]]).sum(1)), g


run([0, 5, 0, 700, 1, 0], 3, 3)          # empty first / middle / last groups; 700 worlds = 2 chunks at E = 3
run([0, 512, 3, 0], 300, 16)             # 64 chunks at E = 300; 400 planes of partials in two slices
run([1] * 40 + [0] * 20 + [5000], 1, 2)  # many one-chunk groups, a run of empty ones, one group of 3 chunks


def state(M, E, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(M, E, 25)) + np.arange(M)[:, None, None] * 1e-3
    x[rng.random(x.shape) < 0.02] = np.nan
    return x


def handle(x):
    M, E, _ = x.shape
    ine = np.broadcast_to(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 7))
    ex = el.B200Exec(E, M, 0.01, None, [], "rk4", "exact", trajectory_every=1, trajectory_capacity=1, trajectory_full=True)
    ex.set_state(x[..., :7], x[..., 7:13], ine, accel=x[..., 13:19], force=x[..., 19:25])
    return ex


Q = (0.0, 0.01, 0.5, 0.99, 1.0)
SEL = (4, 5, 6, 10, 11, 12)


def run_quantiles(sizes, E, planes=range(25)):
    x = state(sum(sizes), E, sum(sizes) + E)
    with handle(x) as ex:
        ex.set_world_groups(sizes)
        st = ex.state_group_quantiles(Q)
        ex.step(1)
        tr = ex.trajectory_group_quantiles(Q)
        traj = ex.trajectory()
    o = np.concatenate([[0], np.cumsum(sizes)])
    for g in range(len(sizes)):
        for e in range(E):
            for i in planes:
                for got, v in ((st[g, e, i], x[o[g]:o[g + 1], e, i]), (tr[0, g, e, i], traj[0, o[g]:o[g + 1], e, i])):
                    f = v[np.isfinite(v)]
                    want = np.quantile(f, Q) if f.size else np.full(len(Q), np.nan)
                    assert np.array_equal(got, want, equal_nan=True), (g, e, i)


def run_covariance(sizes, E, p_planes=SEL):
    x = state(sum(sizes), E, sum(sizes) + 2 * E)
    with handle(x) as ex:
        ex.set_world_groups(sizes)
        st = ex.state_group_covariance(p_planes)
        ex.step(1)
        tr = ex.trajectory_group_covariance(p_planes)
        traj = ex.trajectory()
    o = np.concatenate([[0], np.cumsum(sizes)])
    for g in range(len(sizes)):
        ok = np.isfinite(x[o[g]:o[g + 1]][..., list(p_planes)]).all(-1).sum(0)
        assert np.array_equal(st[g, :, 0], ok), g
        ok = np.isfinite(traj[0, o[g]:o[g + 1]][..., list(p_planes)]).all(-1).sum(0)
        assert np.array_equal(tr[0, g, :, 0], ok), g


run_quantiles([0, 5, 0, 300, 9000, 0], 2)      # empty first / middle / last groups; warp, block and radix routes
run_quantiles([3, 8193, 8200], 30, (0, 24))    # 50 (group, plane) rows of the radix groups: two slices of 45 rows
run_covariance([0, 5, 0, 700, 64, 65, 0], 3)   # empty first / middle / last groups, one- and several-chunk groups
run_covariance([528 * 64] * 100, 1, tuple(range(25)))  # 2.75 MB of partials per group: slices of 97 and 3 groups
with el.B200Exec(0, 4, 0.01, None, [], "rk4", "exact") as ex:  # a world without entities takes groups too
    ex.set_world_groups([4, 0])
    assert ex.state_group_stats().shape == (2, 0, 25, 5)
    assert ex.state_group_quantiles(Q).shape == (2, 0, 25, len(Q))
    assert ex.state_group_covariance(SEL).shape == (2, 0, 1 + 6 + 36)
print("done")
