"""compute-sanitizer target for the grouped ensemble entries (world_stats_chunk_kernel / world_stats_merge_kernel and
hist_kernel driven by a world-group table):

    compute-sanitizer --tool memcheck python scripts/sanitizer_group_kernels.py

Every grouped entry (state / trajectory statistics and histograms) and its ungrouped twin, on small batches with empty
leading, middle and trailing groups, groups of one and of several chunks (the merge launch), and a ring whose partials
run in two slices of planes (E = 300, a 512-world group of 64 chunks, 16 samples of 25 planes).  The group index
arithmetic an out-of-bounds access would come from: the binary search over the table, the empty groups (one empty
statistics chunk, no histogram chunk), the group table placed after the edges in the staging buffer and the per-slice
scratch offsets.  Each case also checks what a wrong index would change: group counts against numpy, and the sum of the
grouped histograms against the ungrouped table.  Small sizes: the tool slows every kernel by 10-50x."""
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
with el.B200Exec(0, 4, 0.01, None, [], "rk4", "exact") as ex:  # a world without entities takes groups too
    ex.set_world_groups([4, 0])
    assert ex.state_group_stats().shape == (2, 0, 25, 5)
print("done")
