"""compute-sanitizer target for the run scores (the kScores fold of summary_fold_kernel, scores_clear_kernel and
moment_table_kernel behind b200_sixdof_summary_start, b200_sixdof_moments_download and b200_sixdof_dwells_download):

    compute-sanitizer --tool memcheck python scripts/sanitizer_scores.py

The index arithmetic an out-of-bounds access would come from: the last body before the padding to the plane stride
(n_bodies not a multiple of 128), several entities a world, one world, ring folds and state folds, moments of raw and
channel planes, dwells on several (entity, plane) pairs, and the host- and device-destination downloads.  The tables
are checked against the numpy fold, so a wrong index also shows as a wrong value.  Small sizes: the tool slows every
kernel by 10-50x."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import elodin_b200 as el
from elodin_b200 import _lib

MOMENTS = [0, 6, 24, 25, 12]
CHANNELS = [(_lib.CHANNEL_NORM, 3, (10, 11, 12))]


def fold(rows):
    """the header's sequential fold of rows [R, ...]: (n, mean, m2)"""
    n, K, S1, S2 = (np.zeros(rows.shape[1:]) for _ in range(4))
    with np.errstate(all="ignore"):
        for x in rows:
            fin = np.isfinite(x)
            K = np.where(fin & (n == 0.0), x, K)
            y = x - K
            S1, S2, n = np.where(fin, S1 + y, S1), np.where(fin, S2 + y * y, S2), np.where(fin, n + 1.0, n)
        d = S2 - S1 * (S1 / n)
        return np.stack([n, K + S1 / n, np.where(np.isinf(S2), np.inf, np.where(d < 0.0, 0.0, d))], -1)


def run(M, E, capacity, steps):
    rng = np.random.default_rng(M * E + capacity)
    x = rng.normal(size=(M, E, 25))
    ine = np.broadcast_to(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 7))
    dwells = [(E - 1, 6, True, 0.0), (0, 25, False, 1.5), (0, 6, False, 0.0)]
    with el.B200Exec(E, M, 0.01, None, [], "rk4", "exact", trajectory_every=1, trajectory_capacity=capacity,
                     trajectory_full=True) as ex:
        ex.set_state(x[..., :7], x[..., 7:13], ine, accel=x[..., 13:19], force=x[..., 19:25])
        ex.set_channels(CHANNELS)
        ex.summary_begin(True, [(0, 25, True, 1.0)], MOMENTS, dwells)
        ex.summary_add_state()
        rows = [np.concatenate([x, ex.state_channels()], -1)]
        ex.step(steps)
        ex.sync()
        ex.summary_add_trajectory()
        rows += list(np.concatenate([ex.trajectory(), ex.trajectory_channels()], -1))
        got = ex.moments()
        assert np.array_equal(got, fold(np.stack(rows)[..., MOMENTS]), equal_nan=True), (M, E)
        d = ex.dwells()
        assert d.shape == (M, len(dwells), 3)
        import torch

        dev = torch.empty(got.shape, dtype=torch.float64, device="cuda")
        _lib.check(_lib.lib().b200_sixdof_moments_download(ex._h, dev.data_ptr(), got.nbytes))
        assert np.array_equal(dev.cpu().numpy(), got, equal_nan=True)
        ex.extrema()
        ex.thresholds()


run(300, 1, 3, 3)    # 300 bodies: the last one is the padding edge of a 384-body stride; a full ring
run(43, 3, 4, 2)     # 129 bodies, 3 entities a world; a ring of 2 of its 4 slots
run(1, 1, 1, 1)      # one world
print("done")
