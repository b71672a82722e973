"""compute-sanitizer target for the derived channels (channel_kernel behind b200_sixdof_set_channels, the reductions
and run summaries that read channel planes, and b200_sixdof_{trajectory,state}_channels):

    compute-sanitizer --tool memcheck python scripts/sanitizer_channels.py

Every channel kind, on the index arithmetic an out-of-bounds access would come from: the first and the last body
before the padding to the plane stride (n_bodies not a multiple of 128), one world, ring slices (the ring's samples,
then a ring that is not full), and state calls; each reduction that reads a channel plane (statistics, quantiles,
covariance, histograms, their grouped forms, extrema and thresholds) runs once.  The channel values are checked against
a numpy restatement of the NORM channels, so a wrong index also shows as a wrong value.  Small sizes: the tool slows
every kernel by 10-50x."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import elodin_b200 as el
from elodin_b200 import _lib

CHANNELS = [(_lib.CHANNEL_NORM, 3, (10, 11, 12)), (_lib.CHANNEL_NORM, 2, (4, 5), (1.0, -1.0)),
            (_lib.CHANNEL_NORM, 1, (24,), (), (), 2.0), (_lib.CHANNEL_AXIS_ANGLE, 0, (), (-1.0, 0.0, 0.0), (0.0, 0.0, 1.0)),
            (_lib.CHANNEL_AXIS_ANGLE, 3, (22,), (0.0, 1.0, 0.0))]


def norms(rows):
    return np.stack([np.sqrt((rows[..., 10] * rows[..., 10] + rows[..., 11] * rows[..., 11]) + rows[..., 12] * rows[..., 12]),
                     np.sqrt((rows[..., 4] - 1.0) * (rows[..., 4] - 1.0) + (rows[..., 5] + 1.0) * (rows[..., 5] + 1.0)),
                     np.sqrt(rows[..., 24] * rows[..., 24]) - 2.0], -1)


def run(M, E, capacity, steps):
    rng = np.random.default_rng(M * E + capacity)
    x = rng.normal(size=(M, E, 25))
    ine = np.broadcast_to(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 7))
    with el.B200Exec(E, M, 0.01, None, [], "rk4", "exact", trajectory_every=1, trajectory_capacity=capacity,
                     trajectory_full=True) as ex:
        ex.set_state(x[..., :7], x[..., 7:13], ine, accel=x[..., 13:19], force=x[..., 19:25])
        ex.set_channels(CHANNELS)
        ex.set_world_groups([M // 2, M - M // 2])
        ex.summary_begin(True, [(E - 1, 26, True, 0.5), (0, 29, False, 1.0)])
        ex.summary_add_state()
        now = ex.state_channels()
        assert np.array_equal(now[..., :3], norms(x)), (M, E)
        ex.step(steps)
        ex.sync()
        ex.summary_add_trajectory()
        got = ex.trajectory_channels()
        assert np.array_equal(got[..., :3], norms(ex.trajectory())), (M, E)
        for pre in ("trajectory", "state"):
            getattr(ex, f"{pre}_stats")()
            getattr(ex, f"{pre}_quantiles")((0.0, 0.5, 1.0))
            getattr(ex, f"{pre}_covariance")([25, 29, 4])
            getattr(ex, f"{pre}_histograms")([(E - 1, 27, 8, 0.0, 4.0), (0, (25, 28), (4, 4), (0.0, 0.0), (3.0, 3.2))])
            getattr(ex, f"{pre}_group_stats")()
            getattr(ex, f"{pre}_group_quantiles")((0.5,))
            getattr(ex, f"{pre}_group_covariance")([29, 25])
            getattr(ex, f"{pre}_group_histograms")([(0, 29, 4, 0.0, 3.2)])
        ex.extrema()
        ex.thresholds()


run(300, 1, 3, 3)    # 300 bodies: the last one is the padding edge of a 384-body stride; a full ring
run(43, 3, 4, 2)     # 129 bodies, 3 entities a world; a ring of 2 of its 4 slots
run(1, 1, 1, 1)      # one world
print("done")
