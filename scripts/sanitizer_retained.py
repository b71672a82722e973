"""compute-sanitizer target for the retained-world entries (gather_worlds_kernel behind
b200_sixdof_trajectory_download_worlds and b200_sixdof_state_download_worlds):

    compute-sanitizer --tool memcheck python scripts/sanitizer_retained.py

Both entries, host and device destinations, on the index arithmetic an out-of-bounds access would come from: the first
world, the last world, whose last entity is the last body before the padding to the plane stride (n_bodies not a
multiple of 128), a tile of output bodies that ends inside a world, a 13-wide ring, and a call whose rows run in two
staging slices (65 536 retained bodies x 25 planes, 21 samples: 20 + 1).  Each case is checked against the full
download, so a wrong index also shows as a wrong value.  Small sizes elsewhere: the tool slows every kernel by
10-50x."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import elodin_b200 as el


def handle(M, E, width, samples):
    rng = np.random.default_rng(M * E + width)
    x = rng.normal(size=(M, E, 25))
    ine = np.broadcast_to(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 7))
    ex = el.B200Exec(E, M, 0.01, None, [], "rk4", "exact", trajectory_every=1, trajectory_capacity=samples,
                     trajectory_full=width == 25)
    ex.set_state(x[..., :7], x[..., 7:13], ine, accel=x[..., 13:19], force=x[..., 19:25])
    ex.step(samples)
    return ex


def run(M, E, width, samples, worlds):
    with handle(M, E, width, samples) as ex:
        traj = ex.trajectory()
        now = np.concatenate([ex.download(c) for c in ("world_pos", "world_vel", "world_accel", "force")], -1)
        got = ex.trajectory_worlds(worlds)
        assert got.tobytes() == np.ascontiguousarray(traj[:, worlds]).tobytes(), (M, E, width)
        assert ex.state_worlds(worlds).tobytes() == np.ascontiguousarray(now[worlds]).tobytes(), (M, E, width)
        dev = torch.empty(got.shape, dtype=torch.float64, device="cuda")
        ex.trajectory_worlds(worlds, dev.data_ptr(), dev.numel() * 8)
        assert dev.cpu().numpy().tobytes() == got.tobytes(), (M, E, width)
        dev = torch.empty((len(worlds), E, 25), dtype=torch.float64, device="cuda")
        ex.state_worlds(worlds, dev.data_ptr(), dev.numel() * 8)
        assert dev.cpu().numpy().tobytes() == np.ascontiguousarray(now[worlds]).tobytes(), (M, E, width)


run(300, 1, 25, 3, [0, 299])                     # 300 bodies: the last one is the padding edge of a 384-body stride
run(43, 3, 13, 2, [42, 0, 21, 42])               # 129 bodies, 3 entities a world; repeats; tiles end inside a world
run(1, 1, 25, 1, [0])                            # one world
run(100, 7, 25, 2, list(range(100)) * 3)         # 2100 output bodies: 9 tiles, the last one partial
run(2048, 1, 25, 21, list(np.arange(65536) % 2048)[::-1])  # 13.1 MB a sample: two staging slices (20 + 1)
print("done")
