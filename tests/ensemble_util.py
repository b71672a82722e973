"""Helpers shared by the ensemble tests (statistics, quantiles, covariance, run summaries) and the gloo tests: the test
worlds and handles, the 25-plane sample layout, and a two-process gloo harness."""

import os
import socket

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import world as world_mod

# the 25-plane sample layout (B200_TRAJ_FULL), kept here independently of the library's own copy
SAMPLED = {"world_pos": (0, 7), "world_vel": (7, 13), "world_accel": (13, 19), "force": (19, 25)}

ROCKET, FREE = "rocket", "free"


def need_gpu():
    if el.device_count() < 1:
        pytest.skip("needs a CUDA device")


def sampled_state(ex):
    """The handle's current state in the sample layout: [M, N, 25]."""
    from elodin_b200.executor import FORCE, WORLD_ACCEL, WORLD_POS, WORLD_VEL

    return np.concatenate([ex.download(c) for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)], axis=-1)


def handle(kind, M, N, math_mode, width=25, every=1, capacity=4, seed=0, state=None):
    """A handle with a trajectory ring and a random initial state (or `state`); returns (handle, (pos, vel, ine,
    columns, dt)).  ROCKET adds gravity, thrust and drag with per-world thrust and wind columns."""
    from tests.util import near_world

    pos, vel, ine, cols, dt = near_world(seed, M, N) if state is None else state
    effs, up = [], {}
    if kind == ROCKET:
        effs = [el.GravityConst((0.0, 0.0, -9.81)), el.ThrustBody((-1.0, 0.0, 0.0), "thrust"),
                el.DragQuadratic(0.6125, 0.0025, "wind")]
        up = {"thrust": cols["thrust"], "wind": cols["wind"]}
    ex = el.B200Exec(N, M, dt, None, effs, "rk4", math_mode, trajectory_every=every, trajectory_capacity=capacity,
                     trajectory_full=width == 25)
    ex.set_state(pos, vel, ine, **up)
    return ex, (pos, vel, ine, cols, dt)


def rocket_world(n_worlds, seed=4):
    """A thrusting rocket at z = 1 and a ball at the origin, both under gravity, with per-world thrust, wind and mass;
    returns (world, six_dof system, world_params)."""
    rng = np.random.default_rng(seed)
    Thrust = el.Annotated[np.ndarray, el.Component("thrust", el.ComponentType.F64)]
    Wind = el.Annotated[np.ndarray, el.Component("wind", el.ComponentType(el.PrimitiveType.F64, (3,)))]

    @el.dataclass
    class Rocket(el.Archetype):
        thrust: Thrust
        wind: Wind

    w = el.World()
    w.spawn([el.Body(world_pos=el.SpatialTransform(angular=el.Quaternion.from_euler([0.0, np.radians(70.0), 0.0]),
                                                   linear=np.array([0.0, 0.0, 1.0])),
                     inertia=el.SpatialInertia(3.0, np.array([0.1, 1.0, 1.0]))),
             Rocket(np.array([88.426]), np.zeros(3))], name="rocket")
    w.spawn(el.Body(world_vel=el.SpatialMotion(linear=[1.0, 2.0, 0.0])), name="ball")
    effs = el.GravityConst((0.0, 0.0, -9.81)) | el.ThrustBody((-1.0, 0.0, 0.0), "thrust") | el.DragQuadratic(0.6125, 0.0025, "wind")
    params = {"thrust": 88.426 * rng.uniform(0.8, 1.2, (n_worlds, 1, 1)),
              "wind": np.concatenate([rng.normal(0, 2, (n_worlds, 1, 1)), np.zeros((n_worlds, 1, 2))], -1),
              "inertia": np.tile(np.array([0.1, 1.0, 1.0, 0, 0, 0, 3.0]), (n_worlds, 2, 1))}
    params["inertia"][:, 0, 6] = rng.uniform(2.5, 3.5, n_worlds)
    return w, el.six_dof(sys=effs), params


def two_body_world():
    w = el.World()
    w.spawn(el.Body(world_pos=el.SpatialTransform(linear=np.array([0.0, 0.0, 1.0]))), name="rocket")
    w.spawn(el.Body(), name="ball")
    return w


@pytest.fixture
def no_device(monkeypatch):
    """Fail the test if World.build reaches the device (the handle is created through world.B200Exec)."""
    def boom(*a, **k):
        raise AssertionError("validation must finish before the handle is created")
    monkeypatch.setattr(world_mod, "B200Exec", boom)


def split(rng, n, k):
    """k parts of n values (empty parts included) in random sizes."""
    cuts = np.sort(rng.integers(0, n + 1, size=k - 1))
    return np.split(np.arange(n), cuts)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_rank(worker, rank, world_size, port, q, args):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world_size)
    q.put((rank, worker(rank, world_size, *args)))
    dist.barrier()
    dist.destroy_process_group()


def run_gloo(worker, world_size, *args):
    """worker(rank, world_size, *args) in `world_size` spawned processes that share one gloo group on 127.0.0.1;
    returns the workers' results in rank order, after every process has exited with 0.  `worker` must be importable
    (a module-level function)."""
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_rank, args=(worker, r, world_size, port, q, args)) for r in range(world_size)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in range(world_size))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return [got[r] for r in range(world_size)]
