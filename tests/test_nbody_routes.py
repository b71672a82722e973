"""Every FAST route of the all-pairs edge_fold gravity, against the oracle body by body.

The launchers pick the gravity kernel from the world size N, the batch's CTA count gridf = ceil(N/8) * M against
3 x 132 SMs, and the world kernel's four-source item count against 8 x 16 x SMs (graph_kernels.cu).  Each case
asserts the kernels that actually ran (torch.profiler, CUDA activity), so a change of threshold or a card with
another SM count fails loudly instead of quietly testing another route, and compares what the run changed with
the oracle per body (tests.util.assert_nbody_close).  EXACT stays bit-identical.  The B200_* route switches are read
once per process, so their cases run in child processes.
"""

import os

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200.executor import FORCE, INERTIA, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from tests.util import assert_nbody_close, assert_route, launched_kernels, nbody_world, run_child

pytestmark = pytest.mark.gpu

DT = 1e-3

# kernel name prefixes (template arguments: RK4 / SPLIT / TJ, and for the world kernel RK4, TJ, threads, min CTAs,
# sources x targets per item, FUSE, body signature; signature 32 = gravity alone, 2147483648 = run-time interpreter)
FUSED = "nbody_tick_fused_kernel<1024>"
WORLD_4x1 = "graph_dense_world_kernel<true, 1024, 512, 1, 4, 1, "
WORLD_2x2 = "graph_dense_world_kernel<true, 1024, 512, 1, 2, 2, "
WORLD_SEMI = "graph_dense_world_kernel<false, 1024, 512, 1, 2, 2, false, "
DENSE_FAST = "graph_dense_fast_kernel<true, false, 256>"
DENSE_SPLIT = "graph_dense_fast_kernel<true, true, 1024>"
DENSE_SEMI = "graph_dense_fast_kernel<false, false, 256>"
BODY_RK4 = "body_fast_spec_kernel<0, 32, false, 128, 4, 1>"  # gravity-only signature, one body per thread
BODY_RK4_PAIR = "body_fast_spec_kernel<0, 32, false, 128, 3, 2>"  # ... two bodies per thread
BODY_SEMI = "body_fast_spec_kernel<1, 32, false, 128, 4, 1>"


def _world_kernel(prefix, fuse, gravity_only):
    return prefix + f"{'true' if fuse else 'false'}, {32 if gravity_only else 2147483648}>"


def _threads(O):
    return max(1, min(O.max_threads(), os.cpu_count() or 1))


def _setup(O, M, N, extra):
    """The seeded world of a (M, N) case: (pos, vel, ine, S), oracle effectors (None without an oracle), library
    effectors, effector columns."""
    pos, vel, ine, k, soft, S = nbody_world(1000 * N + M, M, N, DT)
    edges = el.all_pairs_edges(N)
    ge = [el.GravityEdges("softened", k_squared=k, softening=soft, edges=edges)]
    oe = [O.Effector(O.EFF_GRAVITY_EDGES_SOFTENED, p=(k, soft), edges=edges)] if O else None
    cols = {}
    if extra:  # a body-frame thrust comparable to the gravity: the integration then runs the interpreter
        thrust = np.random.default_rng(N + M).uniform(0.5, 2.0, (M, N, 1)) * ine[..., 6:7] * np.median(S)
        ge.append(el.ThrustBody((-1.0, 0.0, 0.0), "thrust"))
        cols["thrust"] = thrust
        if O:
            oe.append(O.Effector(O.EFF_THRUST_BODY, p=(-1.0, 0.0, 0.0), column=thrust))
    return (pos, vel, ine, S), oe, ge, cols


def _oracle_states(O, start, effs, integrator, ticks):
    """The oracle's (pos, vel, accel, force) after each cumulative tick count in `ticks`."""
    pos, vel, ine = start[:3]
    w = O.World(pos, vel, ine)
    out, done = [], 0
    for t in ticks:
        if integrator == "rk4":
            w.rk4(DT, t - done, effs, threads=_threads(O))
        else:
            w.semi_implicit(DT, t - done, effs, threads=_threads(O))
        done = t
        out.append(tuple(a.copy() for a in (w.pos, w.vel, w.accel, w.force)))
    return out


def _download(ex):
    return tuple(ex.download(c) for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE))


def _table(ex, tick, state, ine, cols):
    M, N = state[0].shape[:2]
    t = {el.component_id("tick"): np.array([tick], dtype=np.uint64), FORCE: np.zeros((M, N, 6)), INERTIA: ine,
         WORLD_POS: state[0], WORLD_ACCEL: np.zeros((M, N, 6)), el.component_id("simulation_time_step"): np.array([DT]),
         WORLD_VEL: state[1]}
    t.update({el.component_id(k): v for k, v in cols.items()})
    return [t[c] for c in ex.input_ids]


def _counted_step(ex, n):
    """step(n); returns how many kernels the library launched for it."""
    n0 = ex.timings()["kernel_launches"]
    ex.step(n, sync=True)
    return ex.timings()["kernel_launches"] - n0


def _check(got, want, start, ticks, what):
    pos, vel, ine, S = start
    return assert_nbody_close(got, want, (pos, vel, ine), DT, ticks, S, what=what)


# (M, N), integrator, thrust next to the gravity, expected tick kernels, one-launch (ping-pong) route
ROUTES = [
    # nbody_tick_fused_kernel: N in 33..63 or > 1024 on a grid below 396 CTAs (gridf 395 at (79, 40); two
    # 1024-target tiles at N = 1100)
    *[((M, N), "rk4", x, [FUSED], True) for (M, N) in ((1, 33), (7, 63), (79, 40), (2, 1100)) for x in (False, True)],
    # two launches: graph_dense_fast_kernel<RK4, non-split, 256> + the gravity-signature body kernel (gridf 400 / 414:
    # the twin of (79, 40) on the other side of 396; a partial 256-target tile)
    ((80, 40), "rk4", False, [DENSE_FAST, BODY_RK4], False),
    ((3, 1100), "rk4", False, [DENSE_FAST, BODY_RK4], False),
    # 103 400 bodies: the body-pair kernel, with pairs that straddle two worlds (odd N)
    ((2200, 47), "rk4", False, [DENSE_FAST, BODY_RK4_PAIR], False),
    # semi-implicit: graph_dense_fast_kernel<SEMI> outside 64..1024, the world kernel without fusion inside
    ((2, 40), "semi_implicit", False, [DENSE_SEMI, BODY_SEMI], False),
    ((1, 1100), "semi_implicit", False, [DENSE_SEMI, BODY_SEMI], False),
    ((41, 97), "semi_implicit", False, [WORLD_SEMI, BODY_SEMI], False),
    ((3, 1024), "semi_implicit", False, [WORLD_SEMI, BODY_SEMI], False),
    # world kernel, 4 sources x 1 target per item: items4 = 18 432 with 5 CTAs per world; 17 280 with M > 132 CTAs,
    # so a CTA walks several worlds
    *[((M, N), "rk4", x, [_world_kernel(WORLD_4x1, True, not x)], True) for (M, N) in ((24, 1024), (180, 128)) for x in (False, True)],
    # small_world_kernel<FAST, SEMI, gravity signature>
    ((41, 7), "semi_implicit", False, ["small_world_kernel<false, 1, 4, 32>"], False),
]


def _route_id(r):
    (M, N), integ, extra, _, _ = r
    return f"{M}x{N}-{'rk4' if integ == 'rk4' else 'semi'}{'-thrust' if extra else ''}"


# ---------------------------------------------------------------------------- which kernels ran
#
# torch.profiler sees the library's launches, but it loses the records of a short profiling window now and then, more
# often once the process has run other CUDA work (seen with torch 2.11 / CUDA 12.8 on an H100).  So the kernel names
# are recorded in a fresh child process per set of route switches, and an attempt counts only when it saw as many
# launches as the library counts.  The parent checks the names, and in its own runs the launch count per tick.


def _child_run(out_path, cases, attempts=3):
    """Child process: run each case ([M, N, integrator, thrust, math, invoke range in worlds or 0 for step()]) for two
    ticks on a fresh handle under the profiler; write the kernel names and the final state of each case."""
    res = {}
    for k, (M, N, integ, extra, math, chunk) in enumerate(cases):
        start, _, ge, cols = _setup(None, M, N, extra)
        pos, vel, ine, _ = start
        for _ in range(attempts):
            with el.B200Exec(N, M, DT, None, ge, integ, math, invoke_chunk_bodies=chunk * N) as ex:
                ex.set_state(pos, vel, ine, **cols)
                n0 = ex.timings()["kernel_launches"]
                if chunk:
                    ins = _table(ex, 0, (pos, vel), ine, cols)
                    outs, names = launched_kernels(lambda: ex.invoke_batch(ins, 2))
                    launches = ex.timings()["kernel_launches"] - n0
                    out = dict(zip(ex.output_ids, outs))
                    state = (out[WORLD_POS], out[WORLD_VEL], out[WORLD_ACCEL], out[FORCE])
                else:
                    _, names = launched_kernels(lambda: ex.step(2, sync=True))
                    launches = ex.timings()["kernel_launches"] - n0
                    state = _download(ex)
            names = [n for n in names if not n.startswith(("Memcpy", "Memset"))]
            if len(names) == launches:
                break
        for name, a in zip(("pos", "vel", "accel", "force"), state):
            res[f"{k}_{name}"] = a
        res[f"{k}_kernels"] = np.array(names)
        res[f"{k}_launches"] = launches
    np.savez(out_path, **res)


def _run_child(cases, out, setting=None):
    """Run _child_run in a child process (with one B200_* route switch set) and load what it wrote."""
    return run_child("tests.test_nbody_routes:_child_run", out, cases, setting)


def _names(res, k, kernels, what):
    names, launches = list(res[f"{k}_kernels"]), int(res[f"{k}_launches"])
    assert len(names) == launches, f"{what}: the profiler saw {len(names)} of {launches} launches in every attempt: {names}"
    assert_route(names, kernels, what)


# every default-route case below, recorded once: (key, [M, N, integrator, thrust, math, invoke range])
def _default_cases():
    cases = [(_route_id(r), [r[0][0], r[0][1], r[1], r[2], "fast", 0]) for r in ROUTES]
    cases.append(("80x40-split", [80, 40, "rk4", False, "fast", 10]))
    cases += [(f"exact-{M}x{N}", [M, N, integ, False, "exact", 0]) for (M, N), integ, _ in EXACT]
    return cases


@pytest.fixture(scope="module")
def default_routes(tmp_path_factory):
    cases = _default_cases()
    res = _run_child([c for _, c in cases], str(tmp_path_factory.mktemp("routes") / "default.npz"))
    return {key: (res, k) for k, (key, _) in enumerate(cases)}


@pytest.mark.parametrize("route", ROUTES, ids=[_route_id(r) for r in ROUTES])
def test_fast_nbody_route_matches_the_oracle(oracle, default_routes, route):
    """Two ticks in one step() on the expected kernels, per body against the oracle.  The one-launch routes keep the
    new state in the second plane set every other tick: they also run an odd tick count, then a chunked
    invoke_batch, and the device-resident state must equal what invoke_batch returned."""
    O = oracle
    (M, N), integ, extra, kernels, fused = route
    what = _route_id(route)
    _names(*default_routes[what], kernels, what)
    start, oe, ge, cols = _setup(O, M, N, extra)
    pos, vel, ine, _ = start
    want = _oracle_states(O, start, oe, integ, (2, 3, 5) if fused else (2,))
    with el.B200Exec(N, M, DT, None, ge, integ, "fast") as ex:
        ex.set_state(pos, vel, ine, **cols)
        assert _counted_step(ex, 2) == 2 * len(kernels), what
        _check(_download(ex), want[0], start, 2, f"{what} step(2)")
    if not fused:
        return
    with el.B200Exec(N, M, DT, None, ge, integ, "fast", invoke_chunk_bodies=max(1, (M * 3) // 4) * N) as ex:
        ex.set_state(pos, vel, ine, **cols)
        assert _counted_step(ex, 3) == 3, what
        mid = _download(ex)
        _check(mid, want[1], start, 3, f"{what} step(3)")
        out = dict(zip(ex.output_ids, ex.invoke_batch(_table(ex, 3, mid, ine, cols), 2)))
        got = (out[WORLD_POS], out[WORLD_VEL], out[WORLD_ACCEL], out[FORCE])
        _check(got, want[2], start, 5, f"{what} step(3) + invoke_batch(2)")
        assert np.array_equal(ex.download(WORLD_POS), out[WORLD_POS]) and np.array_equal(ex.download(WORLD_VEL), out[WORLD_VEL])
        assert int(out[el.component_id("tick")][0]) == 5


def test_split_dense_kernel_through_invoke_batch_ranges(oracle, default_routes):
    """invoke_batch splits 80 worlds of 40 bodies into 10-world ranges: the handle's batch is past 396 CTAs (two
    launches per tick), each range's grid (50 CTAs) is not, so the gravity runs on the split 1024-target kernel."""
    O = oracle
    M, N = 80, 40
    res, k = default_routes["80x40-split"]
    _names(res, k, [DENSE_SPLIT, BODY_RK4], "80x40 in 10-world ranges")
    start, oe, _, _ = _setup(O, M, N, False)
    want = _oracle_states(O, start, oe, "rk4", (2,))
    _check(tuple(res[f"{k}_{n}"] for n in ("pos", "vel", "accel", "force")), want[0], start, 2, "80x40 split")


EXACT = [((1, 1100), "rk4", ["graph_dense_kernel<true, true>", "body_exact_kernel<0, "]),
         ((3, 130), "semi_implicit", ["graph_dense_kernel<true, false>", "body_exact_kernel<1, "])]


@pytest.mark.parametrize("shape,integ,kernels", EXACT, ids=["1x1100-rk4", "3x130-semi"])
def test_exact_nbody_beyond_one_block_is_bit_exact(oracle, default_routes, shape, integ, kernels):
    """EXACT all-pairs gravity past one 1024-body block (RK4) and past 33 bodies (semi-implicit): bit for bit."""
    O = oracle
    M, N = shape
    _names(*default_routes[f"exact-{M}x{N}"], kernels, f"exact {shape}")
    start, oe, ge, cols = _setup(O, M, N, False)
    pos, vel, ine, _ = start
    want = _oracle_states(O, start, oe, integ, (2,))[0]
    with el.B200Exec(N, M, DT, None, ge, integ, "exact") as ex:
        ex.set_state(pos, vel, ine)
        assert _counted_step(ex, 2) == 4
        got = _download(ex)
    for name, a, b in zip(("pos", "vel", "accel", "force"), got, want):
        assert np.array_equal(a, b), f"exact {shape} {name}: max abs diff {np.max(np.abs(a - b))}"


# --------------------------------------------------------------------------- route switches, one process each

# B200_* setting -> cases ((M, N), integrator, expected tick kernels)
SWITCHES = {
    "B200_GRAPH_CFG=0": [((80, 40), "rk4", ["graph_dense_kernel<false, true>", BODY_RK4]),
                         ((41, 97), "semi_implicit", ["graph_dense_kernel<false, false>", BODY_SEMI])],
    "B200_GRAPH_CFG=2": [((3, 1100), "rk4", [DENSE_SPLIT, BODY_RK4]),
                         ((41, 97), "semi_implicit", [DENSE_SEMI, BODY_SEMI])],
    "B200_NBODY_FUSED=0": [((41, 97), "rk4", [_world_kernel(WORLD_2x2, False, False), BODY_RK4]),
                           ((1, 33), "rk4", [DENSE_SPLIT, BODY_RK4])],
    "B200_NBODY_FUSED=2": [((180, 128), "rk4", [_world_kernel(WORLD_4x1, False, False), BODY_RK4]),
                           ((1, 33), "rk4", [FUSED])],
    "B200_NBODY_WORLD_MIN=396": [((2, 333), "rk4", [FUSED]), ((3, 1024), "rk4", [FUSED]),
                                 ((41, 97), "rk4", [_world_kernel(WORLD_2x2, True, True)])],
    "B200_SMALL_WORLD=0": [((41, 7), "semi_implicit", [DENSE_SEMI, BODY_SEMI]), ((41, 7), "rk4", [FUSED])],
}


@pytest.mark.parametrize("setting", list(SWITCHES))
def test_route_switch_in_a_child_process(oracle, setting, tmp_path):
    """Each B200_* route switch sends its shapes to the fallback kernels it names (DESIGN §8a); the results are
    compared with the oracle exactly like the default routes'."""
    O = oracle
    cases = SWITCHES[setting]
    res = _run_child([[M, N, integ, False, "fast", 0] for (M, N), integ, _ in cases], str(tmp_path / "child.npz"), setting)
    for k, ((M, N), integ, kernels) in enumerate(cases):
        what = f"{setting} {M}x{N} {integ}"
        _names(res, k, kernels, what)
        start, oe, _, _ = _setup(O, M, N, False)
        want = _oracle_states(O, start, oe, integ, (2,))[0]
        _check(tuple(res[f"{k}_{n}"] for n in ("pos", "vel", "accel", "force")), want, start, 2, what)
