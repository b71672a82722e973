"""The row-sharded n-body step (b200_sixdof_step_row_sharded) on both exchanges, against the oracle.

One world, its source rows split over the ranks of a communicator.  The NCCL exchange all-gathers the rows' new x, v
planes after every tick; the peer window (b200_comm_peer_attach) stores them into every rank's window instead
(peer_fill_kernel, peer_wait_kernel, peer_push_kernel in sixdof_comm.cu).  A one-rank communicator runs both exchanges
end to end on one GPU, so every case here does:

  * CPU: the launches each call makes and the fold kernel launch_graph_force picks, restated and checked on
    hand-worked cases, and a case list that reaches every boundary of that choice;
  * GPU: calls of 1, 2 and 3 ticks on both exchanges.  EXACT equals the oracle bit for bit; FAST peer equals NCCL and
    both equal a plain step() of the two-launch route (the same fold and body kernels) bit for bit, within
    tests.util.assert_nbody_close of the oracle.  Schedules mix the calls with plain steps, set_state, invoke_batch,
    trajectory_reset and a caller stream; the ring of row-sharded ticks equals the ring of plain steps; the window's
    life cycle and the refusals leave the handle usable;
  * CPU: a model of the peer-window protocol at 2..4 ranks, at the level of the kernels' memory events, driven by an
    adversarial scheduler.  Keyed to the window's own tick count it passes every schedule; keyed to the handle's
    ticks_done it fails after a trajectory reset, and it fails on each seeded fault.  With one rank the old rule cannot
    fail (the rank's own push lands before its wait), which is why only the model shows it.

Anything that creates a communicator or needs a route switch runs in a fresh child process: the B200_* switches are
read once per process.
"""

import itertools
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from tests.util import assert_nbody_close, nbody_pair_scale, nbody_world

DT = 1e-3
BENCH_DT = 3600.0  # bench.py's one-world n-body: N = 1024, softened, dt = 3600 s
CALLS = (1, 2, 3)  # ticks of the calls every case makes, in this order
SMS = 132  # kNumSMs
BLOCK_G = 64  # kBlockG: sources per CTA of the EXACT fold
FAST_SRC = 8  # kFastSrc: sources per CTA of graph_dense_fast_kernel

# --------------------------------------------------------------------------- CPU: what a call launches

EXACT_RK4, EXACT_SEMI = "graph_dense_kernel<true, true>", "graph_dense_kernel<true, false>"
WORLD_RK4 = "graph_dense_world_kernel<true, 1024, 512, 1, 2, 2, false"
WORLD_SEMI = "graph_dense_world_kernel<false, 1024, 512, 1, 2, 2, false"
DENSE_SPLIT = "graph_dense_fast_kernel<true, true, 1024>"
DENSE_FAST = "graph_dense_fast_kernel<true, false, 256>"
DENSE_SEMI = "graph_dense_fast_kernel<false, false, 256>"
FILL, WAIT, PUSH = "peer_fill_kernel", "peer_wait_kernel", "peer_push_kernel"


def call_launches(T, peer):
    """kernel_launches of one call of T ticks: fold + body per tick; with a window, the fill and the first wait, then
    fold + body + push per tick (the NCCL all-gathers are not kernels the library counts)."""
    return 2 + 3 * T if peer else 2 * T


def fold_kernel(math, integ, N, rows=None, cfg=1):
    """The kernel launch_graph_force(dense=true) picks for one world of N bodies folding `rows` sources (B200_GRAPH_CFG
    = cfg).  Returns (name prefix, CTAs)."""
    rows = N if rows is None else rows
    rk4 = integ == "rk4"
    if math == "exact" or cfg == 0:
        return ("graph_dense_kernel<" + ("true" if math == "exact" else "false") + (", true>" if rk4 else ", false>"),
                -(-rows // BLOCK_G))
    if cfg == 1 and 64 <= N <= 1024:
        items2 = -(-rows // 2) * (3 if rk4 else 1)  # one world: CTAs until a CTA keeps four warps busy
        return (WORLD_RK4 if rk4 else WORLD_SEMI), max(1, min(SMS, -(-items2 // 4)))
    gridf = -(-rows // FAST_SRC)
    if not rk4:
        return DENSE_SEMI, gridf
    return (DENSE_SPLIT if cfg == 2 or (cfg == 1 and gridf < 3 * SMS) else DENSE_FAST), gridf


def call_kernels(math, integ, N, T, peer):
    """The kernel name prefixes of one call, in launch order."""
    fold = fold_kernel(math, integ, N)[0]
    tick = [fold, "body_"] + ([PUSH] if peer else [])
    return ([FILL, WAIT] if peer else []) + tick * T


def test_restatement_on_hand_worked_cases():
    assert [call_launches(T, False) for T in CALLS] == [2, 4, 6]
    assert [call_launches(T, True) for T in CALLS] == [5, 8, 11]
    assert call_kernels("fast", "rk4", 96, 2, True) == [FILL, WAIT, WORLD_RK4, "body_", PUSH, WORLD_RK4, "body_", PUSH]
    assert call_kernels("exact", "semi_implicit", 7, 1, False) == [EXACT_SEMI, "body_"]
    # EXACT: tiles of 64 sources
    assert fold_kernel("exact", "rk4", 64) == (EXACT_RK4, 1)
    assert fold_kernel("exact", "rk4", 65) == (EXACT_RK4, 2)
    assert fold_kernel("exact", "semi_implicit", 3161) == (EXACT_SEMI, 50)
    # FAST: the world-resident kernel for 64 <= N <= 1024 (at N = 1024, 512 pairs x 3 slots over 4 warps: 384 CTAs,
    # capped at one per SM)
    assert fold_kernel("fast", "rk4", 63)[0] == DENSE_SPLIT
    assert fold_kernel("fast", "rk4", 64) == (WORLD_RK4, 24)
    assert fold_kernel("fast", "rk4", 1024) == (WORLD_RK4, 132)
    assert fold_kernel("fast", "rk4", 1025) == (DENSE_SPLIT, 129)
    assert fold_kernel("fast", "semi_implicit", 65) == (WORLD_SEMI, 9)
    # split while ceil(N / 8) < 396
    assert fold_kernel("fast", "rk4", 3160) == (DENSE_SPLIT, 395)
    assert fold_kernel("fast", "rk4", 3161) == (DENSE_FAST, 396)
    assert fold_kernel("fast", "semi_implicit", 3161) == (DENSE_SEMI, 396)
    assert fold_kernel("fast", "semi_implicit", 2) == (DENSE_SEMI, 1)
    # the route switch: B200_GRAPH_CFG=2 always splits, 0 takes the generic tiles
    assert fold_kernel("fast", "rk4", 5000, cfg=2)[0] == DENSE_SPLIT
    assert fold_kernel("fast", "rk4", 96, cfg=0) == ("graph_dense_kernel<false, true>", 2)


# --------------------------------------------------------------------------- the GPU cases

# key: (N, graph kind, integrator, const gravity + body thrust after the edge-fold)
CASES = {
    "2-soft-rk4": (2, "softened", "rk4", False),
    "3-newton-semi": (3, "newton", "semi_implicit", False),
    "32-soft-rk4-extra": (32, "softened", "rk4", True),
    "33-soft-semi": (33, "softened", "semi_implicit", False),
    "63-newton-rk4": (63, "newton", "rk4", False),
    "64-soft-rk4": (64, "softened", "rk4", False),
    "65-soft-semi-extra": (65, "softened", "semi_implicit", True),
    "1023-newton-rk4-extra": (1023, "newton", "rk4", True),
    "1024-soft-rk4-bench": (1024, "softened", "rk4", False),
    "1025-soft-rk4": (1025, "softened", "rk4", False),
    "3161-soft-rk4": (3161, "softened", "rk4", False),
}
MATHS = ("exact", "fast")
ROUTES = ("nccl", "peer")


def test_gpu_cases_reach_every_boundary():
    """The case list reaches both sides of every boundary of the fold choice, both kinds, both integrators and the
    lists with effectors after the edge-fold, in both math modes."""
    got = {(m, fold_kernel(m, CASES[k][2], CASES[k][0])[0]) for k in CASES for m in MATHS}
    assert got >= {("exact", EXACT_RK4), ("exact", EXACT_SEMI), ("fast", WORLD_RK4), ("fast", WORLD_SEMI),
                   ("fast", DENSE_SPLIT), ("fast", DENSE_FAST), ("fast", DENSE_SEMI)}
    Ns = {c[0] for c in CASES.values()}
    assert {2, 3, 32, 33, 63, 64, 65, 1023, 1024, 1025} <= Ns and max(Ns) >= 3161
    # EXACT: one tile and two; FAST past 1024: split below 396 CTAs and unsplit at exactly 396
    assert {fold_kernel("exact", "rk4", N)[1] for N in (64, 65)} == {1, 2}
    assert any(fold_kernel("fast", "rk4", N)[0] == DENSE_SPLIT for N in Ns if N > 1024)
    assert any(-(-N // FAST_SRC) == 3 * SMS for N in Ns)
    assert {c[1] for c in CASES.values()} == {"softened", "newton"}
    assert {c[2] for c in CASES.values()} == {"rk4", "semi_implicit"}
    assert {(c[2], c[3]) for c in CASES.values()} >= {("rk4", True), ("semi_implicit", True)}
    # the plain two-launch reference needs both route switches for N <= 32 (small-world kernel) and one above
    assert any(c[0] <= 32 for c in CASES.values()) and any(c[0] > 32 for c in CASES.values())


def _edges(N):
    import elodin_b200 as el

    return el.all_pairs_edges(N)


def setup_case(key, O=None):
    """(start = (pos, vel, ine), dt, S, library effectors, columns, oracle effectors or None)."""
    import elodin_b200 as el

    N, kind, integ, extra = CASES[key]
    edges = _edges(N)
    seed = 7000 + N + (1 if kind == "newton" else 0)
    if N == 1024:
        dt = BENCH_DT
        pos, vel, ine, k, soft, S = nbody_world(seed, 1, N, dt, size=1e11, speed=1e3)
    else:
        dt = DT
        pos, vel, ine, k, soft, S = nbody_world(seed, 1, N, dt, edges=edges if kind == "newton" else None, kind=kind)
    if kind == "newton":
        ge = [el.GravityEdges("newton", G=k, edges=edges)]
        oe = [O.Effector(O.EFF_GRAVITY_EDGES_NEWTON, p=(k,), edges=edges)] if O else None
    else:
        ge = [el.GravityEdges("softened", k_squared=k, softening=soft, edges=edges)]
        oe = [O.Effector(O.EFF_GRAVITY_EDGES_SOFTENED, p=(k, soft), edges=edges)] if O else None
    cols = {}
    if extra:  # a const gravity and a body-frame thrust comparable to the edge-fold gravity
        a = float(np.median(S))
        thrust = np.random.default_rng(seed).uniform(0.5, 2.0, (1, N, 1)) * ine[..., 6:7] * a
        ge += [el.GravityConst((0.0, 0.3 * a, -a)), el.ThrustBody((-1.0, 0.0, 0.0), "thrust")]
        cols["thrust"] = thrust
        if O:
            oe += [O.Effector(O.EFF_GRAVITY_CONST, p=(0.0, 0.3 * a, -a)), O.Effector(O.EFF_THRUST_BODY, p=(-1.0, 0.0, 0.0), column=thrust)]
    return (pos, vel, ine), dt, S, ge, cols, oe


def open_case(key, math, **kw):
    import elodin_b200 as el

    start, dt, _, ge, cols, _ = setup_case(key)
    ex = el.B200Exec(CASES[key][0], 1, dt, None, ge, CASES[key][2], math, device=0, **kw)
    ex.set_state(*start, **cols)
    return ex


def state(ex):
    from elodin_b200.executor import FORCE, WORLD_ACCEL, WORLD_POS, WORLD_VEL

    ex.sync()
    return tuple(ex.download(c) for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE))


STATE_NAMES = ("pos", "vel", "accel", "force")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def assert_same_bits(got, want, what):
    for name, a, b in zip(STATE_NAMES, got, want):
        bad = np.argwhere(_bits(a) != _bits(b))
        assert bad.size == 0, (f"{what} {name}: {len(bad)} values differ, first at {tuple(bad[0])}: {a[tuple(bad[0])]!r} "
                               f"vs {b[tuple(bad[0])]!r}")


# --------------------------------------------------------------------------- child processes


def run_in_child(fn, args, out, settings=()):
    """Run this module's `fn`(**args) in a fresh child process with every inherited B200_* switch removed and
    `settings` ("B200_X=v" each) set; it returns a dict of arrays, which the child saves to `out` and this loads.
    (tests.util.run_child sets one switch; the two-launch reference needs two.)"""
    env = {k: v for k, v in os.environ.items() if not k.startswith("B200_")}
    for s in settings:
        key, val = s.split("=")
        env[key] = val
    code = ("import json, sys; import numpy as np; from tests.test_row_shards import _child_main; "
            "_child_main(sys.argv[1], sys.argv[2], json.loads(sys.argv[3]))")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    argv = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, fn, out, json.dumps(args)]
    p = subprocess.run(argv, cwd=root, env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, f"{fn} {' '.join(settings) or '(default)'} child failed ({p.returncode}):\n{p.stderr[-6000:]}"
    with np.load(out, allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


def _child_main(fn, out, args):
    # torch first: the library binds the libnccl.so.2 the process already loaded, and torch needs its own copy
    import torch  # noqa: F401

    res = globals()[fn](**args)
    np.savez(out, **res)


def _comm():
    from elodin_b200.sharding import Comm

    return Comm(Comm.unique_id(), 1, 0, 0)


def _named_call(comm, key, math, route, n, attempts=3):
    """Kernel names (library kernels only, in launch order) and the launch count of one call of n ticks on a fresh
    handle; an attempt counts when the profiler saw as many launches as the library counted."""
    from tests.util import launched_kernels

    for _ in range(attempts):
        ex = open_case(key, math)
        try:
            if route == "peer":
                comm.peer_attach(ex)
            n0 = ex.timings()["kernel_launches"]
            _, names = launched_kernels(lambda: (comm.step_row_sharded(ex, n), ex.sync()))
            launches = ex.timings()["kernel_launches"] - n0
            if route == "peer":
                comm.peer_detach()
        finally:
            ex.close()
        names = [s for s in names if not s.startswith(("Memcpy", "Memset", "nccl"))]
        if len(names) == launches:
            break
    return names, launches


def child_cases(keys):
    """Every case: kernel names of a 2-tick call per math and exchange; then calls of CALLS ticks, the state and the
    launch count after each."""
    res = {}
    comm = _comm()
    try:
        for key in keys:
            for math in MATHS:
                for route in ROUTES:
                    tag = f"{key}|{math}|{route}"
                    names, launches = _named_call(comm, key, math, route, 2)
                    res[f"{tag}|names"] = np.array(names)
                    res[f"{tag}|named_launches"] = np.array(launches)
                    ex = open_case(key, math)
                    try:
                        if route == "peer":
                            comm.peer_attach(ex)
                        counts, ticks = [], []
                        for c, n in enumerate(CALLS):
                            n0 = ex.timings()["kernel_launches"]
                            comm.step_row_sharded(ex, n)
                            counts.append(ex.timings()["kernel_launches"] - n0)
                            ticks.append(ex.tick)
                            for name, a in zip(STATE_NAMES, state(ex)):
                                res[f"{tag}|{c}|{name}"] = a
                        res[f"{tag}|launches"] = np.array(counts)
                        res[f"{tag}|ticks"] = np.array(ticks)
                        if route == "peer":
                            comm.peer_detach()
                    finally:
                        ex.close()
    finally:
        comm.close()
    return res


def child_plain(keys):
    """The two-launch plain route (run with B200_NBODY_FUSED=0 B200_SMALL_WORLD=0): step() of CALLS ticks, FAST."""
    res = {}
    for key in keys:
        ex = open_case(key, "fast")
        try:
            for c, n in enumerate(CALLS):
                n0 = ex.timings()["kernel_launches"]
                ex.step(n)
                res[f"{key}|{c}|launches"] = np.array(ex.timings()["kernel_launches"] - n0)
                for name, a in zip(STATE_NAMES, state(ex)):
                    res[f"{key}|{c}|{name}"] = a
        finally:
            ex.close()
    return res


TWO_LAUNCH = ("B200_NBODY_FUSED=0", "B200_SMALL_WORLD=0")


@pytest.fixture(scope="module")
def recorded(tmp_path_factory):
    d = tmp_path_factory.mktemp("row_shards")
    keys = list(CASES)
    rows = run_in_child("child_cases", {"keys": keys}, str(d / "rows.npz"))
    plain = run_in_child("child_plain", {"keys": keys}, str(d / "plain.npz"), TWO_LAUNCH)
    return rows, plain


def _threads(O):
    return max(1, min(O.max_threads(), os.cpu_count() or 1))


def oracle_states(O, start, effs, integ, dt, calls):
    """The oracle's (pos, vel, accel, force) after each call of `calls` ticks."""
    w = O.World(*start)
    out = []
    for n in calls:
        (w.rk4 if integ == "rk4" else w.semi_implicit)(dt, n, effs, threads=_threads(O))
        out.append(tuple(a.copy() for a in (w.pos, w.vel, w.accel, w.force)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(CASES))
def test_both_exchanges_match_the_oracle(oracle, recorded, key):
    rows, plain = recorded
    N, kind, integ, extra = CASES[key]
    start, dt, S, _, _, oe = setup_case(key, oracle)
    want = oracle_states(oracle, start, oe, integ, dt, CALLS)
    for math in MATHS:
        fold = fold_kernel(math, integ, N)[0]
        got = {}
        for route in ROUTES:
            tag = f"{key}|{math}|{route}"
            peer = route == "peer"
            # which kernels ran, in order: the restated list, the fold kernel by name
            names, launches = list(rows[f"{tag}|names"]), int(rows[f"{tag}|named_launches"])
            assert launches == call_launches(2, peer), f"{tag}: {launches} launches in a 2-tick call"
            assert len(names) == launches, f"{tag}: the profiler saw {len(names)} of {launches} launches: {names}"
            expected = call_kernels(math, integ, N, 2, peer)
            for i, (nm, e) in enumerate(zip(names, expected)):
                assert nm.startswith(e), f"{tag}: launch {i} is {nm}, expected {e}... (all: {names})"
            assert list(rows[f"{tag}|launches"]) == [call_launches(n, peer) for n in CALLS], tag
            assert list(rows[f"{tag}|ticks"]) == list(itertools.accumulate(CALLS)), tag
            got[route] = [tuple(rows[f"{tag}|{c}|{nm}"] for nm in STATE_NAMES) for c in range(len(CALLS))]
        for c, T in enumerate(itertools.accumulate(CALLS)):
            what = f"{key} {math} after call {c} ({T} ticks)"
            assert_same_bits(got["peer"][c], got["nccl"][c], f"{what}: peer vs NCCL")
            if math == "exact":
                assert_same_bits(got["nccl"][c], want[c], f"{what}: vs the oracle")
                continue
            ref = tuple(plain[f"{key}|{c}|{nm}"] for nm in STATE_NAMES)
            assert int(plain[f"{key}|{c}|launches"]) == 2 * CALLS[c], f"{what}: the plain reference is not two-launch"
            assert_same_bits(got["nccl"][c], ref, f"{what}: vs the two-launch plain step")
            assert_nbody_close(got["nccl"][c], want[c], start, dt, T, S, what=f"{what}: vs the oracle")


# --------------------------------------------------------------------------- mixed schedules


SCHED_KEYS = {"40-soft-rk4": (40, "softened", "rk4", False), "96-soft-rk4": (96, "softened", "rk4", False)}

# ("rows", n) row-sharded call; ("step", n) plain step; ("set_state", seed); ("invoke", n) invoke_batch of the current
# state; ("reset",) trajectory_reset; ("stream", "side" | None) a torch side stream / the handle's own
SCHEDULE = [("stream", "side"), ("rows", 1), ("step", 1), ("rows", 2), ("step", 2), ("rows", 3), ("stream", None),
            ("reset",), ("rows", 2), ("set_state", 1), ("step", 3), ("rows", 1), ("invoke", 2), ("rows", 2),
            ("stream", "side"), ("step", 1), ("rows", 3), ("invoke", 1), ("rows", 1)]


def test_schedule_reaches_every_mix():
    """Odd plain steps (the one-launch tick swaps the ping-pong planes), calls that start at odd ticks_done, a reset,
    an upload and invoke_batch each followed by a row-sharded call, and calls on a side stream."""
    done, odd_start, after = 0, 0, set()
    prev, stream = None, None
    side_rows = 0
    for op in SCHEDULE:
        if op[0] == "stream":
            stream = op[1]
            continue
        if op[0] == "rows":
            odd_start += done % 2
            side_rows += stream == "side"
            after.add(prev)
        if op[0] in ("rows", "step", "invoke"):
            done += op[1]
        if op[0] == "reset":
            done = 0
        prev = op[0]
    assert odd_start >= 2 and side_rows >= 2
    assert after >= {None, "step", "reset", "invoke"}
    assert any(op[0] == "step" and op[1] % 2 for op in SCHEDULE) and any(op[0] == "step" and op[1] % 2 == 0 for op in SCHEDULE)
    assert ("set_state", 1) in SCHEDULE


def _sched_world(key, seed=0):
    """((pos, vel, ine), k, soft, S) of a schedule world; seed > 0: new positions and velocities of the same bodies
    (inertia and gravity constant stay those of seed 0, which the handle keeps)."""
    N = SCHED_KEYS[key][0]
    pos, vel, ine, k, soft, S = nbody_world(9100 + N, 1, N, DT)
    if seed:
        pos, vel = nbody_world(9100 + N + 31 * seed, 1, N, DT)[:2]
        S = k * nbody_pair_scale(pos, ine, 1.0, soft)
    return (pos, vel, ine), k, soft, S


def child_schedules():
    res = {}
    for key in SCHED_KEYS:
        for math in MATHS:
            for route in ROUTES:
                res.update({f"{key}|{math}|{route}|{k}": v for k, v in _schedule_run(key, math, route).items()})
    return res


def _schedule_run(key, math, route):
    import torch

    import elodin_b200 as el
    from elodin_b200.executor import FORCE, INERTIA, WORLD_ACCEL, WORLD_POS, WORLD_VEL

    N = SCHED_KEYS[key][0]
    (pos, vel, ine), k, soft, _ = _sched_world(key)
    res = {}
    comm = _comm()
    side = torch.cuda.Stream()
    ex = el.B200Exec(N, 1, DT, None, [el.GravityEdges("softened", k_squared=k, softening=soft, edges=_edges(N))], "rk4",
                     math, device=0, trajectory_every=1, trajectory_capacity=4)
    try:
        ex.set_state(pos, vel, ine)
        if route == "peer":
            comm.peer_attach(ex)
        for i, op in enumerate(SCHEDULE):
            n0 = ex.timings()["kernel_launches"]
            if op[0] == "stream":
                ex.set_stream(side.cuda_stream if op[1] else None)
                continue
            if op[0] == "rows":
                comm.step_row_sharded(ex, op[1])
            elif op[0] == "step":
                ex.step(op[1])
            elif op[0] == "reset":
                ex.trajectory_reset()
            elif op[0] == "set_state":
                (p, v, I), _, _, _ = _sched_world(key, op[1])
                ex.set_state(p, v, I)
            elif op[0] == "invoke":
                p, v, _, _ = state(ex)
                t = {el.component_id("tick"): np.array([ex.tick], dtype=np.uint64), FORCE: np.zeros((1, N, 6)),
                     INERTIA: ine, WORLD_POS: p, WORLD_ACCEL: np.zeros((1, N, 6)),
                     el.component_id("simulation_time_step"): np.array([DT]), WORLD_VEL: v}
                res[f"{i}|in_pos"], res[f"{i}|in_vel"] = p, v
                ex.invoke_batch([t[c] for c in ex.input_ids], op[1])
            res[f"{i}|launches"] = np.array(ex.timings()["kernel_launches"] - n0)
            res[f"{i}|tick"] = np.array(ex.tick)
            for name, a in zip(STATE_NAMES, state(ex)):
                res[f"{i}|{name}"] = a
        if route == "peer":
            assert comm.peer_attached
            comm.peer_detach()
    finally:
        ex.close()
        comm.close()
    return res


@pytest.fixture(scope="module")
def schedules(tmp_path_factory):
    res = run_in_child("child_schedules", {}, str(tmp_path_factory.mktemp("row_sched") / "sched.npz"))
    out = {}
    for key, math, route in itertools.product(SCHED_KEYS, MATHS, ROUTES):
        tag = f"{key}|{math}|{route}|"
        out[(key, math, route)] = {k[len(tag):]: v for k, v in res.items() if k.startswith(tag)}
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("math", MATHS)
@pytest.mark.parametrize("key", list(SCHED_KEYS))
def test_schedules_mixing_row_shards_with_other_entries(oracle, schedules, key, math):
    O = oracle
    N = SCHED_KEYS[key][0]
    (pos, vel, ine), k, soft, S = _sched_world(key)
    effs = [O.Effector(O.EFF_GRAVITY_EDGES_SOFTENED, p=(k, soft), edges=_edges(N))]
    nccl, peer = schedules[(key, math, "nccl")], schedules[(key, math, "peer")]
    start, T, tick = (pos, vel, ine), 0, 0
    w = O.World(pos, vel, ine)
    for i, op in enumerate(SCHEDULE):
        if op[0] == "stream":
            continue
        what = f"{key} {math} op {i} {op}"
        got = tuple(peer[f"{i}|{nm}"] for nm in STATE_NAMES)
        assert_same_bits(got, tuple(nccl[f"{i}|{nm}"] for nm in STATE_NAMES), f"{what}: peer vs NCCL")
        if op[0] == "rows":
            assert int(peer[f"{i}|launches"]) == call_launches(op[1], True), what
            assert int(nccl[f"{i}|launches"]) == call_launches(op[1], False), what
        if op[0] == "set_state":
            (p, v, I), _, _, S = _sched_world(key, op[1])
            start, T, w = (p, v, I), 0, O.World(p, v, I)
        elif op[0] == "invoke":
            p, v = peer[f"{i}|in_pos"], peer[f"{i}|in_vel"]
            if math == "fast":  # a new segment from the state the handle held
                start, T, w = (p, v, ine), 0, O.World(p, v, ine)
                S = k * nbody_pair_scale(p, ine, 1.0, soft)
        if op[0] in ("rows", "step", "invoke"):
            w.rk4(DT, op[1], effs, threads=_threads(O))
            T += op[1]
            tick += op[1]
        assert int(peer[f"{i}|tick"]) == tick, what
        if op[0] in ("reset", "set_state") and T == 0:
            continue
        want = (w.pos, w.vel, w.accel, w.force)
        if math == "exact":
            assert_same_bits(got, want, f"{what}: vs the oracle")
        elif T:
            assert_nbody_close(got, want, start, DT, T, S, what=f"{what}: vs the oracle")


# --------------------------------------------------------------------------- the trajectory ring

RING_CALLS = (1, 1, 2, 3, 1, 2)  # calls start at ticks 0, 1, 2, 4, 7, 8: every phase of every 2 and every 3


def test_ring_calls_start_at_every_phase():
    starts = [0] + list(itertools.accumulate(RING_CALLS))[:-1]
    for every in (2, 3):
        assert {s % every for s in starts} == set(range(every))
    assert sum(RING_CALLS) // 3 > 2  # more samples than the ring of capacity 2 holds: it wraps


RING_GRID = list(itertools.product(MATHS, (1, 2, 3), (2, 5), (False, True)))  # math, every, capacity, 25 planes


def child_ring():
    """Run with the two-launch switches: the ring of row-sharded calls (both exchanges) and of plain steps of the same
    tick counts, at every sampling interval 1..3, capacities 2 and 5, 13 and 25 planes."""
    import elodin_b200 as el

    key = "96-soft-rk4"
    N = SCHED_KEYS[key][0]
    (pos, vel, ine), k, soft, _ = _sched_world(key)
    res = {}
    comm = _comm()
    try:
        for math, every, cap, full in RING_GRID:
            for route in ("plain", "nccl", "peer"):
                ex = el.B200Exec(N, 1, DT, None, [el.GravityEdges("softened", k_squared=k, softening=soft, edges=_edges(N))],
                                 "rk4", math, device=0, trajectory_every=every, trajectory_capacity=cap, trajectory_full=full)
                try:
                    ex.set_state(pos, vel, ine)
                    if route == "peer":
                        comm.peer_attach(ex)
                    for n in RING_CALLS:
                        if route == "plain":
                            ex.step(n)
                        else:
                            comm.step_row_sharded(ex, n)
                    tag = f"{math}|{every}|{cap}|{int(full)}|{route}"
                    res[f"{tag}|ring"] = ex.trajectory()
                    res[f"{tag}|len"] = np.array(ex.trajectory_len())
                    if route == "peer":
                        comm.peer_detach()
                finally:
                    ex.close()
    finally:
        comm.close()
    return res


@pytest.mark.gpu
def test_ring_of_row_sharded_ticks_equals_the_plain_ring(tmp_path):
    res = run_in_child("child_ring", {}, str(tmp_path / "ring.npz"), TWO_LAUNCH)
    for math, every, cap, full in RING_GRID:
        base = f"{math}|{every}|{cap}|{int(full)}"
        want = res[f"{base}|plain|ring"]
        assert int(res[f"{base}|plain|len"]) == min(sum(RING_CALLS) // every, cap)
        assert want.shape[0] == min(sum(RING_CALLS) // every, cap)
        assert np.all(np.isfinite(want)), base
        for route in ("nccl", "peer"):
            got = res[f"{base}|{route}|ring"]
            assert got.shape == want.shape, f"{base} {route}"
            bad = np.argwhere(np.any(_bits(got) != _bits(want), axis=-1))
            assert bad.size == 0, f"{math} every {every} capacity {cap} full {full} {route}: {len(bad)} ring rows differ, first {tuple(bad[0])}"


# --------------------------------------------------------------------------- the window's life cycle, refusals


def child_life_cycle():
    """Launch counts and states of the window's life cycle (see test_window_life_cycle)."""
    key = "96-soft-rk4"
    res = {}

    def mk():
        import elodin_b200 as el

        (pos, vel, ine), k, soft, _ = _sched_world(key)
        ex = el.B200Exec(96, 1, DT, None, [el.GravityEdges("softened", k_squared=k, softening=soft, edges=_edges(96))], "rk4",
                         "fast", device=0)
        ex.set_state(pos, vel, ine)
        return ex

    def rows(comm, ex, n, tag):
        n0 = ex.timings()["kernel_launches"]
        comm.step_row_sharded(ex, n)
        res[f"{tag}|launches"] = np.array(ex.timings()["kernel_launches"] - n0)
        for name, a in zip(STATE_NAMES, state(ex)):
            res[f"{tag}|{name}"] = a

    comm = _comm()
    try:
        # reference: the NCCL route, calls of 2, 1 and 3 ticks
        ref = mk()
        for c, n in enumerate((2, 1, 3)):
            rows(comm, ref, n, f"ref{c}")
        ref.close()
        # attach to A, step B: B takes the NCCL route, A keeps the window
        a, b = mk(), mk()
        comm.peer_attach(a)
        rows(comm, b, 2, "b0")
        rows(comm, a, 2, "a0")
        # detach: A takes the NCCL route; re-attach after ticks: the window again
        comm.peer_detach()
        res["attached_after_detach"] = np.array(int(comm.peer_attached))
        rows(comm, a, 1, "a1")
        comm.peer_attach(a)
        rows(comm, a, 3, "a2")
        b.close()
        # destroy the attached handle, create one of the same shape: the serial check sends it to the NCCL route
        addr = a._h.value
        a.close()
        res["attached_after_close"] = np.array(int(comm.peer_attached))
        c = mk()
        res["address_reused"] = np.array(int(c._h.value == addr))
        rows(comm, c, 2, "c0")
        # closing the communicator with a window attached detaches it; the handle stays usable
        comm.peer_attach(c)
        rows(comm, c, 1, "c1")
        comm.close()
        comm = None
        c.step(1)
        res["c_tick"] = np.array(c.tick)
        c.close()
        # B200_ROW_PEER (read once per process) is the caller's; reported here for the parent
        res["row_peer"] = np.array(int(os.environ.get("B200_ROW_PEER", "1")))
        comm = _comm()
        d = mk()
        comm.peer_attach(d)
        rows(comm, d, 2, "d0")
        comm.peer_detach()
        d.close()
    finally:
        if comm is not None:
            comm.close()
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("setting", ["default", "B200_ROW_PEER=0"])
def test_window_life_cycle(setting, tmp_path):
    res = run_in_child("child_life_cycle", {}, str(tmp_path / "life.npz"), () if setting == "default" else (setting,))
    peer_on = setting == "default"
    L = lambda tag: int(res[f"{tag}|launches"])
    st = lambda tag: tuple(res[f"{tag}|{nm}"] for nm in STATE_NAMES)
    assert [L(f"ref{c}") for c in range(3)] == [call_launches(n, False) for n in (2, 1, 3)]
    assert L("b0") == call_launches(2, False), "a handle the window is not attached to must take the NCCL route"
    assert L("a0") == call_launches(2, peer_on)
    assert int(res["attached_after_detach"]) == 0
    assert L("a1") == call_launches(1, False)
    assert L("a2") == call_launches(3, peer_on)
    assert int(res["attached_after_close"]) == 1  # the window outlives its handle until detach
    assert L("c0") == call_launches(2, False), (f"a new handle (address reused: {bool(res['address_reused'])}) must not "
                                                 "use the window of a destroyed one")
    assert L("c1") == call_launches(1, peer_on)
    assert L("d0") == call_launches(2, peer_on)
    assert int(res["c_tick"]) == 4
    # the same calls give the same bits whatever the exchange: B and D are at the reference's first call, A and C
    # after 2, 1 (+3) ticks
    assert_same_bits(st("b0"), st("ref0"), "B after attaching A")
    assert_same_bits(st("a0"), st("ref0"), "A through the window")
    assert_same_bits(st("a1"), st("ref1"), "A after detach")
    assert_same_bits(st("a2"), st("ref2"), "A after re-attach")
    assert_same_bits(st("c0"), st("ref0"), "a new handle of the same shape")
    assert_same_bits(st("d0"), st("ref0"), "a handle attached to a new communicator")


def child_refusals():
    """Every refusal: the error code, and the handle's tick and state before, after, and after one more step."""
    import elodin_b200 as el
    from elodin_b200 import _lib

    res = {}
    comm = _comm()
    N = 8
    pos, vel, ine, k, soft, _ = nbody_world(8800, 2, N, DT)
    soft_all = lambda: el.GravityEdges("softened", k_squared=k, softening=soft, edges=_edges(N))
    ring_edges = np.array([[i, (i + 1) % N] for i in range(N)], dtype=np.uint32)
    cb, sb = np.zeros((3, 3)), np.zeros((3, 3))
    cb[0, 0], cb[2, 0] = 1.0, -4.8e-4
    cases = {
        "two_worlds": (2, [soft_all()]),
        "csr_graph": (1, [el.GravityEdges("softened", k_squared=k, softening=soft, edges=ring_edges)]),
        "no_graph": (1, [el.GravityConst()]),
        "egm08_beside_graph": (1, [soft_all(), el.GravityEGM08(cb, sb, 2)]),
    }
    try:
        for name, (M, effs) in cases.items():
            ex = el.B200Exec(N, M, DT, None, effs, "rk4", "exact", device=0)
            try:
                ex.set_state(pos[:M], vel[:M], ine[:M])
                ex.step(1)
                before, t0 = state(ex), ex.tick
                code = 0
                try:
                    comm.step_row_sharded(ex, 2)
                except _lib.B200Error as e:
                    code = int(e.code)
                res[f"{name}|code"] = np.array(code)
                res[f"{name}|tick"] = np.array([t0, ex.tick])
                after = state(ex)
                res[f"{name}|unchanged"] = np.array(int(all(np.array_equal(_bits(a), _bits(b)) for a, b in zip(before, after))))
                ex.step(1)
                res[f"{name}|tick_after_step"] = np.array(ex.tick)
                res[f"{name}|finite"] = np.array(int(all(np.all(np.isfinite(a)) for a in state(ex))))
            finally:
                ex.close()
        # a sharded-quantile round after a row-sharded call: refused (the rows changed since begin); without the call
        # in between, the rounds run to the end
        for with_rows in (False, True):
            ex = el.B200Exec(N, 1, DT, None, [soft_all()], "rk4", "exact", device=0)
            try:
                ex.set_state(pos[:1], vel[:1], ine[:1])
                q = np.array([0.5])
                mx = ex.sharded_quantiles_begin(q, "state")
                if with_rows:
                    comm.step_row_sharded(ex, 1)
                partial = np.zeros(max(mx // 4, 1), dtype=np.uint32)
                code, nb = 0, 0
                try:
                    while True:
                        nb = ex.sharded_quantiles_round(partial.copy() if nb else None, nb, partial)
                        if nb == 0:
                            table = ex.sharded_quantiles_end()
                            res[f"quantiles{int(with_rows)}|table"] = table
                            res[f"quantiles{int(with_rows)}|want"] = ex.state_quantiles(q)
                            break
                except _lib.B200Error as e:
                    code = int(e.code)
                res[f"quantiles{int(with_rows)}|code"] = np.array(code)
                res[f"quantiles{int(with_rows)}|tick"] = np.array(ex.tick)
            finally:
                ex.close()
    finally:
        comm.close()
    return res


@pytest.mark.gpu
def test_refusals_leave_the_handle_usable(tmp_path):
    from elodin_b200 import _lib

    res = run_in_child("child_refusals", {}, str(tmp_path / "refusals.npz"))
    for name in ("two_worlds", "csr_graph", "no_graph", "egm08_beside_graph"):
        assert int(res[f"{name}|code"]) == _lib.ERR_UNSUPPORTED, name
        t0, t1 = res[f"{name}|tick"]
        assert t0 == t1 == 1, f"{name}: tick {t0} -> {t1}"
        assert int(res[f"{name}|unchanged"]) == 1, f"{name}: the refused call changed the state"
        assert int(res[f"{name}|tick_after_step"]) == 2 and int(res[f"{name}|finite"]) == 1, name
    assert int(res["quantiles0|code"]) == 0
    assert np.array_equal(_bits(res["quantiles0|table"]), _bits(res["quantiles0|want"]))
    assert int(res["quantiles1|code"]) != 0, "a sharded-quantile round after a row-sharded call must be refused"
    assert int(res["quantiles1|tick"]) == 1


# --------------------------------------------------------------------------- CPU: a model of the peer window
#
# Each rank runs one program: the ops its stream executes, in order, at the granularity of the kernels' memory
# events.  Shared memory holds every rank's window: X[rank][half][owner] (the owner's rows in that half, tagged with
# the world state they belong to: a counter advanced by every tick and every upload) and F[rank][src] (the delivery
# counter rank src releases into rank's window).  Ops:
#   ("st", addr, v)    a store (the fill's half write, a row store, a counter release, a window's zeroing)
#   ("max", addr, v)   the fill's atomicMax on a counter
#   ("wait", addr, v)  an acquire spin: enabled once mem[addr] >= v
#   ("read", addr, v)  the gravity read of one owner's rows: it must see state v, or the protocol failed
#   ("arrive", i) / ("gather", i)  a collective (the last tick's all-gather, detach / attach): "gather" is enabled once
#                      every rank has passed its "arrive" of the same collective
# A tick's rows are tagged with the state they were computed from, so a stale read cannot hide behind equal values.

EMPTY = -1
FAULTS = ("push_after_wait", "parity", "fill_without_max", "wait_value", "release_before_rows")


def rank_program(r, R, schedule, rule="window", fault=None):
    """Rank r's ops for `schedule` (items: ("rows", n) a row-sharded call, ("step", n) plain ticks, ("upload",),
    ("reset",) trajectory_reset, ("reattach",) detach + attach).  rule "window": the window's own tick count keys the
    protocol; "ticks_done": the handle's (reset by trajectory_reset)."""
    ops, ver, ticks_done, seq, coll = [], 0, 0, 0, 0
    for item in schedule:
        kind = item[0]
        if kind == "step":
            ver += item[1]
            ticks_done += item[1]
        elif kind == "upload":
            ver += 1
        elif kind == "reset":
            ticks_done = 0
        elif kind == "reattach":  # detach (barrier after unmapping), then attach: a zeroed window, exchanged collectively
            ops += [("arrive", coll), ("gather", coll)]
            ops += [("st", ("X", r, h, o), EMPTY) for h in (0, 1) for o in range(R)]
            ops += [("st", ("F", r, s), 0) for s in range(R)]
            ops += [("arrive", coll + 1), ("gather", coll + 1)]
            coll += 2
            seq = 0
        elif kind == "rows":
            n = item[1]
            K0 = seq if rule == "window" else ticks_done
            ops += [("st", ("X", r, K0 & 1, o), ver) for o in range(R)]  # fill: the local world into the current half
            if fault != "fill_without_max":  # raise the counters: plain ticks since the last call advanced the count
                ops += [("max", ("F", r, s), K0) for s in range(R)]
            ops += [("wait", ("F", r, s), K0) for s in range(R)]
            for t in range(n):
                K, last = K0 + t, t + 1 == n
                ops += [("read", ("X", r, K & 1, o), ver) for o in range(R)]  # gravity
                ver += 1  # the body kernel: this rank's rows of the next state
                half = (K if fault == "parity" else K + 1) & 1
                rows = [("st", ("X", d, half, r), ver) for d in range(R)]
                rel = [("st", ("F", d, r), K + 1) for d in range(R)]
                waits = [] if last else [("wait", ("F", r, s), K if fault == "wait_value" else K + 1) for s in range(R)]
                if fault == "push_after_wait":
                    ops += waits + rows + rel
                elif fault == "release_before_rows":
                    ops += rel + rows + waits
                else:
                    ops += rows + rel + waits
            ops += [("arrive", coll), ("gather", coll)]  # the last tick's all-gather: every rank holds the whole world
            coll += 1
            ticks_done += n
            seq += n
        else:
            raise KeyError(kind)
    return ops


class Model:
    def __init__(self, R, schedule, rule="window", fault=None):
        self.R = R
        self.progs = [rank_program(r, R, schedule, rule, fault) for r in range(R)]
        addrs = [("X", r, h, o) for r in range(R) for h in (0, 1) for o in range(R)] + [("F", r, s) for r in range(R) for s in range(R)]
        self.index = {a: i for i, a in enumerate(addrs)}
        self.mem0 = tuple(EMPTY if a[0] == "X" else 0 for a in addrs)
        self.arrive = [{op[1]: k for k, op in enumerate(p) if op[0] == "arrive"} for p in self.progs]

    def enabled(self, pcs, mem, r):
        p, pc = self.progs[r], pcs[r]
        if pc >= len(p):
            return False
        op = p[pc]
        if op[0] == "wait":
            return mem[self.index[op[1]]] >= op[2]
        if op[0] == "gather":
            return all(pcs[s] > self.arrive[s][op[1]] for s in range(self.R))
        return True

    def step(self, pcs, mem, r):
        """Run rank r's next op: (pcs, mem, failure or None)."""
        op = self.progs[r][pcs[r]]
        pcs = pcs[:r] + (pcs[r] + 1,) + pcs[r + 1:]
        if op[0] in ("st", "max"):
            i = self.index[op[1]]
            v = op[2] if op[0] == "st" else max(mem[i], op[2])
            mem = mem[:i] + (v,) + mem[i + 1:]
        elif op[0] == "read":
            got = mem[self.index[op[1]]]
            if got != op[2]:
                return pcs, mem, f"rank {r} read owner {op[1][3]}'s rows of state {got} from half {op[1][2]}, needed {op[2]}"
        return pcs, mem, None

    def done(self, pcs):
        return all(pc == len(p) for pc, p in zip(pcs, self.progs))

    def exhaustive(self, limit=3_000_000):
        """Every interleaving (DFS over the reachable states): None, or the first failure found (a stale read or a
        deadlock)."""
        start = (tuple(0 for _ in range(self.R)), self.mem0)
        seen, stack = {start}, [start]
        while stack:
            pcs, mem = stack.pop()
            moved = False
            for r in range(self.R):
                if not self.enabled(pcs, mem, r):
                    continue
                moved = True
                npcs, nmem, bad = self.step(pcs, mem, r)
                if bad:
                    return bad
                s = (npcs, nmem)
                if s not in seen:
                    seen.add(s)
                    stack.append(s)
            if not moved and not self.done(pcs):
                return f"deadlock at {pcs}"
            assert len(seen) < limit, "state space too large for an exhaustive search"
        return None

    def random_run(self, seed):
        """One adversarial interleaving: a random rank runs a random burst of ops (a rank that races ahead or stalls
        is what breaks a protocol).  None, or the failure."""
        rng = random.Random(seed)
        pcs, mem = tuple(0 for _ in range(self.R)), self.mem0
        while not self.done(pcs):
            ready = [r for r in range(self.R) if self.enabled(pcs, mem, r)]
            if not ready:
                return f"deadlock at {pcs}"
            r = rng.choice(ready)
            for _ in range(rng.choice((1, 1, 2, 3, 8, 40))):
                if not self.enabled(pcs, mem, r):
                    break
                pcs, mem, bad = self.step(pcs, mem, r)
                if bad:
                    return bad
        return None


# schedules between and around the calls: step, upload, trajectory_reset, detach / attach
MODEL_SCHEDULES = {
    "calls": [("rows", 2), ("rows", 3)],
    "reset": [("rows", 3), ("reset",), ("rows", 2)],
    "mixed": [("rows", 2), ("step", 1), ("rows", 1), ("upload",), ("rows", 2), ("reset",), ("step", 3), ("rows", 2)],
    "reattach": [("rows", 3), ("reattach",), ("step", 1), ("rows", 2), ("reset",), ("reattach",), ("rows", 2)],
}
RANDOM_RUNS = 300


@pytest.mark.parametrize("name", list(MODEL_SCHEDULES))
def test_peer_window_model_passes_with_the_window_count(name):
    sched = MODEL_SCHEDULES[name]
    assert Model(2, sched).exhaustive() is None
    for R in (3, 4):
        m = Model(R, sched)
        for seed in range(RANDOM_RUNS):
            bad = m.random_run(seed)
            assert bad is None, f"{R} ranks, seed {seed}: {bad}"


def test_peer_window_model_fails_on_the_ticks_done_rule_after_a_reset():
    """Keyed to ticks_done, the counters hold the old, larger counts after a trajectory reset: a wait passes before the
    peers' rows of its tick landed.  Without a reset the same rule passes; with one rank it cannot fail."""
    for name in ("reset", "mixed"):
        sched = MODEL_SCHEDULES[name]
        bad = Model(2, sched, rule="ticks_done").exhaustive()
        assert bad is not None and "read" in bad, f"{name}: {bad}"
        for R in (3, 4):
            m = Model(R, sched, rule="ticks_done")
            assert any(m.random_run(seed) for seed in range(RANDOM_RUNS)), f"{name}, {R} ranks: no seed found the stale read"
    assert Model(2, MODEL_SCHEDULES["calls"], rule="ticks_done").exhaustive() is None
    assert Model(2, [("rows", 2), ("step", 1), ("upload",), ("rows", 3)], rule="ticks_done").exhaustive() is None
    assert Model(1, MODEL_SCHEDULES["reset"], rule="ticks_done").exhaustive() is None


@pytest.mark.parametrize("fault", FAULTS)
def test_peer_window_model_fails_on_a_seeded_fault(fault):
    """Push after the wait: deadlock.  Counter release before the rows, parity off by one, a wait on the count it
    already has: a stale read.  A fill that does not raise the counters: the first wait of a call after plain ticks
    never passes when the count is ticks_done (keyed to the window's count, the counters already hold it, and the
    model passes without the max)."""
    rule, sched = ("ticks_done", [("rows", 2), ("step", 1), ("rows", 2)]) if fault == "fill_without_max" else ("window", MODEL_SCHEDULES["calls"])
    bad = Model(2, sched, rule, fault).exhaustive()
    assert bad is not None, fault
    expect = "deadlock" if fault in ("push_after_wait", "fill_without_max") else "read"
    assert expect in bad, f"{fault}: {bad}"
    for R in (3, 4):
        m = Model(R, sched, rule, fault)
        assert any(m.random_run(seed) for seed in range(RANDOM_RUNS)), f"{fault}, {R} ranks"
    if fault == "fill_without_max":
        for name in MODEL_SCHEDULES:
            assert Model(2, MODEL_SCHEDULES[name], fault=fault).exhaustive() is None, name


def test_model_programs_follow_the_kernels():
    """Hand-worked: the ops of one rank of two for one 2-tick call, as fill / wait / (gravity, push, release, wait)
    launch them."""
    p = rank_program(0, 2, [("rows", 2)])
    assert p == [("st", ("X", 0, 0, 0), 0), ("st", ("X", 0, 0, 1), 0), ("max", ("F", 0, 0), 0), ("max", ("F", 0, 1), 0),
                 ("wait", ("F", 0, 0), 0), ("wait", ("F", 0, 1), 0),
                 ("read", ("X", 0, 0, 0), 0), ("read", ("X", 0, 0, 1), 0),
                 ("st", ("X", 0, 1, 0), 1), ("st", ("X", 1, 1, 0), 1), ("st", ("F", 0, 0), 1), ("st", ("F", 1, 0), 1),
                 ("wait", ("F", 0, 0), 1), ("wait", ("F", 0, 1), 1),
                 ("read", ("X", 0, 1, 0), 1), ("read", ("X", 0, 1, 1), 1),
                 ("st", ("X", 0, 0, 0), 2), ("st", ("X", 1, 0, 0), 2), ("st", ("F", 0, 0), 2), ("st", ("F", 1, 0), 2),
                 ("arrive", 0), ("gather", 0)]
    # the window count keeps going across a reset; ticks_done starts over
    assert rank_program(0, 2, [("rows", 3), ("reset",), ("rows", 1)])[-10][2] == 3
    assert rank_program(0, 2, [("rows", 3), ("reset",), ("rows", 1)], rule="ticks_done")[-10][2] == 0
