"""Every route of the edge-fold gravity over a sparse or irregular edge list, against the oracle body by body.

build_graph calls a graph dense only when every source lists all other bodies in ascending order; every other list
folds in spawn order through small_world_kernel (N <= 32: a world per warp, whole ticks in registers) or
graph_csr_kernel plus a body kernel.  A graph next to an EGM08 field leaves the fused kernels even when dense.  The
graphs here are irregular: edges in shuffled spawn order, bodies without out-edges, a source that lists a target
twice, and (softened) a self-edge.  Each case asserts the kernels that ran, so a changed threshold or a card with
another SM count fails loudly instead of quietly testing another route; FAST is compared per body with
tests.util.assert_body_close (the edge-fold term scaled by S_i = sum of |a_ij| over body i's out-edges), EXACT bit
for bit.

The CPU tests at the bottom prove the bound first: k scaled by 1 + 1e-8, one edge removed and one target's mass
scaled by 1 + 1e-6 must be rejected; the same run with every source's out-edges folded in reverse order (rounding
FAST is allowed) must be accepted.
"""

import functools
import os

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200.executor import FORCE, INERTIA, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from tests.util import (GRAPH_KINDS, MU_EARTH, assert_body_close, assert_route, body_effectors, body_scales,
                        graph_pair_scale, launched_kernels, mutate_term, nbody_pair_scale, nbody_world, orbit_world,
                        run_child)

DT = 1e-3
INTEGRATORS = ("rk4", "semi_implicit")
_I = {"rk4": 0, "semi_implicit": 1}
PAIR_MIN = 2 * 128 * 3 * 132  # kPairMinBodies: body pairs from one full wave up
GENERIC = 2147483648  # SIG_GENERIC: the run-time interpreter


def irregular_edges(N, seed, self_edge):
    """Random out-edges in shuffled spawn order: body N - 1 (and about a fifth of the others, never body 0) has none,
    the others 1..6 distinct targets; body 0 lists one target twice; `self_edge` adds (0, 0)."""
    rng = np.random.default_rng(seed)
    edges = []
    for i in range(N):
        others = [j for j in range(N) if j != i]
        if not others or (i > 0 and (i == N - 1 or rng.random() < 0.2)):
            continue
        deg = int(rng.integers(1, min(6, len(others)) + 1))
        edges += [(i, int(j)) for j in rng.choice(others, deg, replace=False)]
    if edges:
        edges.append(next(e for e in edges if e[0] == 0))
    if self_edge:
        edges.append((0, 0))
    edges = np.array(edges, dtype=np.int64).reshape(-1, 2)
    rng.shuffle(edges)
    return edges.astype(np.uint32)


def _graph(graph, N, seed, kind):
    if graph == "irregular":
        return irregular_edges(N, seed, kind == "softened")
    if graph == "empty":
        return np.zeros((0, 2), dtype=np.uint32)
    if graph == "all":
        return el.all_pairs_edges(N)
    if graph == "perm":  # all pairs, per source: descending (i % 3 == 0), permuted (1) or ascending (2)
        rng = np.random.default_rng(seed)
        rows = []
        for i in range(N):
            t = [j for j in range(N) if j != i]
            rows += [(i, j) for j in (t[::-1] if i % 3 == 0 else rng.permutation(t) if i % 3 == 1 else t)]
        return np.array(rows, dtype=np.uint32)
    if graph == "desc":  # all pairs, per source: descending (even sources) or ascending (odd)
        return np.array([(i, j) for i in range(N) for j in (range(N - 1, -1, -1) if i % 2 == 0 else range(N)) if i != j],
                        dtype=np.uint32)
    if graph == "tmajor":  # all pairs listed target by target: every source's targets still ascend
        return np.array([(i, j) for j in range(N) for i in range(N) if i != j], dtype=np.uint32)
    raise KeyError(graph)


# name: (worlds, entities per world, graph, what follows the gravity in the list)
CASES = {
    **{f"alone{N}": (41, N, "irregular", "") for N in (2, 3, 7, 31, 32)},
    "g_thrust7": (41, 7, "irregular", "g_thrust"),
    "g_thrust32": (41, 32, "irregular", "g_thrust"),
    "self1": (41, 1, "irregular", ""),  # softened only: the self-edge is its one edge
    "empty7": (41, 7, "empty", ""),
    "empty7_g_thrust": (41, 7, "empty", "g_thrust"),
    **{f"alone{N}": (M, N, "irregular", "") for M, N in ((5, 40), (3, 97), (3, 333))},
    "then_g40": (5, 40, "irregular", "g"),
    "then_thrust40": (5, 40, "irregular", "thrust"),
    "pair47": (2200, 47, "irregular", ""),  # 103 400 bodies: body pairs, pairs that straddle two worlds
    "inv7": (1000, 7, "irregular", ""),
    "inv47": (2 * 2201, 47, "irregular", ""),
    "perm100": (3, 100, "perm", ""),
    "desc100": (3, 100, "desc", ""),
    "g_first7": (41, 7, "irregular", "g_first"),  # EXACT only: the gravity ahead of the graph, which overwrites it
    "tmajor100": (3, 100, "tmajor", ""),
    "egm7": (3, 7, "all", "egm08"),
    "egm100": (3, 100, "all", "egm08"),
    "egm40": (3, 40, "irregular", "egm08"),
}


def _kinds(name):
    return ("softened",) if name == "self1" else GRAPH_KINDS


@functools.lru_cache(maxsize=8)
def _case(name, kind, M=None):
    """(start = (pos, vel, ine), effector list, dt) of a case; M overrides the world count (the CPU self-tests)."""
    M0, N, graph, extra = CASES[name]
    M = M or M0
    seed = 7000 + 31 * sorted(CASES).index(name) + (kind == "newton")
    edges = _graph(graph, N, seed, kind)
    if extra == "egm08":
        from tests.test_oracle_golden import _egm08_random_tables

        pos, vel, ine, _, dt = orbit_world(seed, M, N)
        soft = 1e-2
        S1 = graph_pair_scale(pos, ine, edges, kind, 1.0, soft)
        field = MU_EARTH / np.sum(pos[..., 4:] ** 2, -1)
        k = np.median(field) / np.median(S1[S1 > 0])  # the edge-fold term comparable to the field
        cb, sb = _egm08_random_tables(8, np.random.default_rng(5))
        tail = [("egm08", {"c_bar": cb, "s_bar": sb, "L": 8})]
    else:
        pos, vel, ine, k, soft, _ = nbody_world(seed, M, N, DT, edges=edges, kind=kind)
        dt = DT
        rng = np.random.default_rng(seed + 2)
        tail = []
        if extra in ("g_thrust", "g", "g_first"):
            tail.append(("gravity", {"g": (0.0, 3.0, -9.81)}))
        if extra in ("g_thrust", "thrust", "g_first"):
            tail.append(("thrust", {"thrust": rng.uniform(5.0, 20.0, (M, N, 1)) * ine[..., 6:7]}))
    kw = {"edges": edges, "k2": k, "soft": soft} if kind == "softened" else {"edges": edges, "G": k}
    if extra == "g_first":
        return (pos, vel, ine), tail[:1] + [(kind, kw)] + tail[1:], dt
    return (pos, vel, ine), [(kind, kw)] + tail, dt


def _oracle(O, start, spec, integ, dt, ticks):
    """The oracle's (pos, vel, accel, force) after each tick 1..ticks."""
    w = O.World(*start)
    oe = body_effectors(O, spec)[0]
    out = []
    for _ in range(ticks):
        (w.rk4 if integ == "rk4" else w.semi_implicit)(dt, 1, oe, threads=max(1, min(O.max_threads(), os.cpu_count() or 1)))
        out.append(tuple(a.copy() for a in (w.pos, w.vel, w.accel, w.force)))
    return out


# --------------------------------------------------------------------------- the runs, in a child process per switch


def _table(ex, start, dt, cols):
    pos, vel, ine = start
    M, N = pos.shape[:2]
    t = {el.component_id("tick"): np.array([0], dtype=np.uint64), FORCE: np.zeros((M, N, 6)), INERTIA: ine,
         WORLD_POS: pos, WORLD_ACCEL: np.zeros((M, N, 6)), el.component_id("simulation_time_step"): np.array([dt]),
         WORLD_VEL: vel}
    t.update({el.component_id(k): v for k, v in cols.items()})
    return [t[c] for c in ex.input_ids]


def _child_run(out_path, jobs, attempts=3):
    """Child process: run each job [name, kind, integrator, math, {ticks, fused, traj, chunk}] on a fresh handle under
    the profiler; write the kernel names, the launch count and what it computed (final state or trajectory)."""
    res = {}
    for k, (name, kind, integ, math, run) in enumerate(jobs):
        start, spec, dt = _case(name, kind)
        M, N = start[0].shape[:2]
        _, ge, cols = body_effectors(None, spec)
        ticks, traj, chunk = run["ticks"], run.get("traj", 0), run.get("chunk", 0)
        kw = dict(max_fused_ticks=run.get("fused", 1), invoke_chunk_bodies=chunk)
        if traj:
            kw.update(trajectory_every=1, trajectory_capacity=ticks, trajectory_full=traj == 25)
        for _ in range(attempts):
            with el.B200Exec(N, M, dt, None, ge, integ, math, **kw) as ex:
                if chunk:
                    ins = _table(ex, start, dt, cols)
                    n0 = ex.timings()["kernel_launches"]
                    outs, names = launched_kernels(lambda: ex.invoke_batch(ins, ticks))
                    launches = ex.timings()["kernel_launches"] - n0
                    out = dict(zip(ex.output_ids, outs))
                    state = (out[WORLD_POS], out[WORLD_VEL], out[WORLD_ACCEL], out[FORCE])
                else:
                    ex.set_state(*start, **cols)
                    n0 = ex.timings()["kernel_launches"]
                    _, names = launched_kernels(lambda: ex.step(ticks, sync=True))
                    launches = ex.timings()["kernel_launches"] - n0  # (a download launches a layout kernel)
                    state = tuple(ex.download(c) for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE))
                if traj:
                    res[f"{k}_traj"] = ex.trajectory()
            names = [n for n in names if not n.startswith(("Memcpy", "Memset"))]
            if len(names) == launches:
                break
        res[f"{k}_state"] = np.concatenate(state, -1)
        res[f"{k}_names"] = np.array(names, dtype=str)
        res[f"{k}_launches"] = launches
    np.savez(out_path, **res)


def _expected(name, kind, integ, math, run, setting=None):
    """Prefixes of the tick kernels a job must launch (and nothing else)."""
    M, N, graph, extra = CASES[name]
    i, r = _I[integ], "true" if integ == "rk4" else "false"
    exact = math == "exact"
    ex_s = "true" if exact else "false"
    traj = "true" if run.get("traj") else "false"
    body_exact = f"body_exact_kernel<{i}, "
    if extra == "egm08":  # never fused: the field's stage forces precede every body launch
        if exact:
            g = f"graph_dense_kernel<true, {r}>" if graph == "all" else f"graph_csr_kernel<true, {r}>"
        elif graph != "all":
            g = f"graph_csr_kernel<false, {r}>"
        elif N >= 64:
            g = f"graph_dense_world_kernel<{r}, 1024, 512, 1, 2, 2, false, {GENERIC}>"
        else:
            g = "graph_dense_fast_kernel<true, true, 1024>" if integ == "rk4" else "graph_dense_fast_kernel<false, false, 256>"
        return [g, f"egm08_force_kernel<{ex_s}, {r}>", body_exact if exact else f"body_fast_kernel<{i}, 128, 4, false>"]
    if N <= 32 and setting != "B200_SMALL_WORLD=0":
        minb = setting.split("=")[1] if setting and setting.startswith("B200_SMALL_WORLD_CFG") else "4"
        sig = 32 if extra == "" and not exact else GENERIC
        return [f"small_world_kernel<{ex_s}, {i}, {minb}, {sig}>"]
    if graph == "tmajor":
        if exact:
            return [f"graph_dense_kernel<true, {r}>", body_exact]
        if integ == "rk4":  # the persistent world kernel with the integration fused in, compiled for gravity alone
            return ["graph_dense_world_kernel<true, 1024, 512, 1, 2, 2, true, 32>"]
        return [f"graph_dense_world_kernel<false, 1024, 512, 1, 2, 2, false, {GENERIC}>",
                f"body_fast_spec_kernel<1, 32, false, 128, 4, 1>"]
    if exact:
        return [f"graph_csr_kernel<true, {r}>", body_exact]
    g = f"graph_csr_kernel<false, {r}>"
    if extra == "thrust":  # graph + thrust: no compiled signature
        return [g, f"body_fast_kernel<{i}, 128, 4, {traj}>"]
    pair = M * N >= PAIR_MIN and not run.get("chunk")
    body = [f"body_fast_spec_kernel<{i}, 32, {traj}, 128, {'3, 2' if pair else '4, 1'}>"]
    if run.get("chunk") and name == "inv47":
        body.append(f"body_fast_spec_kernel<{i}, 32, false, 128, 3, 2>")
    return [g] + body


SMALL = [f"alone{N}" for N in (2, 3, 7, 31, 32)]
SMALL_RUNS = [{"ticks": 7, "fused": f} for f in (1, 3, 64)]
ONE = [{"ticks": 2}]
TRAJ_RUNS = [{"ticks": 2, "traj": 13}, {"ticks": 2, "traj": 25}]
# FAST rows: name -> runs (each against the oracle)
FAST = {**{n: SMALL_RUNS for n in SMALL}, "g_thrust7": ONE, "g_thrust32": ONE, "self1": SMALL_RUNS, "empty7": ONE,
        "empty7_g_thrust": ONE, "alone40": ONE + TRAJ_RUNS, "alone97": ONE, "alone333": ONE, "then_g40": ONE,
        "then_thrust40": ONE + TRAJ_RUNS, "pair47": ONE, "perm100": ONE, "desc100": ONE, "tmajor100": ONE, "egm7": ONE, "egm100": ONE,
        "egm40": ONE}
EXACT = [n for n in FAST if n != "pair47"] + ["g_first7"]
INVOKE = {"inv7": 7 * 292, "inv47": 2201 * 47}  # invoke_chunk_bodies: whole worlds per range


def _fast_ids():
    return [(n, k, g) for n in FAST for k in _kinds(n) for g in INTEGRATORS]


def _default_jobs():
    jobs = {}
    for n, k, g in _fast_ids():
        for r, run in enumerate(FAST[n]):
            jobs[f"fast-{n}-{k}-{g}-{r}"] = [n, k, g, "fast", run]
    for n in EXACT:
        for k in _kinds(n):
            for g in INTEGRATORS:
                jobs[f"exact-{n}-{k}-{g}"] = [n, k, g, "exact", {"ticks": 2}]
    for n, chunk in INVOKE.items():
        for k in GRAPH_KINDS:
            for g in INTEGRATORS:
                jobs[f"invoke-{n}-{k}-{g}"] = [n, k, g, "fast", {"ticks": 2, "chunk": chunk}]
                jobs[f"step-{n}-{k}-{g}"] = [n, k, g, "fast", {"ticks": 2}]
    return jobs


# B200_* switch -> jobs that run in its child; the small-world launch bounds change no instruction of the kernel
SWITCH_JOBS = {s: [[n, k, g, m, {"ticks": 7, "fused": 3}] for n in ("alone7", "g_thrust32") for k in GRAPH_KINDS
                   for g in INTEGRATORS for m in ("fast", "exact")]
               for s in ("B200_SMALL_WORLD_CFG=2", "B200_SMALL_WORLD_CFG=3")}
SWITCH_JOBS["B200_SMALL_WORLD=0"] = [["alone7", k, g, "fast", {"ticks": 2}] for k in GRAPH_KINDS for g in INTEGRATORS]
SWITCH_JOBS[""] = SWITCH_JOBS["B200_SMALL_WORLD_CFG=2"]  # the same jobs on the default bounds, for the comparison


@pytest.fixture(scope="module")
def routes(tmp_path_factory):
    """{key: (results, index)} of every job, recorded once per child process."""
    d = tmp_path_factory.mktemp("graph_routes")
    jobs = _default_jobs()
    res = run_child("tests.test_graph_routes:_child_run", str(d / "default.npz"), list(jobs.values()))
    out = {key: (res, k) for k, key in enumerate(jobs)}
    for s, sj in SWITCH_JOBS.items():
        r = run_child("tests.test_graph_routes:_child_run", str(d / f"switch{len(out)}.npz"), sj, s or None)
        out.update({(s, k): (r, k) for k in range(len(sj))})
    return out


def _state(res, k):
    a = res[f"{k}_state"]
    return a[..., :7], a[..., 7:13], a[..., 13:19], a[..., 19:25]


def _names(res, k, kernels, what):
    names, launches = list(res[f"{k}_names"]), int(res[f"{k}_launches"])
    assert len(names) == launches, f"{what}: the profiler saw {len(names)} of {launches} launches in every attempt: {names}"
    return assert_route(names, kernels, what)


def _merge(worst, new, label):
    for q, r in new.items():
        if r > worst.get(q, (-1.0, ""))[0]:
            worst[q] = (r, label)


def _report(key, worst):
    print(f"\n{key}: worst error / bound " + ", ".join(f"{q} {r:.3g} ({lab})" for q, (r, lab) in worst.items()))


# --------------------------------------------------------------------------- GPU


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,integ", _fast_ids(), ids=["-".join(x) for x in _fast_ids()])
def test_fast_route_matches_the_oracle(oracle, routes, name, kind, integ):
    """The expected kernels, and every run per body against the oracle: several ticks per small-world launch (bit
    for bit equal to one tick per launch), a trajectory sample every tick against the oracle after that tick."""
    start, spec, dt = _case(name, kind)
    runs = FAST[name]
    want = _oracle(oracle, start, spec, integ, dt, max(r["ticks"] for r in runs))
    sc = body_scales(spec, *start)
    worst, finals = {}, []
    for r, run in enumerate(runs):
        key = f"fast-{name}-{kind}-{integ}-{r}"
        res, k = routes[key]
        ticks = run["ticks"]
        _names(res, k, _expected(name, kind, integ, "fast", run), key)
        if "fused" in run:  # small world: n ticks per launch
            assert int(res[f"{k}_launches"]) == -(-ticks // run["fused"]), key
        if run.get("traj"):
            for t in range(ticks):
                s = res[f"{k}_traj"][t]
                got = (s[..., :7], s[..., 7:13]) + ((s[..., 13:19], s[..., 19:25]) if s.shape[-1] == 25 else want[t][2:])
                _merge(worst, assert_body_close(got, want[t], start, dt, t + 1, sc, what=f"{key} sample {t}"), key)
        else:
            finals.append(_state(res, k))
            _merge(worst, assert_body_close(finals[-1], want[ticks - 1], start, dt, ticks, sc, what=key), key)
    for other in finals[1:]:
        for q, a, b in zip(("pos", "vel", "accel", "force"), finals[0], other):
            assert np.array_equal(a, b), f"{name} {kind} {integ}: {q} depends on the ticks per launch"
    _report(f"{name}-{kind}-{integ}", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("name", EXACT)
def test_exact_route_is_bit_exact(oracle, routes, name):
    """Every list above in EXACT math: the CSR or dense EXACT gravity and body_exact_kernel, or small_world_kernel
    alone; bit for bit, NaNs where the oracle has them."""
    for kind in _kinds(name):
        start, spec, dt = _case(name, kind)
        for integ in INTEGRATORS:
            key = f"exact-{name}-{kind}-{integ}"
            res, k = routes[key]
            _names(res, k, _expected(name, kind, integ, "exact", {"ticks": 2}), key)
            want = _oracle(oracle, start, spec, integ, dt, 2)[-1]
            for q, a, b in zip(("pos", "vel", "accel", "force"), _state(res, k), want):
                assert np.array_equal(a, b, equal_nan=True), f"{key} {q}: max abs diff {np.nanmax(np.abs(a - b))}"


@pytest.mark.gpu
@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("kind", GRAPH_KINDS)
def test_invoke_batch_ranges(oracle, routes, kind, integ):
    """Pipelined invoke_batch.  1000 worlds of 7 in ranges of 292 worlds: the small-world kernel per range, bit for
    bit equal to step().  2 x 2201 worlds of 47 in ranges of 2201 worlds (103 447 bodies): the first range runs body
    pairs, the second starts at an odd body and runs one body per thread, in that order; per body against the oracle."""
    res, k = routes[f"invoke-inv7-{kind}-{integ}"]
    run = {"ticks": 2, "chunk": INVOKE["inv7"]}
    names = _names(res, k, _expected("inv7", kind, integ, "fast", run), "inv7")
    assert len(names) == 2 * -(-1000 // 292), names
    sres, sk = routes[f"step-inv7-{kind}-{integ}"]
    for q, a, b in zip(("pos", "vel", "accel", "force"), _state(res, k), _state(sres, sk)):
        assert np.array_equal(a, b), f"inv7 {kind} {integ}: invoke_batch {q} differs from step()"

    res, k = routes[f"invoke-inv47-{kind}-{integ}"]
    i, r = _I[integ], "true" if integ == "rk4" else "false"
    csr, pair, one = f"graph_csr_kernel<false, {r}>", f"body_fast_spec_kernel<{i}, 32, false, 128, 3, 2>", \
        f"body_fast_spec_kernel<{i}, 32, false, 128, 4, 1>"
    order = [csr, pair] * 2 + [csr, one] * 2
    ticks = _names(res, k, [csr, pair, one], "inv47")
    assert len(ticks) == len(order) and all(n.startswith(e) for n, e in zip(ticks, order)), \
        f"inv47: tick kernels in launch order {ticks}, expected {order}"
    start, spec, dt = _case("inv47", kind)
    want = _oracle(oracle, start, spec, integ, dt, 2)[-1]
    worst = {}
    _merge(worst, assert_body_close(_state(res, k), want, start, dt, 2, body_scales(spec, *start), what="inv47"), "inv47")
    sres, sk = routes[f"step-inv47-{kind}-{integ}"]
    _names(sres, sk, [csr, pair], "inv47 step()")
    _report(f"invoke-{kind}-{integ}", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("setting", [s for s in SWITCH_JOBS if s])
def test_route_switch_in_a_child_process(oracle, routes, setting):
    """B200_SMALL_WORLD_CFG=2 | 3 compile the same small-world kernel for other launch bounds: bit for bit equal to
    the default's results.  B200_SMALL_WORLD=0 sends a sparse 7-body world to the CSR route: per body against the
    oracle."""
    for j, (name, kind, integ, math, run) in enumerate(SWITCH_JOBS[setting]):
        what = f"{setting} {name} {kind} {integ} {math}"
        res, k = routes[(setting, j)]
        _names(res, k, _expected(name, kind, integ, math, run, setting), what)
        if setting.startswith("B200_SMALL_WORLD_CFG"):
            dres, dk = routes[("", j)]
            _names(dres, dk, _expected(name, kind, integ, math, run), what + " (default bounds)")
            for q, a, b in zip(("pos", "vel", "accel", "force"), _state(res, k), _state(dres, dk)):
                assert np.array_equal(a, b, equal_nan=True), f"{what} {q} differs from the default launch bounds"
        else:
            start, spec, dt = _case(name, kind)
            want = _oracle(oracle, start, spec, integ, dt, run["ticks"])[-1]
            assert_body_close(_state(res, k), want, start, dt, run["ticks"], body_scales(spec, *start), what=what)


@pytest.mark.gpu
@pytest.mark.parametrize("math", ["exact", "fast"])
@pytest.mark.parametrize("kind", GRAPH_KINDS)
def test_masked_edge_fold_is_refused(math, kind):
    """An entity mask on an edge-fold gravity effector has no meaning (the fold's members are its edges' sources):
    the library refuses it at create, in both math modes."""
    edges = el.all_pairs_edges(3)
    eff = (el.GravityEdges("softened", k_squared=1.0, softening=1e-3, edges=edges) if kind == "softened"
           else el.GravityEdges("newton", G=1.0, edges=edges)).with_mask(np.array([1, 0, 1], dtype=np.uint8))
    with pytest.raises(el.B200Error) as ei:
        el.B200Exec(3, 2, 0.01, None, [eff], "rk4", math)
    assert ei.value.code == _lib.ERR_UNSUPPORTED
    with el.B200Exec(3, 2, 0.01, None, [eff.with_mask(None)], "rk4", math) as ex:  # the same effector unmasked is fine
        ex.step(1, sync=True)


# --------------------------------------------------------------------------- CPU: the bound is sensitive and not tight

CPU_CASES = ["alone7", "self1", "g_thrust7", "alone40", "then_g40", "then_thrust40", "perm100", "egm40", "egm7"]
CPU_TICKS = 2


def _cpu_ids():
    return [(n, k) for n in CPU_CASES for k in _kinds(n)]


def _cpu_case(name, kind):
    N = CASES[name][1]
    return _case(name, kind, max(1, 129 // N))


def _ratio(O, start, oe, integ, dt, want, sc, ine=None, keep=None):
    """Worst error / bound over every quantity of the oracle run of the effectors `oe` (from the masses `ine`, if
    given) against `want`; `keep`: an entity row taken from `want` (a body the change must not be judged on)."""
    w = O.World(start[0], start[1], start[2] if ine is None else ine)
    for _ in range(CPU_TICKS):
        (w.rk4 if integ == "rk4" else w.semi_implicit)(dt, 1, oe, threads=max(1, min(O.max_threads(), os.cpu_count() or 1)))
    got = tuple(a.copy() for a in (w.pos, w.vel, w.accel, w.force))
    if keep is not None:
        for a, b in zip(got, want):
            a[:, keep] = b[:, keep]
    return max(assert_body_close(got, want, start, dt, CPU_TICKS, sc, check=False).values())


def _largest_edge(start, spec):
    """(index in the edge list, source, target) of the largest |a_ij| at the start positions among the out-edges of
    the sources with out-degree >= 2 (self-edges aside)."""
    pos, _, ine = start
    kind, kw = spec[0]
    e = np.asarray(kw["edges"], dtype=np.int64)
    deg = np.bincount(e[:, 0], minlength=pos.shape[1])
    best = (-1.0, None)
    for idx, (a, b) in enumerate(e):
        if a == b or deg[a] < 2:
            continue
        s = graph_pair_scale(pos, ine, e[idx:idx + 1], kind, 1.0, kw.get("soft", 0.0))[:, a].max()
        if s > best[0]:
            best = (s, (idx, int(a), int(b)))
    return best[1]


WORST = {}


@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("name,kind", _cpu_ids(), ids=["-".join(x) for x in _cpu_ids()])
def test_bound_rejects_graph_faults_and_accepts_reordering(oracle, name, kind, integ):
    """k (or G) scaled by 1 + 1e-8, the largest out-edge of a source of degree >= 2 removed, and the mass of that
    edge's target scaled by 1 + 1e-6 (judged on the other bodies: only the sources with an edge to it see it) must
    fail assert_body_close; every source's out-edges folded in reverse order must pass."""
    O = oracle
    start, spec, dt = _cpu_case(name, kind)
    sc = body_scales(spec, *start)
    want = _oracle(O, start, spec, integ, dt, CPU_TICKS)[-1]
    kw = spec[0][1]
    edges = np.asarray(kw["edges"])
    with_edges = lambda e: body_effectors(O, [(kind, {**kw, "edges": e})] + spec[1:])[0]
    ratios = {}
    if np.any(body_scales(spec[:1], *start)[0] > 0):  # (a lone self-edge pulls with nothing to scale)
        ratios["k"] = _ratio(O, start, mutate_term(O, spec, 0, "graph", 1.0 + 1e-8), integ, dt, want, sc)
    picked = _largest_edge(start, spec)
    if picked is not None:
        idx, _, tgt = picked
        ratios["edge"] = _ratio(O, start, with_edges(np.delete(edges, idx, axis=0)), integ, dt, want, sc)
        ine = start[2].copy()
        ine[:, tgt, 6] *= 1.0 + 1e-6
        ratios["mass"] = _ratio(O, start, body_effectors(O, spec)[0], integ, dt, want, sc, ine=ine, keep=tgt)
    order = np.argsort(edges[:, 0], kind="stable")
    rev = np.concatenate([order[edges[order, 0] == s][::-1] for s in np.unique(edges[:, 0])]) if len(edges) else order
    ratios["reversed"] = _ratio(O, start, with_edges(edges[rev]), integ, dt, want, sc)
    for q, r in ratios.items():
        WORST[q] = max(WORST.get(q, (0.0, "")), (r, f"{name} {kind} {integ}")) if q == "reversed" else \
            min(WORST.get(q, (np.inf, "")), (r, f"{name} {kind} {integ}"))
    print(f"\n{name} {kind} {integ}: error / bound " + ", ".join(f"{q} {r:.3g}" for q, r in ratios.items()))
    print("  over the cases so far (smallest for the faults, largest for the reordering): "
          + ", ".join(f"{q} {r:.3g} ({lab})" for q, (r, lab) in WORST.items()))
    for q in ("k", "edge", "mass"):
        if q in ratios:
            assert ratios[q] > 1.0, f"{name} {kind} {integ}: the {q} fault passes ({ratios[q]:.3g} of the bound)"
    assert ratios["reversed"] <= 1.0, f"{name} {kind} {integ}: the reversed fold order fails ({ratios['reversed']:.3g})"


def test_graph_pair_scale_matches_the_all_pairs_scale():
    """On all-pairs edges, the edge-list scale equals the vectorised all-pairs one (both kinds)."""
    pos, vel, ine, k, soft, S = nbody_world(3, 4, 23, DT)
    edges = el.all_pairs_edges(23)
    np.testing.assert_allclose(graph_pair_scale(pos, ine, edges, "softened", k, soft), S, rtol=1e-13)
    np.testing.assert_allclose(graph_pair_scale(pos, ine, edges, "newton", k, 0.0), nbody_pair_scale(pos, ine, k, 0.0), rtol=1e-13)
    # a self-edge adds nothing, a repeated edge counts twice, a body without out-edges has S = 0
    e = np.array([(0, 0), (0, 1), (0, 1), (2, 1)], dtype=np.uint32)
    one = graph_pair_scale(pos, ine, e[1:2], "softened", k, soft)
    got = graph_pair_scale(pos, ine, e, "softened", k, soft)
    np.testing.assert_allclose(got[:, 0], 2 * one[:, 0], rtol=1e-15)
    assert np.all(got[:, 1] == 0) and np.all(got[:, 3:] == 0)


@pytest.mark.parametrize("kind", GRAPH_KINDS)
def test_graph_scale_bounds_the_oracle_stage(oracle, kind):
    """|a_i| of the edge-fold gravity alone (oracle.World.eval_stage) never exceeds S_i, and equals it for a body
    with one out-edge."""
    start, spec, _ = _cpu_case("alone40", kind)
    pos, vel, ine = start
    S = body_scales(spec, *start)[0]
    e = np.asarray(spec[0][1]["edges"])
    deg = np.bincount(e[:, 0], minlength=pos.shape[1])
    w = oracle.World(pos, vel, ine)
    for world in range(pos.shape[0]):
        _, A = w.eval_stage(world, body_effectors(oracle, spec[:1])[0])
        a = np.sqrt(np.sum(A[:, 3:] ** 2, -1))
        assert np.all(a <= S[world] * (1 + 1e-12))
        one = deg == 1
        np.testing.assert_allclose(a[one], S[world][one], rtol=1e-12)
