"""The trajectory ring on every tick route, at every sampling phase, capacity edge and world range, tick by tick.

The rule that puts a tick into a ring slot is restated in every tick kernel (fast_ticks, body_exact_kernel, the
deferred pair store of body_fast_spec_kernel, traj_due of the EXACT small_world_kernel) and on the host (launch_ticks'
tick0, range_step_params' ring offset, trajectory_len, trajectory_reset).  The contract these tests hold them to:

  R1  After a reset at absolute tick t_r, sample k < C is the state after tick t_r + (k + 1) every (all 13 or 25
      planes), and trajectory_len == min(ticks since the reset // every, C), however the ticks were split into
      launches, step() calls or invoke_batch ranges.
  R2  A full ring does not change any more; the state columns after a recording run equal a ring-less handle's bit
      for bit; the 13-wide ring of a schedule is the first 13 planes of its 25-wide ring.
  R3  EXACT samples equal the oracle bit for bit.  FAST samples equal, bit for bit, the per-tick reference (the same
      handle configuration without a ring, stepped one tick per launch, downloaded after every tick), and that
      reference is within the per-body bounds of tests.util (assert_body_close / assert_nbody_close) of the oracle at
      every sampled tick.
  R4  A step() that ends on a sample tick leaves its state in the last sample, bit for bit.

`plan` restates launch_ticks' partition of a step into launches; every GPU case asserts the kernel_launches delta it
predicts, so a schedule cannot quietly turn into aligned launches.  The CPU tests check the restatement on
hand-worked schedules, that the schedules reach every phase and capacity edge, and that a sample taken one tick off
is rejected by the FAST bound used at its tick.
"""

import functools
import os

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200.executor import FORCE, INERTIA, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from tests import test_body_routes as BR
from tests import test_graph_routes as GR
from tests import test_nbody_routes as NR
from tests.test_run_summary import ref_tables, same
from tests.util import (assert_body_close, assert_nbody_close, assert_route, body_effectors, body_scales,
                        launched_kernels, run_child)

INTEGRATORS = ("rk4", "semi_implicit")
_I = {"rk4": 0, "semi_implicit": 1}
GENERIC = 2147483648  # SIG_GENERIC: the run-time interpreter
_TICK_KERNELS = ("graph_dense_kernel<", "graph_dense_fast_kernel<", "graph_dense_world_kernel<", "graph_csr_kernel<",
                 "nbody_tick_fused_kernel<", "small_world_kernel<", "body_exact_kernel<", "body_fast_kernel<",
                 "body_fast_spec_kernel<", "egm08_force_kernel<")

# --------------------------------------------------------------------------- schedules and their restatement

# steps: the tick counts of successive step() calls; "reset" = trajectory_reset() between two of them
SCHEDULES = {
    # [0,2) [2,6) [6,9) [9,13) [13,17) [17,21) [21,22): [2,6) starts at phase 2 and records ticks 3 and 6, [13,17)
    # fills the ring at tick 15; the reset at tick 22 is mid-phase, then samples at absolute ticks 25, 28 and 31
    "overrun_reset": dict(every=3, fused=4, cap=5, steps=(2, 7, 4, 9, "reset", 5, 6)),
    "exec": dict(every=5, fused=32, cap=3, steps=(23,)),  # Exec's shape: one launch fills the ring at 15, runs 8 more
    "single": dict(every=2, fused=1, cap=4, steps=(9,)),  # one-tick launches: the deferred pair store skips odd ticks
    "sparse": dict(every=7, fused=3, cap=2, steps=(16,)),  # most launches record nothing
    "control": dict(every=1, fused=7, cap=10, steps=(13,)),
}


def plan(sched, multi=True, per_launch=1):
    """launch_ticks' partition of a schedule: `multi` = the route runs several ticks per launch (max_fused_ticks),
    else one; `per_launch` = kernels per launch (EGM08 field + body, gravity + body: 2).

    Returns (steps, rings).  steps: one dict per step() with its launches [(first tick since the reset, ticks,
    starting phase, [absolute ticks it records])], the expected kernel_launches delta, the absolute tick it ends on
    and trajectory_len after it.  rings: the absolute tick of every slot in the ring read before each reset and at
    the end."""
    every, cap = sched["every"], sched["cap"]
    fuse = sched["fused"] if multi else 1
    t_abs = t_rel = r0 = 0
    steps, rings = [], []
    slots = lambda: [r0 + (k + 1) * every for k in range(min(t_rel // every, cap))]
    for op in sched["steps"]:
        if op == "reset":
            rings.append(slots())
            r0, t_rel = t_abs, 0
            continue
        launches, left = [], op
        while left:
            n = min(left, fuse)
            rec = [r0 + t for t in range(t_rel + 1, t_rel + n + 1) if t % every == 0 and t // every <= cap]
            launches.append((t_rel, n, t_rel % every, rec))
            t_rel, t_abs, left = t_rel + n, t_abs + n, left - n
        steps.append(dict(n=op, launches=launches, delta=per_launch * len(launches), tick=t_abs,
                          len=min(t_rel // every, cap), slots=slots()))
    rings.append(slots())
    return steps, rings


def _total(sched):
    return sum(s for s in sched["steps"] if s != "reset")


# --------------------------------------------------------------------------- the route cases

SPEC = ("free", "thrust_drag", "frame_wrench", "wheels_j2")
ALL = tuple(SCHEDULES)
WIDTHS = (13, 25)
FUSED = NR.FUSED


def _body_case(name, integ, size="small", math="fast", runs=None):
    sig = BR.CASES[name][3] if math == "fast" else None
    if math == "exact":
        kern = lambda w: [f"body_exact_kernel<{_I[integ]}, "]
    elif sig is None:
        kern = lambda w: [BR._interp_kernel(integ, True)] + (["egm08_force_kernel<"] if name == "egm08" else [])
    else:
        kern = lambda w: [BR._spec_kernel(integ, sig, True, size == "pair")]
    egm = name == "egm08"
    return dict(fam="body", name=name, integ=integ, size=size, math=math, kernels=kern, multi=not egm,
                per_launch=2 if egm else 1, runs=runs or [(s, w) for s in ALL for w in WIDTHS])


def _nbody_case(M, N, integ, kernels, per_launch, math="fast", runs=None, multi=False):
    return dict(fam="nbody", name=(M, N), integ=integ, size=None, math=math, kernels=lambda w: kernels, multi=multi,
                per_launch=per_launch, runs=runs or [(s, w) for s in ALL for w in WIDTHS])


def _graph_case(name, integ, math, kernels, multi, per_launch, runs=None):
    return dict(fam="graph", name=name, integ=integ, size=None, math=math, kernels=lambda w: kernels, multi=multi,
                per_launch=per_launch, runs=runs or [(s, w) for s in ALL for w in WIDTHS])


# the pair cases run ~1e5 bodies: one schedule per ring width (the 13-wide one-tick launches are the deferred store,
# and the mass-class summary serves the free bodies' launches that write no Force)
PAIR_RUNS = [("single", 13), ("exec", 25)]
CASES = {}
for _g in INTEGRATORS:
    _gi = _I[_g]
    _r = "true" if _g == "rk4" else "false"
    CASES[f"exact-g_thrust_drag-{_g}"] = _body_case("g_thrust_drag", _g, math="exact")
    for _n in SPEC:
        CASES[f"spec-{_n}-{_g}"] = _body_case(_n, _g)
    CASES[f"pair-free-{_g}"] = _body_case("free", _g, "pair", runs=PAIR_RUNS)
    for _n in ("masked", "two_thrusts", "egm08"):
        CASES[f"interp-{_n}-{_g}"] = _body_case(_n, _g)
    # small_world_kernel: an all-pairs world and an irregular graph, EXACT and FAST
    CASES[f"small-dense-{_g}"] = _nbody_case(41, 7, _g, [f"small_world_kernel<false, {_gi}, 4, 32>"], 1, multi=True)
    CASES[f"small-dense-exact-{_g}"] = _nbody_case(41, 7, _g, [f"small_world_kernel<true, {_gi}, 4, {GENERIC}>"], 1, "exact",
                                                   multi=True)
    CASES[f"small-irregular-{_g}"] = _graph_case("alone7", _g, "fast", [f"small_world_kernel<false, {_gi}, 4, 32>"], True, 1)
    CASES[f"small-irregular-exact-{_g}"] = _graph_case("alone7", _g, "exact", [f"small_world_kernel<true, {_gi}, 4, {GENERIC}>"],
                                                        True, 1)
    # graph_csr_kernel + the gravity-signature body kernel: an irregular graph of 40 bodies
    CASES[f"csr-{_g}"] = _graph_case("alone40", _g, "fast", [f"graph_csr_kernel<false, {_r}>",
                                                             f"body_fast_spec_kernel<{_gi}, 32, true, 128, 4, 1>"], False, 2)
_TJ = lambda k: k.replace(", false, 128, ", ", true, 128, ")  # the body kernel instantiated with the ring
CASES.update({
    # nbody_tick_fused_kernel: the ping-pong planes, after odd and even tick counts (the shape of the n-body world
    # test_parity_gpu.test_resident_run_equals_invoke_batch_run runs on this kernel)
    "nbody-fused": _nbody_case(3, 40, "rk4", [FUSED], 1),
    # the persistent world kernel with the integration fused in (the shape of that test's world-kernel world)
    "nbody-world": _nbody_case(180, 128, "rk4", [NR._world_kernel(NR.WORLD_4x1, True, True)], 1),
    # dense gravity + body kernel, RK4 and semi-implicit
    "nbody-dense": _nbody_case(80, 40, "rk4", [NR.DENSE_FAST, _TJ(NR.BODY_RK4)], 2),
    "nbody-world-semi": _nbody_case(41, 97, "semi_implicit", [NR.WORLD_SEMI, _TJ(NR.BODY_SEMI)], 2),
    # 103 400 bodies: the body-pair kernel behind dense gravity, pairs straddling two worlds
    "nbody-pair": _nbody_case(2200, 47, "rk4", [NR.DENSE_FAST, _TJ(NR.BODY_RK4_PAIR)], 2, runs=PAIR_RUNS),
    # EXACT dense gravity + body_exact_kernel
    "nbody-exact": _nbody_case(3, 130, "semi_implicit", ["graph_dense_kernel<true, false>", "body_exact_kernel<1, "], 2, "exact"),
})

# invoke_batch with every > 1: the small (packed) path, pipelined ranges of 31 three-body worlds (a range length that
# does not divide the 101 worlds, and ranges that start at the odd bodies 93 and 279: one body per thread), and two
# pipelined ranges past kPairMinBodies (body pairs, the deferred store, then a range at an odd body)
INVOKE_RUNS = [("overrun_reset", 13), ("sparse", 25), ("single", 13)]
INVOKE = {
    "invoke-small": dict(_body_case("thrust_drag", "rk4", runs=INVOKE_RUNS), worlds=101, chunk=0),
    "invoke-ranges": dict(_body_case("thrust_drag", "semi_implicit", runs=INVOKE_RUNS), worlds=101, chunk=31 * 3),
    "invoke-pair": dict(_body_case("free", "rk4", "misaligned", runs=[("single", 13)]), worlds=None, chunk=BR._chunk("free")),
}
for _k, _c in INVOKE.items():
    _one = BR._spec_kernel(_c["integ"], BR.CASES[_c["name"]][3], True, False)
    _pair = BR._spec_kernel(_c["integ"], BR.CASES[_c["name"]][3], True, True)
    _c["kernels"] = (lambda ks: lambda w: ks)([_one, _pair] if _k == "invoke-pair" else [_one])
    CASES[_k] = _c

HEAD = 300  # the worlds compared with the oracle in the largest cases: the first HEAD and the last


@functools.lru_cache(maxsize=2)
def _world(key):
    """(start = (pos, vel, ine), effector spec or None, dt, lib effectors, columns, S or None) of a case."""
    c = CASES[key]
    if c["fam"] == "nbody":
        M, N = c["name"]
        (pos, vel, ine, S), _, ge, cols = NR._setup(None, M, N, False)
        return (pos, vel, ine), None, NR.DT, ge, cols, S
    if c["fam"] == "graph":
        start, spec, dt = GR._case(c["name"], "softened")
    elif c["math"] == "exact":
        start, spec, dt = BR._exact_world(c["name"])
    elif c.get("worlds"):
        start, spec, dt = BR._world(c["name"], c["worlds"])
    else:
        start, spec, dt = BR._sized(c["name"], c["size"])
    _, ge, cols = body_effectors(None, spec)
    return start, spec, dt, ge, cols, None


def _select(M):
    return np.unique(np.r_[np.arange(min(M, HEAD)), M - 1])


def _subset(key, sel):
    """The start, oracle-side spec and S of the worlds `sel` of a case."""
    start, spec, dt, _, _, S = _world(key)
    cut = lambda a: a[sel] if isinstance(a, np.ndarray) and a.ndim == 3 else a
    spec = None if spec is None else [(k, {n: cut(v) for n, v in kw.items()}) for k, kw in spec]
    return tuple(a[sel] for a in start), spec, None if S is None else S[sel]


def _oracle_effs(O, key, spec):
    if spec is None:
        M, N = CASES[key]["name"]
        return NR._setup(O, M, N, False)[1]
    return body_effectors(O, spec)[0]


def _oracle_run(O, key, sel, ticks):
    """The oracle's (pos, vel, accel, force) of the worlds `sel` after each tick 0..ticks (tick 0: the start, with
    zero accel and force)."""
    c = CASES[key]
    start, spec, S = _subset(key, sel)
    dt = _world(key)[2]
    w = O.World(*start)
    oe = _oracle_effs(O, key, spec)
    z = np.zeros(start[0].shape[:2] + (6,))
    out = [(start[0], start[1], z, z)]
    for _ in range(ticks):
        (w.rk4 if c["integ"] == "rk4" else w.semi_implicit)(dt, 1, oe, threads=max(1, min(O.max_threads(), os.cpu_count() or 1)))
        out.append(tuple(a.copy() for a in (w.pos, w.vel, w.accel, w.force)))
    return out, start, spec, S


def _fast_check(key, got, want, start, spec, S, t, check=True):
    """The FAST comparison at tick t: {quantity: worst ratio}; raises unless check=False (then the ratios of the
    body checks; the n-body check has no such mode and raises)."""
    dt = _world(key)[2]
    if S is not None:
        return assert_nbody_close(got, want, start, dt, t, S, what=f"{key} tick {t}")
    return assert_body_close(got, want, start, dt, t, body_scales(spec, *start), what=f"{key} tick {t}", check=check)


# --------------------------------------------------------------------------- the runs, in a child process

_COLS = (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)


def _state(ex):
    return np.concatenate([ex.download(c) for c in _COLS], -1)


def _open(key, ring, fused, sched=None, width=13):
    start, _, dt, ge, cols, _ = _world(key)
    c = CASES[key]
    M, N = start[0].shape[:2]
    kw = dict(max_fused_ticks=fused, invoke_chunk_bodies=c.get("chunk", 0))
    if ring:
        kw.update(trajectory_every=sched["every"], trajectory_capacity=sched["cap"], trajectory_full=width == 25)
    ex = el.B200Exec(N, M, dt, None, ge, c["integ"], c["math"], **kw)
    ex.set_state(*start, **cols)
    return ex


def _invoke_table(ex, key):
    start, _, dt, _, cols, _ = _world(key)
    pos, vel, ine = start
    M, N = pos.shape[:2]
    t = {el.component_id("tick"): np.array([0], dtype=np.uint64), FORCE: np.zeros((M, N, 6)), INERTIA: ine,
         WORLD_POS: pos, WORLD_ACCEL: np.zeros((M, N, 6)), el.component_id("simulation_time_step"): np.array([dt]),
         WORLD_VEL: vel}
    t.update({el.component_id(k): v for k, v in cols.items()})
    return [t[c] for c in ex.input_ids]


def _record(key, sched_name, width, invoke):
    """One recording run of a schedule: per step, its kernel_launches delta (step() only), trajectory_len, the ring
    and the state after it."""
    sched = SCHEDULES[sched_name]
    ex = _open(key, True, sched["fused"], sched, width)
    out = {"delta": [], "len": [], "rings": [], "states": []}
    first = True
    for op in sched["steps"]:
        if op == "reset":
            ex.trajectory_reset()
            continue
        n0 = ex.timings()["kernel_launches"]
        if invoke:
            ins = _invoke_table(ex, key) if first else [None] * len(ex.input_ids)
            res = dict(zip(ex.output_ids, ex.invoke_batch(ins, op)))
            out["delta"].append(ex.timings()["kernel_launches"] - n0)
            st = np.concatenate([res[c] for c in _COLS], -1)
        else:
            ex.step(op, sync=True)
            out["delta"].append(ex.timings()["kernel_launches"] - n0)  # before the downloads' layout launches
            st = _state(ex)
        first = False
        out["len"].append(ex.trajectory_len())
        out["rings"].append(ex.trajectory())
        out["states"].append(st)
    ex.close()
    return out


def _needed_ticks(key):
    """The absolute ticks whose reference state a case compares: every sample and every step end."""
    c = CASES[key]
    need = set()
    for s, _ in c["runs"]:
        for st in plan(SCHEDULES[s], c["multi"], c["per_launch"])[0]:
            need.update(st["slots"])
            need.add(st["tick"])
    return sorted(need)


def _child(done_path, args, attempts=3):
    """Child process: per case of args = [out_dir, keys], every recording run under the profiler (kernel names of the
    whole window), then the per-tick reference; one .npz per case in out_dir, then done_path."""
    out_dir, keys = args
    for key in keys:
        c = CASES[key]
        invoke = "chunk" in c
        for attempt in range(attempts):
            runs = {}

            def go():
                for s, w in c["runs"]:
                    runs[(s, w, False)] = _record(key, s, w, False)
                    if invoke:
                        runs[(s, w, True)] = _record(key, s, w, True)

            _, names = launched_kernels(go, settle=0.05 * 4 ** attempt)
            ticks = [n for n in names if n.startswith(_TICK_KERNELS)]
            want = sum(sum(r["delta"]) for (s, w, inv), r in runs.items() if not inv)
            if invoke:  # every range of every invoke_batch call runs the schedule's tick launches
                M = _world(key)[0][0].shape[0]
                ranges = 1 if not c["chunk"] else -(-M // max(1, c["chunk"] // _world(key)[0][0].shape[1]))
                want += ranges * sum(sum(st["delta"] for st in plan(SCHEDULES[s], c["multi"], c["per_launch"])[0])
                                     for s, w in c["runs"])
            if len(ticks) == want:
                break
        res = {"names": np.array(ticks, dtype=str), "names_ok": len(ticks) == want, "names_want": want,
               "all_names": np.array(sorted(set(names)), dtype=str)}
        for (s, w, inv), r in runs.items():
            p = f"{s}_{w}_{'inv' if inv else 'step'}"
            res[f"{p}_delta"] = np.array(r["delta"])
            res[f"{p}_len"] = np.array(r["len"])
            for i, (ring, st) in enumerate(zip(r["rings"], r["states"])):
                res[f"{p}_ring{i}"] = ring
                res[f"{p}_state{i}"] = st
        # the per-tick reference: no ring, one tick per launch, the state downloaded after every tick
        need = _needed_ticks(key)
        ex = _open(key, False, 1)
        ref = []
        for t in range(1, need[-1] + 1):
            ex.step(1, sync=True)
            if t in need:
                ref.append(_state(ex))
        ex.close()
        res["ref_ticks"] = np.array(need)
        res["ref"] = np.stack(ref)
        np.savez(os.path.join(out_dir, key + ".npz"), **res)
    np.savez(done_path, ok=True)


@pytest.fixture(scope="module")
def recorded(request, tmp_path_factory):
    """The directory of the child's results, for the cases this session selected."""
    keys = [it.callspec.params["key"] for it in request.session.items
            if getattr(it, "originalname", "") == "test_ring_follows_the_slot_rule_on_every_route"]
    d = tmp_path_factory.mktemp("trajectory_routes")
    run_child("tests.test_trajectory_routes:_child", str(d / "done.npz"), [str(d), keys], timeout=1800)
    return d


def _load(d, key):
    with np.load(os.path.join(d, key + ".npz")) as z:
        return {k: z[k] for k in z.files}


def _eq(a, b, what):
    assert a.shape == b.shape, f"{what}: shape {a.shape} != {b.shape}"
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        raise AssertionError(f"{what}: {len(bad)} values differ, first at {tuple(bad[0])}: {a[tuple(bad[0])]!r} != "
                             f"{b[tuple(bad[0])]!r}")


# --------------------------------------------------------------------------- GPU: every route


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(CASES))
def test_ring_follows_the_slot_rule_on_every_route(oracle, recorded, key):
    """R1 - R4 on one route: the kernels and launch counts each schedule predicts, every slot and trajectory_len after
    every step, the ring-less state, the 13 / 25-wide rings, and the per-tick reference against the oracle."""
    O = oracle
    c = CASES[key]
    res = _load(recorded, key)
    assert bool(res["names_ok"]), (f"{key}: the profiler saw {len(res['names'])} of {int(res['names_want'])} tick launches "
                                   f"in every attempt: {sorted(set(res['names']))} {list(res['all_names'])}")
    assert_route(list(res["names"]), c["kernels"](13), key)
    ref_ticks = list(res["ref_ticks"])
    ref = lambda t: res["ref"][ref_ticks.index(t)]
    sampled = set()
    for s, w in c["runs"]:
        steps, _ = plan(SCHEDULES[s], c["multi"], c["per_launch"])
        modes = ("step", "inv") if "chunk" in c else ("step",)
        for mode in modes:
            p = f"{s}_{w}_{mode}"
            what = f"{key} {s} width {w} {mode}"
            if mode == "step":
                assert list(res[f"{p}_delta"]) == [st["delta"] for st in steps], f"{what}: kernel launches per step()"
            assert list(res[f"{p}_len"]) == [st["len"] for st in steps], f"{what}: trajectory_len per step"
            for i, st in enumerate(steps):
                ring, state = res[f"{p}_ring{i}"], res[f"{p}_state{i}"]
                assert ring.shape[0] == st["len"] and ring.shape[-1] == w, what
                # R1 / R3: sample k is the reference state at its tick (every plane the ring holds)
                for k, t in enumerate(st["slots"]):
                    _eq(ring[k], ref(t)[..., :w], f"{what} step {i} sample {k} (tick {t})")
                    sampled.add(t)
                # R2: the state columns equal the ring-less handle's; R4: a step ending on a sample tick
                _eq(state, ref(st["tick"]), f"{what} step {i} state")
                if st["slots"] and st["slots"][-1] == st["tick"]:
                    _eq(ring[-1], state[..., :w], f"{what} step {i} last sample vs download")
                if mode == "inv":
                    _eq(ring, res[f"{s}_{w}_step_ring{i}"], f"{what} step {i}: invoke_batch ring vs step() ring")
        if w == 25 and (s, 13) in c["runs"]:  # R2: the 13-wide ring is the 25-wide ring's first 13 planes
            for i in range(len(steps)):
                _eq(res[f"{s}_13_step_ring{i}"], res[f"{s}_25_step_ring{i}"][..., :13], f"{key} {s} step {i}: 13 vs 25 planes")
    # R3: the reference against the oracle at every sampled tick
    M = _world(key)[0][0].shape[0]
    sel = _select(M)
    want, start, spec, S = _oracle_run(O, key, sel, max(sampled))
    worst = {}
    for t in sorted(sampled):
        r = ref(t)[sel]
        got = (r[..., :7], r[..., 7:13], r[..., 13:19], r[..., 19:25])
        if c["math"] == "exact":
            for q, a, b in zip(("pos", "vel", "accel", "force"), got, want[t]):
                _eq(a, b, f"{key} tick {t} {q} against the oracle")
        else:
            for q, v in _fast_check(key, got, want[t], start, spec, S, t).items():
                worst[q] = max(worst.get(q, 0.0), v)
    if worst:
        print(f"\n{key}: worst error / bound over the sampled ticks " + ", ".join(f"{q} {v:.3g}" for q, v in worst.items()))


# --------------------------------------------------------------------------- GPU: run summaries over a ring with every > 1

SUMMARY_SCHED = SCHEDULES["overrun_reset"]


@pytest.mark.gpu
@pytest.mark.parametrize("math", ["exact", "fast"])
def test_summary_labels_ring_samples_with_their_ticks(math):
    """summary_add_trajectory on a 25-wide ring with every = 3, C = 5, read after overrunning and after a mid-phase
    reset: the extrema and threshold tables, ticks included, equal ref_tables on the R1 rows (ticks t_r + (k+1) every)
    of a per-tick reference run.  Thresholds cross between two samples of one world."""
    M, N = 37, 3
    every, cap = SUMMARY_SCHED["every"], SUMMARY_SCHED["cap"]
    pos, vel, ine, cols, dt = BR.near_world(11, M, N)
    effs = [el.GravityConst((0.0, 0.0, -9.81)), el.ThrustBody((-1.0, 0.0, 0.0), "thrust"),
            el.DragQuadratic(0.6125, 0.0025, "wind")]
    _, rings = plan(SUMMARY_SCHED)
    T = _total(SUMMARY_SCHED)
    with el.B200Exec(N, M, dt, None, effs, "rk4", math) as ref:
        ref.set_state(pos, vel, ine, thrust=cols["thrust"], wind=cols["wind"])
        rows = [None]
        for _ in range(T):
            ref.step(1, sync=True)
            rows.append(_state(ref))
    ex = el.B200Exec(N, M, dt, None, effs, "rk4", math, max_fused_ticks=SUMMARY_SCHED["fused"], trajectory_every=every,
                     trajectory_capacity=cap, trajectory_full=True)
    ex.set_state(pos, vel, ine, thrust=cols["thrust"], wind=cols["wind"])
    folds = []
    try:
        for op in SUMMARY_SCHED["steps"] + ("end",):
            if op in ("reset", "end"):
                slots = rings[len(folds)]
                R = np.stack([rows[t] for t in slots])
                mid = R.shape[0] // 2
                thr = [(0, 6, bool(R[mid, 0, 0, 6] > R[mid - 1, 0, 0, 6]), float(0.5 * (R[mid, 0, 0, 6] + R[mid - 1, 0, 0, 6]))),
                       (N - 1, 10, bool(R[-1, -1, N - 1, 10] > R[-2, -1, N - 1, 10]),
                        float(0.5 * (R[-1, -1, N - 1, 10] + R[-2, -1, N - 1, 10]))),
                       (1, 4, False, float(np.median(R[0, :, 1, 4])))]
                ex.summary_begin(True, thr)
                ex.summary_add_trajectory()
                got = (ex.extrema(), ex.thresholds())
                want = ref_tables(R, slots, thr)
                for g, w_, q in zip(got, want, ("extrema", "thresholds")):
                    assert g.shape == w_.shape and same(g, w_), f"{math} ring {len(folds)} {q}"
                hit = want[1][:, :, 0]
                assert np.any((hit > slots[0]) & (hit < slots[-1])), "no threshold fires mid-ring"
                folds.append(slots)
                if op == "reset":
                    ex.trajectory_reset()
                continue
            ex.step(op, sync=True)
    finally:
        ex.close()
    assert folds == [[3, 6, 9, 12, 15], [25, 28, 31]]


# --------------------------------------------------------------------------- CPU: the restatement and its reach


def test_plan_on_hand_worked_schedules():
    """The launches, sample ticks, trajectory_len and launch counts of the five schedules, worked by hand."""
    steps, rings = plan(SCHEDULES["overrun_reset"])
    assert [[(a, n) for a, n, _, _ in st["launches"]] for st in steps] == [
        [(0, 2)], [(2, 4), (6, 3)], [(9, 4)], [(13, 4), (17, 4), (21, 1)], [(0, 4), (4, 1)], [(5, 4), (9, 2)]]
    assert [st["launches"][0][2] for st in steps] == [0, 2, 0, 1, 0, 2]
    assert steps[1]["launches"][0][3] == [3, 6] and steps[3]["launches"][0][3] == [15]
    assert steps[3]["launches"][1][3] == [] and steps[3]["launches"][2][3] == []
    assert [st["delta"] for st in steps] == [1, 2, 1, 3, 2, 2]
    assert [st["len"] for st in steps] == [0, 3, 4, 5, 1, 3]
    assert [st["tick"] for st in steps] == [2, 9, 13, 22, 27, 33]
    assert rings == [[3, 6, 9, 12, 15], [25, 28, 31]]
    # one launch per tick (EGM08: field + body per tick)
    steps, _ = plan(SCHEDULES["overrun_reset"], multi=False, per_launch=2)
    assert [st["delta"] for st in steps] == [4, 14, 8, 18, 10, 12]
    steps, rings = plan(SCHEDULES["exec"])
    assert [(a, n, p, r) for a, n, p, r in steps[0]["launches"]] == [(0, 23, 0, [5, 10, 15])]
    assert steps[0]["len"] == 3 and rings == [[5, 10, 15]]
    steps, rings = plan(SCHEDULES["single"])
    assert steps[0]["delta"] == 9 and rings == [[2, 4, 6, 8]]
    assert [r for _, _, _, r in steps[0]["launches"]] == [[], [2], [], [4], [], [6], [], [8], []]
    steps, rings = plan(SCHEDULES["sparse"])
    assert [(a, n, p, r) for a, n, p, r in steps[0]["launches"]] == [
        (0, 3, 0, []), (3, 3, 3, []), (6, 3, 6, [7]), (9, 3, 2, []), (12, 3, 5, [14]), (15, 1, 1, [])]
    assert rings == [[7, 14]] and steps[0]["delta"] == 6
    steps, rings = plan(SCHEDULES["control"])
    assert [n for _, n, _, _ in steps[0]["launches"]] == [7, 6] and rings == [list(range(1, 11))] and steps[0]["len"] == 10


def test_schedules_reach_every_phase_and_capacity_edge():
    """Taken together the schedules start a launch at every nonzero phase of some every >= 3, record two samples
    from a nonzero phase, fill the ring strictly inside a launch, have launches that record nothing, reset mid-phase
    and sample less often than a launch is long."""
    phases, two, inside, empty, mid_reset, long_every = {}, False, False, False, False, False
    for s in SCHEDULES.values():
        every, cap = s["every"], s["cap"]
        steps, _ = plan(s)
        long_every |= every > s["fused"]
        t = 0
        for op in s["steps"]:
            if op == "reset":
                mid_reset |= t % every != 0
                t = 0
                continue
            t += op
        for st in steps:
            for a, n, p, rec in st["launches"]:
                if every >= 3:
                    phases.setdefault(every, set()).add(p)
                two |= p != 0 and len(rec) >= 2
                empty |= not rec
                inside |= a < cap * every < a + n
    assert any(ph >= set(range(1, e)) for e, ph in phases.items()), phases
    assert two and inside and empty and mid_reset and long_every


def _sensitivity_keys():
    return [k for k, c in CASES.items() if c["math"] == "fast" and "chunk" not in c]


@pytest.mark.parametrize("key", _sensitivity_keys())
def test_one_tick_off_is_rejected_at_every_sampled_tick(oracle, key):
    """At every tick a FAST case samples, the oracle states one tick before and one tick after must fail the FAST
    comparison used at that tick: a sample in the wrong slot cannot hide inside the bound.  Reports the smallest
    rejected ratio (the accepted side is the GPU test, where the reference passes the same comparison)."""
    O = oracle
    c = CASES[key]
    ticks = set()
    for s, _ in c["runs"]:
        for st in plan(SCHEDULES[s], c["multi"], c["per_launch"])[0]:
            ticks.update(st["slots"])
    M = _world(key)[0][0].shape[0]
    sel = _select(M)[:64] if M > HEAD else _select(M)
    want, start, spec, S = _oracle_run(O, key, sel, max(ticks) + 1)

    def ratio(got, t):
        if S is None:
            return max(_fast_check(key, got, want[t], start, spec, S, t, check=False).values())
        try:
            return max(_fast_check(key, got, want[t], start, spec, S, t).values())
        except AssertionError:
            return np.inf

    rejected = np.inf
    for t in sorted(ticks):
        for u in (t - 1, t + 1):
            r = ratio(want[u], t)
            assert r > 1.0, f"{key}: the oracle state of tick {u} passes the comparison at tick {t} ({r:.3g})"
            rejected = min(rejected, r)
    print(f"\n{key}: one tick off is at least {rejected:.3g} x the bound (inf: an n-body check that raised)")
