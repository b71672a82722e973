"""Every FAST body-kernel route against the oracle, body by body (tests.util.assert_body_close).

The launcher picks the body kernel from the effector list (spec_signature: one compiled kernel per signature of
B200_SPEC_SIGS, the run-time interpreter body_fast_kernel for every other list), the range length (body pairs from
kPairMinBodies = 2 x 128 x 3 x 132 = 101 376 bodies up), the alignment of the planes (a range that starts at an odd
body takes one body per thread) and whether the launch records a trajectory (TRAJ).  Each case asserts the kernels
that ran, so a changed threshold or a signature that quietly falls back to the interpreter fails loudly.

The CPU tests at the top prove the bounds before any GPU run: every effector term scaled by 1 + 1e-8 must be
rejected (in all bodies and in one body), and so must a 1e-6 change of the force-driven displacement and a 1e-8
change of the torque-driven angular velocity; the oracle's golden-host rounding of the same run must be accepted.
"""

import functools
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200.executor import FORCE, INERTIA, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from tests.util import (assert_body_close, assert_route, body_effectors, body_scales, body_term_accels, body_terms,
                        launched_kernels, mutate_term, near_world, orbit_world)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TICKS = 2  # two launches of one tick: forward, then the planes walked in reverse
PAIR_MIN = 2 * 128 * 3 * 132  # kPairMinBodies
INTEGRATORS = ("rk4", "semi_implicit")
_I = {"rk4": 0, "semi_implicit": 1}
_BUILD = {"near": near_world, "orbit": orbit_world}


def _g(c):
    return ("gravity", {})


# name: (world, entities per world, effector list of the world's columns, signature value or None for the interpreter)
SIGNATURES = {
    "free": ("near", 3, lambda c: [], 0),
    "g": ("near", 1, lambda c: [_g(c)], 0),
    "drag": ("near", 1, lambda c: [("drag", {"wind": c["wind"]})], 1),
    "thrust": ("near", 3, lambda c: [_g(c), ("thrust", {"thrust": c["thrust"]})], 4),
    "wrench": ("near", 1, lambda c: [("wrench", {"wrench": c["wrench"]})], 8),
    "frame": ("orbit", 3, lambda c: [("frame", {})], 16),
    "thrust_drag": ("near", 3, lambda c: [_g(c), ("thrust", {"thrust": c["thrust"]}), ("drag", {"wind": c["wind"]})], 5),
    "thrust_drag_pb": ("near", 1, lambda c: [_g(c), ("thrust", {"thrust": c["thrust"]}), ("drag", {"wind": c["wind_pb"]})], 7),
    "thrust_wrench": ("near", 1, lambda c: [_g(c), ("thrust", {"thrust": c["thrust"]}), ("wrench", {"wrench": c["wrench"]})], 12),
    "frame_wrench": ("orbit", 3, lambda c: [("frame", {}), ("wrench", {"wrench": c["wrench"], "linear_first": True})], 24),
    "frame_wrench_torque_first": ("orbit", 1, lambda c: [("frame", {}), ("wrench", {"wrench": c["wrench"]})], 24),
    "j2": ("orbit", 3, lambda c: [("j2", {})], 64),
    "wheels_j2": ("orbit", 1, lambda c: [("wheels", {"torques": c["wheels"]}), ("j2", {})], 192),
    "wworld": ("near", 3, lambda c: [("wrench_world", {"wrench": c["wrench_world"]})], 256),
    "wheels_wworld": ("near", 1, lambda c: [("wheels", {"torques": c["wheels"]}), ("wrench_world", {"wrench": c["wrench_world"]})], 384),
}


def _egm08(c):
    from tests.test_oracle_golden import _egm08_random_tables

    cb, sb = _egm08_random_tables(8, np.random.default_rng(5))
    return [("egm08", {"c_bar": cb, "s_bar": sb, "L": 8})]


# lists no signature covers: the interpreter body_fast_kernel
INTERPRETED = {
    "masked": ("near", 3, lambda c: [_g(c), ("thrust", {"thrust": c["thrust"], "mask": [1, 0, 1]}),
                                     ("drag", {"wind": c["wind"], "mask": [0, 1, 1]})], None),
    "wrench_then_drag": ("near", 1, lambda c: [("wrench", {"wrench": c["wrench"]}), ("drag", {"wind": c["wind"]}),
                                               ("thrust", {"thrust": c["thrust"]})], None),
    "g_then_wheels": ("near", 3, lambda c: [_g(c), ("wheels", {"torques": c["wheels"]})], None),
    "two_thrusts": ("near", 1, lambda c: [("thrust", {"thrust": c["thrust"]}),
                                          ("thrust", {"thrust": c["thrust2"], "axis": (0.0, 0.6, 0.8), "name": "thrust2"})], None),
    "frame_j2": ("orbit", 3, lambda c: [("frame", {}), ("j2", {})], None),
    "egm08": ("orbit", 1, _egm08, None),
}
CASES = {**SIGNATURES, **INTERPRETED}
MISALIGNED = ("free", "thrust_drag", "frame_wrench")  # three entities per world


def _pair_worlds(N):
    """The fewest worlds of N entities whose body count is odd and at least PAIR_MIN + 1."""
    M = -(-(PAIR_MIN + 1) // N)
    return M + (M * N % 2 == 0)


def _small_worlds(N):
    return 301 // N


@functools.lru_cache(maxsize=2)
def _world(name, M):
    """(start = (pos, vel, ine), effector list, dt) of case `name` with M worlds; the first worlds of a larger
    batch are the same bodies, so one oracle run serves every size."""
    fam, N, spec_of, _ = CASES[name]
    pos, vel, ine, cols, dt = _BUILD[fam](9000 + 17 * sorted(CASES).index(name), M, N)
    return (pos, vel, ine), spec_of(cols), dt


def _head(start, spec, m):
    """The first m worlds of a batch: state and effector columns."""
    cut = lambda a: a[:m] if isinstance(a, np.ndarray) and a.ndim == 3 else a
    return tuple(a[:m] for a in start), [(k, {n: cut(v) for n, v in kw.items()}) for k, kw in spec]


def _oracle(O, start, oe, integ, dt, ticks):
    """The oracle's (pos, vel, accel, force) after each tick 1..ticks."""
    w = O.World(*start)
    out = []
    for _ in range(ticks):
        (w.rk4 if integ == "rk4" else w.semi_implicit)(dt, 1, oe, threads=max(1, min(O.max_threads(), os.cpu_count() or 1)))
        out.append(tuple(a.copy() for a in (w.pos, w.vel, w.accel, w.force)))
    return out


def _cut(state, m):
    return tuple(a[:m] for a in state)


# --------------------------------------------------------------------------- runs on the device

# a run: (size, fused, trajectory planes); size "small" = a few hundred bodies, "pair" = past kPairMinBodies
RUNS = [(size, fused, traj) for size in ("small", "pair") for fused, traj in ((False, 0), (True, 0), (False, 13), (True, 25))]


def _spec_kernel(integ, sig, traj, pair):
    return f"body_fast_spec_kernel<{_I[integ]}, {sig}, {'true' if traj else 'false'}, 128, {'3, 2' if pair else '4, 1'}>"


def _interp_kernel(integ, traj):
    return f"body_fast_kernel<{_I[integ]}, 128, 4, {'true' if traj else 'false'}>"


def _expected(name, integ, run, no_spec=False):
    size, _, traj = run
    sig = CASES[name][3]
    if sig is None or no_spec:
        return [_interp_kernel(integ, traj)] + (["egm08_force_kernel<"] if name == "egm08" else [])
    return [_spec_kernel(integ, sig, traj, size == "pair")]


def _open(start, spec, dt, integ, run, math="fast", chunk=0):
    """A handle with the state of `start` set, for one run."""
    _, fused, traj = run
    pos = start[0]
    M, N = pos.shape[:2]
    _, ge, cols = body_effectors(None, spec)
    kw = dict(max_fused_ticks=TICKS if fused else 1, invoke_chunk_bodies=chunk)
    if traj:
        kw.update(trajectory_every=1, trajectory_capacity=TICKS, trajectory_full=traj == 25)
    ex = el.B200Exec(N, M, dt, None, ge, integ, math, **kw)
    if chunk:
        ex._cols = cols
    else:
        ex.set_state(*start, **cols)
    return ex


def _state(ex):
    return tuple(ex.download(c) for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE))


def _table(ex, start, dt):
    pos, vel, ine = start
    M, N = pos.shape[:2]
    t = {el.component_id("tick"): np.array([0], dtype=np.uint64), FORCE: np.zeros((M, N, 6)), INERTIA: ine,
         WORLD_POS: pos, WORLD_ACCEL: np.zeros((M, N, 6)), el.component_id("simulation_time_step"): np.array([dt]),
         WORLD_VEL: vel}
    t.update({el.component_id(k): v for k, v in ex._cols.items()})
    return [t[c] for c in ex.input_ids]


def _go(ex, start, dt, chunk):
    """Advance TICKS ticks (step(), or invoke_batch through ranges of `chunk` bodies); returns the launch count and
    the final state (None for step(): download it afterwards)."""
    n0 = ex.timings()["kernel_launches"]
    if chunk:
        out = dict(zip(ex.output_ids, ex.invoke_batch(_table(ex, start, dt), TICKS)))
        return ex.timings()["kernel_launches"] - n0, (out[WORLD_POS], out[WORLD_VEL], out[WORLD_ACCEL], out[FORCE])
    ex.step(TICKS, sync=True)
    return ex.timings()["kernel_launches"] - n0, None


def _sized(name, size):
    """(start, effector list, dt) of case `name` at a size: "small" = a few hundred bodies (one body per thread),
    "pair" = past kPairMinBodies (body pairs), "misaligned" = two pipelined invoke_batch ranges of that size."""
    N = CASES[name][1]
    if size == "misaligned":
        return _world(name, 2 * _pair_worlds(N))
    big = _world(name, _pair_worlds(N))
    if size == "pair":
        return big
    start, spec, dt = big
    return (*_head(start, spec, _small_worlds(N)), dt)


def _chunk(name):
    """invoke_chunk_bodies of the misaligned case: invoke_batch turns it into whole worlds per range (and, for N = 1,
    a multiple of 128 worlds), so only an odd N > 1 can start the second range at an odd body."""
    N = CASES[name][1]
    assert N % 2 == 1 and N > 1, name
    return _pair_worlds(N) * N


def _do_job(job, out_path, attempts=4):
    """Run one job's runs on fresh handles, all in one profiling window, and write per run: the kernel names it
    launched, its launch count, and what it computed (the final state, or the trajectory of a recording run).  An
    attempt counts only when the profiler saw every launch the library counted; each retry waits longer after the
    last launch before it closes the window (a window of two short EXACT launches lost its records repeatedly)."""
    key, name, integ, math, runs = job
    for attempt in range(attempts):
        handles, counts, outs = [], [], []
        for run in runs:
            start, spec, dt = _exact_world(name) if math == "exact" else _sized(name, run[0])
            chunk = _chunk(name) if run[0] == "misaligned" else 0
            handles.append((_open(start, spec, dt, integ, run, math, chunk), start, dt, chunk))

        def go():
            for ex, start, dt, chunk in handles:
                n, st = _go(ex, start, dt, chunk)
                counts.append(n)
                outs.append(st)

        _, names = launched_kernels(go, settle=0.05 * 5 ** attempt)
        names = [n for n in names if not n.startswith(("Memcpy", "Memset"))]
        if len(names) == sum(counts) or attempt == attempts - 1:
            break
        for ex, *_ in handles:
            ex.close()
    res, k = {"ok": len(names) == sum(counts)}, 0
    for r, ((ex, *_), n, st, run) in enumerate(zip(handles, counts, outs, runs)):
        res[f"{r}_names"] = np.array(names[k:k + n], dtype=str)
        res[f"{r}_launches"] = n
        k += n
        if run[2]:
            res[f"{r}_traj"] = ex.trajectory()
        else:
            res[f"{r}_state"] = np.concatenate(st if st is not None else _state(ex), -1)
        ex.close()
    np.savez(out_path, **res)


def _worker(out_dir):
    """Child process: one job per line of stdin (JSON), its results in out_dir/<job key>.npz, then 'DONE <path>'."""
    for line in sys.stdin:
        key, name, integ, math, runs = json.loads(line)
        path = os.path.join(out_dir, key + ".npz")
        _do_job((key, name, integ, math, [tuple(r) for r in runs]), path)
        print("DONE", path, flush=True)


class _Worker:
    """A child process that runs jobs for this module's tests (with B200_NO_SPEC=1 and B200_EXACT_CFG=12 when
    `no_spec`).  The B200_* route switches are read once per process, and torch.profiler loses launch records of
    short windows more often once a process has run other CUDA work, so the launches run there, and only there: the
    tests read back what they computed."""

    def __init__(self, out_dir, no_spec):
        env = {k: v for k, v in os.environ.items() if not k.startswith("B200_")}
        if no_spec:
            env.update(B200_NO_SPEC="1", B200_EXACT_CFG="12")
        self.what = "B200_NO_SPEC=1" if no_spec else "default"
        self.err_path = os.path.join(out_dir, "stderr.txt")
        self.err = open(self.err_path, "w")
        code = "import sys; from tests.test_body_routes import _worker; _worker(sys.argv[1])"
        argv = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, str(out_dir)]
        self.p = subprocess.Popen(argv, cwd=ROOT, env=env, stdin=subprocess.PIPE, stdout=subprocess.PIPE,
                                  stderr=self.err, text=True)

    def submit(self, job):
        self.p.stdin.write(json.dumps(job) + "\n")
        self.p.stdin.flush()

    def result(self, key):
        """The results of job `key` (replies of jobs an earlier failed test left unread are dropped)."""
        for line in self.p.stdout:
            if not line.startswith("DONE "):
                continue
            path = line[5:].strip()
            with np.load(path) as z:
                res = {k: z[k] for k in z.files}
            os.remove(path)
            if os.path.basename(path) == key + ".npz":
                return res
        self.p.wait()
        with open(self.err_path) as f:
            raise AssertionError(f"{self.what} child ended ({self.p.returncode}):\n{f.read()[-4000:]}")

    def close(self):
        try:
            self.p.stdin.close()
            self.p.wait(timeout=120)
        except Exception:
            self.p.kill()
            self.p.wait()
        self.err.close()


@pytest.fixture(scope="module")
def workers(tmp_path_factory):
    """{no_spec: _Worker}: the default build's routes and the B200_NO_SPEC=1 / B200_EXACT_CFG=12 ones, side by side."""
    w = {ns: _Worker(tmp_path_factory.mktemp("body_routes_no_spec" if ns else "body_routes"), ns) for ns in (False, True)}
    yield w
    for x in w.values():
        x.close()


def _names(res, r, kernels, what):
    assert bool(res["ok"]), f"{what}: the profiler lost launch records in every attempt"
    assert_route(list(res[f"{r}_names"]), kernels, what)


def _state_of(res, r):
    a = res[f"{r}_state"]
    return a[..., :7], a[..., 7:13], a[..., 13:19], a[..., 19:25]


def _traj_state(sample, want):
    """A trajectory sample as (pos, vel, accel, force); a 13-plane sample carries no accel / force: take want's."""
    if sample.shape[-1] == 25:
        return sample[..., :7], sample[..., 7:13], sample[..., 13:19], sample[..., 19:25]
    return sample[..., :7], sample[..., 7:13], want[2], want[3]


def _merge(worst, new, label):
    for q, r in new.items():
        if r > worst.get(q, (-1.0, ""))[0]:
            worst[q] = (r, label)


def _report(key, worst, kernels):
    print(f"\n{key}: kernels {sorted(set(kernels))}; worst error / bound "
          + ", ".join(f"{q} {r:.3g} ({lab})" for q, (r, lab) in worst.items()))


# --------------------------------------------------------------------------- GPU: the compiled signatures


@pytest.mark.gpu
@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("name", list(SIGNATURES))
def test_signature_routes_match_the_oracle(oracle, workers, name, integ):
    """One body per thread and body pairs; one tick per launch (two launches, the second walking the planes in
    reverse) and all ticks fused in one launch, bit for bit equal; a trajectory sample every tick with 13 and 25
    planes; and the interpreter kernel (B200_NO_SPEC=1) at pair size.  Every result against the oracle body by body."""
    O = oracle
    N = CASES[name][1]
    key = f"{name}-{integ}"
    workers[False].submit((key, name, integ, "fast", RUNS))
    workers[True].submit((key, name, integ, "fast", [("pair", False, 0)]))
    start, spec, dt = _sized(name, "pair")
    want = _oracle(O, start, body_effectors(O, spec)[0], integ, dt, TICKS)
    res, res_ns = workers[False].result(key), workers[True].result(key)
    worst, finals, kernels = {}, {}, []
    for r, run in enumerate(RUNS):
        size, fused, traj = run
        what = f"{key} {run}"
        kernels += _expected(name, integ, run)
        _names(res, r, _expected(name, integ, run), what)
        assert int(res[f"{r}_launches"]) == (1 if fused else TICKS), what
        m = _small_worlds(N) if size == "small" else start[0].shape[0]
        s0, sp = _head(start, spec, m)
        sc = body_scales(sp, *s0)
        if traj:  # sample k against the oracle after k + 1 ticks; the last sample is the final state
            for k in range(TICKS):
                w = _cut(want[k], m)
                _merge(worst, assert_body_close(_traj_state(res[f"{r}_traj"][k], w), w, s0, dt, k + 1, sc,
                                                what=f"{what} sample {k}"), what)
        else:
            finals[(size, fused)] = _state_of(res, r)
            _merge(worst, assert_body_close(finals[(size, fused)], _cut(want[-1], m), s0, dt, TICKS, sc, what=what), what)
    for size in ("small", "pair"):
        for a, b, q in zip(finals[(size, False)], finals[(size, True)], ("pos", "vel", "accel", "force")):
            assert np.array_equal(a, b), f"{key} {size}: fused {q} differs from one tick per launch"
    kernels += _expected(name, integ, ("pair", False, 0), no_spec=True)
    _names(res_ns, 0, _expected(name, integ, ("pair", False, 0), no_spec=True), f"{key} B200_NO_SPEC")
    _merge(worst, assert_body_close(_state_of(res_ns, 0), want[-1], start, dt, TICKS, body_scales(spec, *start),
                                    what=f"{key} interpreter"), "interpreter")
    _report(key, worst, kernels)


# --------------------------------------------------------------------------- GPU: misaligned ranges, interpreter lists


@pytest.mark.gpu
@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("name", MISALIGNED)
def test_misaligned_range_takes_the_one_body_kernel(oracle, workers, name, integ):
    """Pipelined invoke_batch over 2 x 33 793 worlds of 3 bodies in ranges of 33 793 worlds (101 379 bodies, one
    wave of pairs and more).  The first range starts at body 0 and runs body pairs with an odd tail; the second starts
    at body 101 379, so its planes are not 16-byte aligned (and it does not start on a 64-body segment of the
    mass-class summary): it takes one body per thread.  The tick kernels must run in that order."""
    O = oracle
    key = f"misaligned-{name}-{integ}"
    workers[False].submit((key, name, integ, "fast", [("misaligned", False, 0)]))
    start, spec, dt = _sized(name, "misaligned")
    assert start[0].shape[0] * CASES[name][1] == 2 * _chunk(name) and _chunk(name) % 2 == 1
    want = _oracle(O, start, body_effectors(O, spec)[0], integ, dt, TICKS)[-1]
    res = workers[False].result(key)
    sig = CASES[name][3]
    order = [_spec_kernel(integ, sig, False, True)] * TICKS + [_spec_kernel(integ, sig, False, False)] * TICKS
    _names(res, 0, order, key)
    ticks = [n for n in res["0_names"] if n.startswith(("body_fast_spec_kernel<", "body_fast_kernel<"))]
    assert len(ticks) == len(order) and all(n.startswith(e) for n, e in zip(ticks, order)), \
        f"{key}: tick kernels in launch order {ticks}, expected {order}"
    worst = {}
    _merge(worst, assert_body_close(_state_of(res, 0), want, start, dt, TICKS, body_scales(spec, *start), what=key), key)
    _report(key, worst, order)


@pytest.mark.gpu
@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("name", list(INTERPRETED))
def test_interpreter_lists_match_the_oracle(oracle, workers, name, integ):
    """Lists no signature covers run body_fast_kernel (EGM08 also egm08_force_kernel): one tick per launch, and
    fused with a full trajectory sample every tick."""
    O = oracle
    key = f"{name}-{integ}"
    runs = [("small", False, 0), ("small", True, 25)]
    workers[False].submit((key, name, integ, "fast", runs))
    start, spec, dt = _sized(name, "small")
    want = _oracle(O, start, body_effectors(O, spec)[0], integ, dt, TICKS)
    sc = body_scales(spec, *start)
    res = workers[False].result(key)
    worst, kernels = {}, []
    for r, run in enumerate(runs):
        what = f"{key} {run}"
        kernels += _expected(name, integ, run)
        _names(res, r, _expected(name, integ, run), what)
        if run[2]:
            for k in range(TICKS):
                _merge(worst, assert_body_close(_traj_state(res[f"{r}_traj"][k], want[k]), want[k], start, dt, k + 1, sc,
                                                what=f"{what} sample {k}"), what)
        else:
            _merge(worst, assert_body_close(_state_of(res, r), want[-1], start, dt, TICKS, sc, what=what), what)
    _report(key, worst, kernels)


# --------------------------------------------------------------------------- GPU: EXACT sequences, bit for bit

# every effector sequence of B200_EXACT_SEQS: (world, entities, list, sequence value)
EXACT_SEQS = {
    "empty": ("near", 3, lambda c: [], 0),
    "g": ("near", 3, lambda c: [_g(c)], 1),
    "g_drag": ("near", 1, lambda c: [_g(c), ("drag", {"wind": c["wind"]})], 0x21),
    "g_thrust_drag": ("near", 3, lambda c: [_g(c), ("thrust", {"thrust": c["thrust"]}), ("drag", {"wind": c["wind"]})], 0x231),
    "g_thrust_wrench": ("near", 1, lambda c: [_g(c), ("thrust", {"thrust": c["thrust"]}), ("wrench", {"wrench": c["wrench"]})], 0x431),
    "frame_wrench": ("orbit", 3, lambda c: [("frame", {}), ("wrench", {"wrench": c["wrench"], "linear_first": True})], 0x45),
    "newton": ("near", 40, lambda c: [("newton", {"edges": el.all_pairs_edges(40)})], 6),
    "softened": ("near", 40, lambda c: [("softened", {"edges": el.all_pairs_edges(40), "k2": 0.2, "soft": 1e-5})], 7),
    "wheels_wworld": ("near", 3, lambda c: [("wheels", {"torques": c["wheels"]}), ("wrench_world", {"wrench": c["wrench_world"]})], 0x89),
}


def _exact_world(name):
    fam, N, spec_of, _ = EXACT_SEQS[name]
    pos, vel, ine, cols, dt = _BUILD[fam](4000 + 31 * sorted(EXACT_SEQS).index(name), max(1, 90 // N), N)
    return (pos, vel, ine), spec_of(cols), dt


def _exact_kernels(name, integ, interpreted):
    seq = 0xFFFFFFFF if interpreted else EXACT_SEQS[name][3]
    body = f"body_exact_kernel<0, 128, 4, false, {seq}>" if integ == "rk4" else f"body_exact_kernel<1, 256, 1, false, {seq}>"
    return [body] + ([f"graph_dense_kernel<true, {'true' if integ == 'rk4' else 'false'}>"] if EXACT_SEQS[name][1] == 40 else [])


@pytest.mark.gpu
@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("name", list(EXACT_SEQS))
def test_exact_sequences_are_bit_exact(oracle, workers, name, integ):
    """Each compiled EXACT sequence, and the EXACT interpreter (B200_EXACT_CFG=12) on the same list: bit for bit."""
    O = oracle
    key = f"exact-{name}-{integ}"
    for ns in (False, True):
        workers[ns].submit((key, name, integ, "exact", [("small", False, 0)]))
    start, spec, dt = _exact_world(name)
    want = _oracle(O, start, body_effectors(O, spec)[0], integ, dt, TICKS)[-1]
    for ns in (False, True):
        res = workers[ns].result(key)
        label = "interpreter (B200_EXACT_CFG=12)" if ns else "sequence"
        _names(res, 0, _exact_kernels(name, integ, ns), f"{key} {label}")
        for q, x, y in zip(("pos", "vel", "accel", "force"), _state_of(res, 0), want):
            assert np.array_equal(x, y), f"{key} {label} {q}: max abs diff {np.max(np.abs(x - y))}"


# --------------------------------------------------------------------------- CPU: the bounds are sensitive and not tight

CPU_BODIES = 129  # odd: the tail body of a pair launch, pair (0, 1) and body 63 of the first 64-body segment


def _cpu_case(name):
    fam, N, spec_of, _ = CASES[name]
    pos, vel, ine, cols, dt = _BUILD[fam](500 + 3 * sorted(CASES).index(name), CPU_BODIES // N, N)
    return (pos, vel, ine), spec_of(cols), dt


def _run_oracle(O, start, oe, integ, dt, ticks=TICKS):
    return _oracle(O, start, oe, integ, dt, ticks)[-1]


def _rejects(got, want, start, dt, sc):
    try:
        assert_body_close(got, want, start, dt, TICKS, sc)
    except AssertionError:
        return True
    return False


def _splice(base, other, b):
    """base with body b (flat index) taken from other: what a run whose mutation touched body b alone gives."""
    out = tuple(a.copy() for a in base)
    for o, x in zip(out, other):
        o.reshape(-1, o.shape[-1])[b] = x.reshape(-1, x.shape[-1])[b]
    return out


@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("name", list(CASES))
def test_bounds_reject_every_term_scaled_by_1e_8(oracle, name, integ):
    """Every term of the list scaled by 1 + 1e-8 must fail assert_body_close, in all bodies and in one body alone
    (the odd tail body, the second body of a pair, body 63 of a 64-body segment)."""
    O = oracle
    start, spec, dt = _cpu_case(name)
    sc = body_scales(spec, *start)
    want = _run_oracle(O, start, body_effectors(O, spec)[0], integ, dt)
    assert not _rejects(want, want, start, dt, sc)
    for i, term in body_terms(spec):
        got = _run_oracle(O, start, mutate_term(O, spec, i, term, 1.0 + 1e-8), integ, dt)
        assert _rejects(got, want, start, dt, sc), f"{name} {integ}: {term} scaled by 1 + 1e-8 passes"
        # for a masked term: the bodies that carry it
        mask = spec[i][1].get("mask")
        N = start[0].shape[1]
        for b in (CPU_BODIES - 1, 1, 63):
            if mask is not None and not mask[b % N]:
                b = next(c for c in (b + 1, b - 1, b + 2, b - 2) if mask[c % N])
            assert _rejects(_splice(want, got, b), want, start, dt, sc), f"{name} {integ}: {term} in body {b} alone passes"


@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("name", list(CASES))
def test_bounds_reject_small_position_and_angular_velocity_errors(oracle, name, integ):
    """Positions moved by 1e-6 of the force-driven displacement, and omega changed by 1e-8 of the torque-driven
    change, must fail assert_body_close."""
    O = oracle
    start, spec, dt = _cpu_case(name)
    sc = body_scales(spec, *start)
    want = _run_oracle(O, start, body_effectors(O, spec)[0], integ, dt)
    pos0, vel0, _ = start
    disp = want[0][..., 4:] - pos0[..., 4:] - TICKS * dt * vel0[..., 3:]
    if np.any(sc[0] > 0):
        p = want[0].copy()
        p[..., 4:] += 1e-6 * disp
        assert _rejects((p,) + want[1:], want, start, dt, sc), f"{name} {integ}: positions off by 1e-6 of the displacement pass"
    if np.any(sc[1] > 0):
        v = want[1].copy()
        v[..., :3] += 1e-8 * (want[1][..., :3] - vel0[..., :3])
        assert _rejects((want[0], v) + want[2:], want, start, dt, sc), f"{name} {integ}: omega off by 1e-8 of its change passes"


def test_bounds_accept_the_golden_host_rounding(oracle):
    """The oracle in golden-host mode (FMA-contracted quaternion dots) is a legitimately different rounding of the
    same run: assert_body_close must accept it on every case.  Reports the worst ratio to the bound."""
    O = oracle
    worst = {}
    try:
        for integ in INTEGRATORS:
            for name in CASES:
                start, spec, dt = _cpu_case(name)
                oe = body_effectors(O, spec)[0]
                O.set_dot_mode(0)
                want = _run_oracle(O, start, oe, integ, dt)
                O.set_dot_mode(1)
                got = _run_oracle(O, start, oe, integ, dt)
                _merge(worst, assert_body_close(got, want, start, dt, TICKS, body_scales(spec, *start), what=f"{name} {integ}"),
                       f"{name} {integ}")
    finally:
        O.set_dot_mode(0)
    print("\ngolden-host rounding, worst error / bound: " + ", ".join(f"{q} {r:.3g} ({lab})" for q, (r, lab) in worst.items()))


@pytest.mark.parametrize("family", ["near", "orbit"])
def test_body_scales_match_the_oracle_stage(oracle, family):
    """The closed forms of body_term_accels against oracle.World.eval_stage, one effector (or one part of it) at a
    time."""
    O = oracle
    pos, vel, ine, cols, _ = _BUILD[family](77, 4, 3)
    if family == "near":
        single = [("gravity", {}, "g"), ("thrust", {"thrust": cols["thrust"]}, "thrust"), ("drag", {"wind": cols["wind"]}, "drag"),
                  ("drag", {"wind": cols["wind_pb"]}, "drag"), ("wrench_world", {"wrench": cols["wrench_world"]}, None),
                  ("wrench", {"wrench": cols["wrench"]}, None), ("wheels", {"torques": cols["wheels"]}, "wheels")]
    else:
        single = [("wrench", {"wrench": cols["wrench"], "linear_first": True}, None), ("frame", {"omega": (0.0, 0.0, 0.0)}, "central"),
                  ("j2", {"j2": 0.0}, "j2_central")]
    w = O.World(pos, vel, ine)
    for kind, kw, term in single:
        for world in range(pos.shape[0]):
            _, A = w.eval_stage(world, body_effectors(O, [(kind, kw)])[0])
            lin, ang = np.sqrt(np.sum(A[:, 3:] ** 2, -1)), np.sqrt(np.sum(A[:, :3] ** 2, -1))
            if term is None:  # both parts of a wrench
                parts = [body_term_accels(kind, kw, t, pos, vel, ine) for _, t in body_terms([(kind, kw)])]
                want_lin, want_ang = sum(p[0] for p in parts)[world], sum(p[1] for p in parts)[world]
            else:
                want_lin, want_ang = (a[world] for a in body_term_accels(kind, kw, term, pos, vel, ine))
            np.testing.assert_allclose(lin, want_lin, rtol=1e-12, err_msg=f"{kind} {term}")
            np.testing.assert_allclose(ang, want_ang, rtol=1e-12, atol=1e-300, err_msg=f"{kind} {term}")
    if family == "orbit":  # Coriolis and centrifugal as differences of frame accelerations; J2 beside its central term
        v0 = vel.copy()
        v0[..., 3:] = 0.0
        frame = body_effectors(O, [("frame", {"mu": 0.0})])[0]
        j2, j2c = (body_effectors(O, [("j2", kw)])[0] for kw in ({}, {"j2": 0.0}))
        for world in range(pos.shape[0]):
            a_full = w.eval_stage(world, frame)[1][:, 3:]
            a_cent = O.World(pos, v0, ine).eval_stage(world, frame)[1][:, 3:]
            a_j2 = w.eval_stage(world, j2)[1][:, 3:] - w.eval_stage(world, j2c)[1][:, 3:]
            for term, a, rtol in (("centrifugal", a_cent, 1e-12), ("coriolis", a_full - a_cent, 1e-9), ("j2", a_j2, 1e-6)):
                want = body_term_accels("frame" if term != "j2" else "j2", {}, term, pos, vel, ine)[0][world]
                np.testing.assert_allclose(np.sqrt(np.sum(a * a, -1)), want, rtol=rtol, err_msg=term)
