"""Every FAST route over a long horizon, against an extended-precision restatement of the tick.

The per-tick FAST bound (1e-12, the route tests) cannot see a kernel that rounds one way systematically: a bias of an
ulp per evaluation of a force or an inverse inertia grows linearly in velocity and quadratically in position, while
unbiased rounding grows like sqrt(T).  So each FAST run here goes T = 1000 ticks and is judged against the truth,
tests/extended_reference.py at np.longdouble, next to the oracle's own f64 error (the f64 baseline: EXACT equals the
oracle bit for bit, and that is asserted too).

The measure.  For each world of the head (the first worlds of the batch: the first worlds of a larger batch are the
same bodies, so one truth serves every size of a case) and each quantity q, eps_q = max over the world's bodies of
the error against the truth, over the largest size of q in the world's truth: position |x|, linear velocity |v|,
angular velocity |w|, and the attitude as the angle between the two quaternions (radians, scale 1).  A FAST run
passes when, for every quantity,
  (a) RMS over the head of eps_FAST <= R RMS of eps_oracle + F,  R = 5, F = sqrt(T) 2^-52 (a random-walk floor), and
  (b) the contract of DESIGN §3 holds: max over the head of the vector-relative difference from the oracle <= 1e-9,
      over the worlds whose oracle run is within 1e-10 of the truth (the others are chaotic: see assert_long_horizon).

R and F are fixed by the CPU proof below, not by the GPU.  R comes from a noise model of an unbiased FAST kernel:
the f64 restatement with every result of eleven operations moved by +-1 ulp of random sign (the nine below, plus every
quaternion rotation and every quaternion normalisation, where FAST replaces the oracle's divisions and square roots
by approximations with Newton steps and contracts the products into FMAs; tests.extended_reference.Perturb).  Over
every GPU case whose truth costs under two minutes (all but the seven n-body worlds of N > 128) and two seeds, that
model's RMS eps is 0.65..2.9x the oracle's on 64-world heads and up to 3.2x (position) and 4.0x (attitude) on the
one-world n-body heads, whose RMS is a single world's error.  R = 5 is that envelope, 4.0, with a margin of 1.25; the
FAST kernels measure 0.7..1.9x on the H100 (DESIGN §6), inside it.  F = sqrt(T) ulps only matters where the oracle's
error is near zero (a torque-free angular velocity).  test_seeded_noise_passes_the_bound runs the model on every
fault case and on a one-world head.

Faults injected into the f64 restatement (each named operation's result scaled by 1 +- 2^-s) must fail (a) on their
case.  The state itself is rounded to f64 every tick, a random walk of sqrt(T) ulps of |x| and |v| in every run, so a
bias of 2^-52 of one force term is only visible where that term changes the state by many times its own size over T
ticks: on these worlds a 1-ulp bias reads 0.1..0.3 of the bound, and no route could be made to fail by one.  The
smallest bias 2^-s each fault's case rejects at both signs, measured at T = 1000, and the worst (a) ratio there:

  fault             case             smallest bias rejected   ratio at it
  g term            g, rk4           2^-42                    2.8
  thrust term       thrust, rk4      2^-44                    2.6
  drag term         drag, rk4        2^-42                    1.45
  frame gravity     frame, rk4       2^-44                    3.9
  J2 term           j2, rk4          2^-44                    3.6
  pair gravity      41x7 all-pairs   2^-44                    2.0
  1/m               g, semi          2^-42                    2.8
  1/I               wrench, rk4      2^-48                    1.6
  RK4 weight sum    g, rk4           2^-48                    1.3

No fault was dropped: each grows with T, none is undone by a renormalisation.  So an approximation that has lost a
Newton step (a bias of about 2^-44 and more) fails here; one that is biased by an ulp or a few does not.

The GPU cases import the catalogues of the route tests: SIGNATURES and INTERPRETED of test_body_routes (without
egm08, whose field kernel is the oracle's arithmetic in both modes) at their "small" and "pair" sizes, each one tick
per launch and with max_fused_ticks=50 (the loop-invariant reciprocals reused over 50 ticks of one launch); every
ROUTE of test_nbody_routes; small_world_kernel on both integrators with 64 ticks per launch; and the sparse
three-body graph alone3 of test_graph_routes (newton and softened).  n-body cases with N > 128 run 100 ticks with the
truth on one world (its cost is O(N^2) per stage in extended precision); the other n-body heads hold at most 2^14
body pairs.  The truths are computed once per module in a process pool.  Each case asserts its launch count per
step(); the kernel names at these shapes are proven by the route tests.
"""

import concurrent.futures as cf
import functools
import multiprocessing
import os
import time

import numpy as np
import pytest

if np.finfo(np.longdouble).nmant < 63:
    pytest.skip("np.longdouble is not x87 extended precision: no truth to judge f64 runs by", allow_module_level=True)

import elodin_b200 as el
from elodin_b200.executor import FORCE, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from oracle import oracle as _O
from tests import extended_reference as X
from tests.ensemble_util import need_gpu
from tests.test_body_routes import _head
from tests.util import body_effectors, max_rel

T = 1000
T_BIG = 100  # n-body worlds of more than 128 bodies
HEAD = 64
PAIRS_MAX = 1 << 14  # body pairs of an n-body head
R = 5.0
F_ULPS = 1.0
CONTRACT = 1e-9
EPS = 2.0 ** -52
QUANTITIES = ("pos", "vel", "omega", "attitude")
FUSED = 50
SMALL_FUSED = 64


# --------------------------------------------------------------------------- the measure


def _angle(q, qt):
    """Angle [M, N] between attitudes q (f64) and qt (truth), in extended precision."""
    a = tuple(np.asarray(q[..., k], dtype=np.longdouble) for k in range(4))
    b = tuple(np.asarray(qt[..., k], dtype=np.longdouble) for k in range(4))
    d = X.qmul(X.qinv(b), a)
    vec = np.sqrt(X.dot3(d, d))
    return 2.0 * np.arcsin(np.minimum(vec / np.sqrt(X.dot4(d, d)), 1.0))


def _rel(a, t):
    """max over bodies of |a - t|, over max over bodies of |t|: [M] (t, the truth, in extended precision)."""
    a = np.asarray(a, dtype=np.longdouble)
    err = np.sqrt(np.sum((a - t) ** 2, -1)).max(-1)
    scale = np.sqrt(np.sum(t * t, -1)).max(-1)
    return np.where(scale > 0, err / np.where(scale > 0, scale, 1), err)


def errors(state, truth):
    """{quantity: eps [M]} of a run's (pos, vel) against the truth's."""
    (p, v), (tp, tv) = state[:2], truth[:2]
    return {"pos": _rel(p[..., 4:], tp[..., 4:]), "vel": _rel(v[..., 3:], tv[..., 3:]),
            "omega": _rel(v[..., :3], tv[..., :3]), "attitude": _angle(p[..., :4], tp[..., :4]).max(-1)}


def _rms(a):
    return float(np.sqrt(np.mean(np.asarray(a, dtype=np.float64) ** 2)))


def bound_ratios(state, base, truth, ticks, with_base=False):
    """{quantity: RMS eps_run / (R RMS eps_base + F)} and {quantity: RMS eps_run / RMS eps_base} (and eps_base)."""
    er, eb = errors(state, truth), errors(base, truth)
    floor = F_ULPS * np.sqrt(ticks) * EPS
    ratio = {q: _rms(er[q]) / (R * _rms(eb[q]) + floor) for q in QUANTITIES}
    raw = {q: _rms(er[q]) / max(_rms(eb[q]), 1e-300) for q in QUANTITIES}
    return (ratio, raw, eb) if with_base else (ratio, raw)


def assert_long_horizon(state, base, truth, ticks, what):
    """(a) and (b) of the module docstring; returns the raw ratios RMS eps_FAST / RMS eps_oracle.  (b) is asserted on
    the worlds whose oracle run is itself within CONTRACT / 10 of the truth: where close encounters make a world
    chaotic (the unsoftened three-body graph), no f64 run can keep to 1e-9 of another, and (a) judges it alone."""
    ratio, raw, eb = bound_ratios(state, base, truth, ticks, with_base=True)
    for q in QUANTITIES:
        assert ratio[q] <= 1.0, (f"{what} {q}: RMS error against the truth is {raw[q]:.3g}x the oracle's "
                                 f"({ratio[q]:.3g}x the bound R RMS eps_oracle + F)")
    ok = np.all([np.asarray(eb[q], dtype=np.float64) <= CONTRACT / 10 for q in QUANTITIES], 0)
    assert np.any(ok), f"{what}: the oracle itself is more than {CONTRACT / 10} from the truth in every world"
    (p, v), (bp, bv) = (a[ok] for a in state[:2]), (a[ok] for a in base[:2])
    for q, a, b in (("pos", p[..., 4:], bp[..., 4:]), ("attitude", p[..., :4], bp[..., :4]),
                    ("vel", v[..., 3:], bv[..., 3:]), ("omega", v[..., :3], bv[..., :3])):
        d = max_rel(a, b)
        assert d <= CONTRACT, f"{what} {q}: {d:.3g} vector-relative from the oracle after {ticks} ticks (> {CONTRACT})"
    if not np.all(ok):
        print(f"\n{what}: (b) on {int(ok.sum())} of {ok.size} worlds; the oracle is more than {CONTRACT / 10} from the "
              f"truth in the others")
    return raw


# --------------------------------------------------------------------------- the cases


@functools.lru_cache(maxsize=4)
def case(key):
    """(full start (pos, vel, ine), effector spec, dt, integrator, ticks, head worlds) of a case key."""
    family, name, integ = key.split(":")
    if family == "body":
        from tests.test_body_routes import _sized

        start, spec, dt = _sized(name, "pair")
        return start, spec, dt, integ, T, min(HEAD, start[0].shape[0])
    if family in ("nbody", "small"):
        from tests.test_nbody_routes import DT, _setup

        M, N, extra = (int(x) for x in name.split("x"))
        (pos, vel, ine, _), _, ge, cols = _setup(None, M, N, bool(extra))
        spec = [("softened", {"edges": ge[0].edges, "k2": ge[0].k_squared, "soft": ge[0].softening})]
        if extra:
            spec.append(("thrust", {"thrust": cols["thrust"]}))
        big = N > 128
        return (pos, vel, ine), spec, DT, integ, T_BIG if big else T, 1 if big else min(M, HEAD, max(1, PAIRS_MAX // (N * N)))
    if family == "graph":
        from tests.test_graph_routes import _case

        start, spec, dt = _case("alone3", name)
        return start, spec, dt, integ, T, min(HEAD, start[0].shape[0])
    raise KeyError(key)


def head_case(key):
    start, spec, dt, integ, ticks, m = case(key)
    return (*_head(start, spec, m), dt, integ, ticks)


def _run_x(key, dtype, perturb=None, ticks=None):
    start, spec, dt, integ, t = head_case(key)
    return X.run(start, body_effectors(_O, spec)[0], integ, dt, ticks or t, dtype, perturb=perturb)


def truth_job(key):
    """(pos, vel) of the truth of a case at its horizon, and the seconds it took."""
    t0 = time.process_time()
    pos, vel, _, _ = _run_x(key, np.longdouble)
    return pos, vel, time.process_time() - t0


def oracle_run(O, key, ticks=None):
    """The oracle's (pos, vel, accel, force) of a case's head at its horizon."""
    start, spec, dt, integ, t = head_case(key)
    w = O.World(*start)
    oe = body_effectors(O, spec)[0]
    (w.rk4 if integ == "rk4" else w.semi_implicit)(dt, ticks or t, oe, threads=max(1, min(O.max_threads(), os.cpu_count() or 1)))
    return w.pos, w.vel, w.accel, w.force


def _pool():
    return cf.ProcessPoolExecutor(max_workers=max(1, min(os.cpu_count() or 1, 16)),
                                  mp_context=multiprocessing.get_context("spawn"))


# --------------------------------------------------------------------------- CPU: the f64 restatement is the oracle

SAMPLE = 100  # ticks between the states compared
WHEEL_COUNTS = (1, 8)


def _proof_spec(name):
    """(start, spec, dt) of a restatement case: every body-route list (2 worlds), the wheel fold at 1 and 8 wheels,
    and the edge gravity all-pairs (7 bodies) and over the irregular graph of test_graph_routes (7 and 40 bodies)."""
    if name.startswith("wheelcount"):
        from tests.util import near_world

        K = int(name[10:])
        pos, vel, ine, cols, dt = near_world(300 + K, 2, 3)
        tq = np.random.default_rng(K).normal(0, 1, (2, 3, 3 * K)) * np.tile(ine[..., :3], K)
        return (pos, vel, ine), [("gravity", {}), ("wheels", {"torques": tq}), ("thrust", {"thrust": cols["thrust"]})], dt
    if name.startswith("graph"):
        from tests.test_graph_routes import _case

        _, gname, kind = name.split("-")
        start, spec, dt = _case(gname, kind)
        return _head(start, spec, 2) + (dt,)
    if name == "allpairs7":
        from tests.test_nbody_routes import DT, _setup

        (pos, vel, ine, _), _, ge, cols = _setup(None, 3, 7, True)
        spec = [("softened", {"edges": ge[0].edges, "k2": ge[0].k_squared, "soft": ge[0].softening}),
                ("thrust", {"thrust": cols["thrust"]})]
        return (pos, vel, ine), spec, DT
    from tests.test_body_routes import _world

    start, spec, dt = _world(name, 2)
    return start, spec, dt


def _proof_names():
    from tests.test_body_routes import CASES

    return ([n for n in CASES if n != "egm08"] + [f"wheelcount{k}" for k in WHEEL_COUNTS] + ["allpairs7"]
            + [f"graph-{g}-{k}" for g in ("alone7", "alone40") for k in ("newton", "softened")])


def proof_job(name, integ):
    """The restatement's and the oracle's states every SAMPLE ticks up to T: the indices where they differ."""
    O = _O  # built by the parent (the oracle fixture) before any job runs
    O.set_dot_mode(0)
    start, spec, dt = _proof_spec(name)
    oe = body_effectors(O, spec)[0]
    got = X.run(start, oe, integ, dt, T, np.float64, every=SAMPLE)
    w = O.World(*start)
    diffs = []
    for k, g in enumerate(got):
        (w.rk4 if integ == "rk4" else w.semi_implicit)(dt, SAMPLE, oe)
        for q, a, b in zip(("pos", "vel", "accel", "force"), g, (w.pos, w.vel, w.accel, w.force)):
            if not np.array_equal(a, b):
                diffs.append(f"tick {(k + 1) * SAMPLE} {q}: max abs diff {np.max(np.abs(a - b)):.3g}")
    return diffs


@pytest.fixture(scope="module")
def pool(oracle):
    """One process pool for every CPU job of the module (spawned: the parent may hold a CUDA context).  The oracle
    fixture builds the oracle library once, in this process, before any worker loads it."""
    with _pool() as p:
        yield p


def truth_key(key):
    """The key whose truth a case shares: the small-world cases are n-body worlds of the same seed."""
    return key.replace("small:", "nbody:", 1)


class _Truths:
    """The truth of each case, computed once in the pool on first request (by a fault case or a GPU case); records
    the CPU seconds of the truths and the seconds the GPU tests spent on the device and waiting for a truth."""

    def __init__(self, pool):
        self.pool, self.futs = pool, {}
        self.t0 = time.perf_counter()
        self.cpu, self.wait, self.gpu = {}, 0.0, 0.0

    def submit(self, keys):
        for k in map(truth_key, keys):
            if k not in self.futs:
                self.futs[k] = self.pool.submit(truth_job, k)

    def __getitem__(self, key):
        key = truth_key(key)
        self.submit([key])
        t0 = time.perf_counter()
        pos, vel, cpu = self.futs[key].result()
        self.wait += time.perf_counter() - t0
        self.cpu[key] = cpu
        return pos, vel

    def report(self):
        print(f"\nlong-horizon truths: {len(self.cpu)} cases, {sum(self.cpu.values()):.0f} s of CPU (worst "
              f"{max(self.cpu.values(), default=0.0):.0f} s), {time.perf_counter() - self.t0:.0f} s wall since the "
              f"first submit; GPU runs {self.gpu:.0f} s, waiting for truths {self.wait:.0f} s")


@pytest.fixture(scope="module")
def truths(pool):
    t = _Truths(pool)
    yield t
    t.report()


@pytest.fixture(scope="module")
def proofs(pool):
    return {(n, i): pool.submit(proof_job, n, i) for n in _proof_names() for i in ("rk4", "semi_implicit")}


@pytest.mark.parametrize("integ", ("rk4", "semi_implicit"))
@pytest.mark.parametrize("name", _proof_names())
def test_f64_restatement_is_the_oracle(proofs, name, integ):
    """At np.float64 the restatement equals the oracle bit for bit on pos, vel, accel and force every 100 ticks up to
    1000: every effector kind, both wrench layouts, 3- and 5-wide wind, 1, 3 and 8 wheels, entity masks, and edge
    gravity (newton and softened) all-pairs and over an irregular graph."""
    diffs = proofs[(name, integ)].result()
    assert not diffs, f"{name} {integ}: " + "; ".join(diffs[:4])


def test_pow6_is_the_oracle_sixth_power():
    """J2's sixth power: the restated pow6 equals the oracle's correctly rounded double-double product, and sits
    within one rounding of the extended-precision power."""
    x = np.random.default_rng(3).uniform(6.0e6, 7.5e6, 4096)
    p = X.pow6_f64(x)
    exact = np.power(x.astype(np.longdouble), 6)
    assert np.all(np.abs(p - exact) <= 0.5 * np.spacing(p).astype(np.longdouble) * (1 + 1e-3))


# --------------------------------------------------------------------------- CPU: the bound catches bias, tolerates noise

# fault: (case key, bits s of the bias 2^-s it must reject on that case); s = 52 is one ulp
FAULTS = {
    "g": ("body:g:rk4", 42),
    "thrust": ("body:thrust:rk4", 44),
    "drag": ("body:drag:rk4", 42),
    "frame": ("body:frame:rk4", 44),
    "j2": ("body:j2:rk4", 44),
    "pair": ("nbody:41x7x0:rk4", 44),
    "inv_mass": ("body:g:semi_implicit", 42),
    "inv_inertia": ("body:wrench:rk4", 48),
    "rk4_weights": ("body:g:rk4", 48),
}
# the noise model also runs on a one-world head (an n-body route above 2^14 body pairs per world)
NOISE_ONLY = ("nbody:1x33x1:rk4",)
NOISE_SEED = 11


def fault_job(key, faults, truth):
    """{label: (bound ratios, raw ratios)} of the faulted runs of one case: each fault of `faults` [(name, bits)]
    at +- 2^-bits, and seeded +-1-ulp noise on every operation, against the case's truth (pos, vel)."""
    base = _run_x(key, np.float64)
    ticks = head_case(key)[4]
    out = {}
    for name, bits in faults:
        for sign in (1, -1):
            got = _run_x(key, np.float64, X.Perturb({name: 1.0 + sign * 2.0 ** -bits}))
            out[f"{name} {'+' if sign > 0 else '-'}2^-{bits}"] = bound_ratios(got, base, truth, ticks)
    got = _run_x(key, np.float64, X.Perturb(noise=NOISE_SEED))
    out["noise"] = bound_ratios(got, base, truth, ticks)
    return out


@pytest.fixture(scope="module")
def fault_results(pool, truths):
    jobs = {}
    for name, (key, bits) in FAULTS.items():
        jobs.setdefault(key, []).append((name, bits))
    for key in NOISE_ONLY:
        jobs.setdefault(key, [])
    truths.submit(list(jobs))
    futs = {key: pool.submit(fault_job, key, f, truths[key]) for key, f in jobs.items()}
    return {key: f.result() for key, f in futs.items()}


def test_each_fault_fails_the_bound(fault_results):
    """Every fault of FAULTS, at + and - its bias, fails (a) on its case in at least one quantity."""
    lines = []
    for name, (key, bits) in FAULTS.items():
        for sign in "+-":
            ratio, raw = fault_results[key][f"{name} {sign}2^-{bits}"]
            q = max(ratio, key=ratio.get)
            lines.append(f"{name} {sign}2^-{bits} on {key}: worst {q} {ratio[q]:.3g}x the bound ({raw[q]:.3g}x the oracle)")
            assert ratio[q] > 1.0, f"{name} {sign}2^-{bits} on {key} passes the bound: {ratio}"
    print("\n" + "\n".join(lines))


def test_seeded_noise_passes_the_bound(fault_results):
    """+-1 ulp of random sign on all eleven operations of the noise model, seeded: (a) holds on every fault case
    and on a one-world head."""
    lines = []
    for key, res in fault_results.items():
        ratio, raw = res["noise"]
        lines.append(f"noise on {key}: " + ", ".join(f"{q} {ratio[q]:.3g} ({raw[q]:.3g}x)" for q in QUANTITIES))
        assert max(ratio.values()) <= 1.0, f"seeded noise on {key} fails the bound: {ratio}"
    print("\n" + "\n".join(lines))


# --------------------------------------------------------------------------- GPU: every FAST route over T ticks

INTEGRATORS = ("rk4", "semi_implicit")


def _body_names():
    from tests.test_body_routes import INTERPRETED, SIGNATURES

    return [n for n in {**SIGNATURES, **INTERPRETED} if n != "egm08"]


def _routes():
    from tests.test_nbody_routes import ROUTES

    return ROUTES


def _route_key(route):
    (M, N), integ, extra, _, _ = route
    return f"nbody:{M}x{N}x{int(extra)}:{integ}"


def _gpu_keys():
    return ([f"body:{n}:{i}" for n in _body_names() for i in INTEGRATORS] + [_route_key(r) for r in _routes()]
            + [f"small:41x7x0:{i}" for i in INTEGRATORS] + [f"graph:{k}:{i}" for k in ("newton", "softened") for i in INTEGRATORS])


def _gpu(truths, start, spec, dt, integ, math, fused, ticks, m):
    """(pos, vel, accel, force) of the first m worlds after step(ticks) from start, and the launch count."""
    truths.submit(_gpu_keys())  # every GPU case's truth computes in the pool while the device runs
    t0 = time.perf_counter()
    M, N = start[0].shape[:2]
    _, ge, cols = body_effectors(None, spec)
    with el.B200Exec(N, M, dt, None, ge, integ, math, max_fused_ticks=fused) as ex:
        ex.set_state(*start, **cols)
        n0 = ex.timings()["kernel_launches"]
        ex.step(ticks, sync=True)
        n = ex.timings()["kernel_launches"] - n0
        st = tuple(ex.download(c)[:m] for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE))
    truths.gpu += time.perf_counter() - t0
    return st, n


def _assert_exact(truths, O, key):
    """EXACT on the case's head equals the oracle bit for bit at the horizon; returns the oracle's state."""
    start, spec, dt, integ, ticks = head_case(key)
    want = oracle_run(O, key)
    got, _ = _gpu(truths, start, spec, dt, integ, "exact", 1, ticks, start[0].shape[0])
    for q, a, b in zip(("pos", "vel", "accel", "force"), got, want):
        assert np.array_equal(a, b), f"{key} EXACT {q} after {ticks} ticks: max abs diff {np.max(np.abs(a - b)):.3g}"
    return want


def _report(key, worst):
    print(f"\n{key}: worst RMS eps_FAST / RMS eps_oracle " + ", ".join(f"{q} {r:.3g} ({lab})" for q, (r, lab) in worst.items()))


def _merge(worst, raw, label):
    for q, r in raw.items():
        if r > worst.get(q, (-1.0, ""))[0]:
            worst[q] = (r, label)


@pytest.mark.gpu
@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("name", _body_names())
def test_body_route_over_1000_ticks(oracle, truths, name, integ):
    """A body-route list at the "small" (one body per thread) and "pair" (body pairs) sizes, one tick per launch and
    50 ticks per launch (bit for bit equal), each against the truth and the oracle after 1000 ticks; EXACT on the
    head bit for bit."""
    need_gpu()
    from tests.test_body_routes import CASES, _small_worlds

    key = f"body:{name}:{integ}"
    start, spec, dt, _, ticks, m = case(key)
    base = _assert_exact(truths, oracle, key)
    finals, worst = {}, {}
    for size in ("small", "pair"):
        M = _small_worlds(CASES[name][1]) if size == "small" else start[0].shape[0]
        s, sp = _head(start, spec, M)
        for fused in (False, True):
            st, n = _gpu(truths, s, sp, dt, integ, "fast", FUSED if fused else 1, ticks, m)
            assert n == (-(-ticks // FUSED) if fused else ticks), f"{key} {size} fused={fused}: {n} launches"
            finals[(size, fused)] = st
        for q, a, b in zip(("pos", "vel", "accel", "force"), finals[(size, False)], finals[(size, True)]):
            assert np.array_equal(a, b), f"{key} {size}: {FUSED} ticks per launch differ from one in {q}"
    truth = truths[key]
    for size in ("small", "pair"):
        _merge(worst, assert_long_horizon(finals[(size, False)], base, truth, ticks, f"{key} {size}"), size)
    _report(key, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("route", _routes(), ids=[_route_key(r).split(":", 1)[1] for r in _routes()])
def test_nbody_route_over_1000_ticks(oracle, truths, route):
    """A route of test_nbody_routes, T ticks in one step() on its launch count, against the truth and the oracle;
    EXACT on the head bit for bit."""
    need_gpu()
    _, _, _, kernels, _ = route
    key = _route_key(route)
    start, spec, dt, integ, ticks, m = case(key)
    base = _assert_exact(truths, oracle, key)
    st, n = _gpu(truths, start, spec, dt, integ, "fast", 1, ticks, m)
    assert n == ticks * len(kernels), f"{key}: {n} launches for {ticks} ticks of {kernels}"
    worst = {}
    _merge(worst, assert_long_horizon(st, base, truths[key], ticks, key), "step")
    _report(key, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("key", [f"small:41x7x0:{i}" for i in INTEGRATORS]
                         + [f"graph:{k}:{i}" for k in ("newton", "softened") for i in INTEGRATORS])
def test_small_world_over_1000_ticks(oracle, truths, key):
    """small_world_kernel, 64 ticks per launch: 41 all-pairs worlds of 7 bodies and the irregular three-body graph of
    test_graph_routes, both integrators; EXACT bit for bit."""
    need_gpu()
    start, spec, dt, integ, ticks, m = case(key)
    base = _assert_exact(truths, oracle, key)
    st, n = _gpu(truths, start, spec, dt, integ, "fast", SMALL_FUSED, ticks, m)
    assert n == -(-ticks // SMALL_FUSED), f"{key}: {n} launches for {ticks} ticks"
    worst = {}
    _merge(worst, assert_long_horizon(st, base, truths[key], ticks, key), "step")
    _report(key, worst)
