"""Reaction-wheel torque folds of 1..8 wheels against the oracle, with both integrators and both math modes.

TorqueBodyFold takes 1..8 wheels (a column of 3 K doubles).  The FAST body kernel compiles the fold only for three
wheels first in the list (SIG_WHEELS, beside J2 or a world wrench); every other count runs the interpreter
body_fast_kernel.  EXACT math compiles the cube-sat replay sequence (wheels, then a world wrench) whatever the wheel
count, since a sequence is keyed on effector kinds; every other list runs the EXACT interpreter.

Each list is fed through set_state, a small invoke_batch (one packed layout launch) and a pipelined invoke_batch whose
ranges start at odd bodies.  EXACT must equal the oracle bit for bit; FAST is checked body by body with
tests.util.assert_body_close, where the wheel term's scale is the sum of the wheels' own torques, sum_k |tau_k|: the
kernels sum the wheels in their own order and rounding, which is bounded relative to that sum and not to |sum_k tau_k|,
which collapses when wheels oppose each other (the "opposed" list: the second half of the wheels negates the first).
The CPU tests at the bottom prove that bound sensitive: one wheel scaled by 1 + 1e-8, or the last wheel dropped, must
be rejected, and the wheels folded in reverse order (a legitimate reordering of the sum) must be accepted.
"""

import os

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200.executor import FORCE, INERTIA, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from tests.util import (assert_body_close, assert_route, body_effectors, body_term_accels, body_terms, launched_kernels,
                        near_world, orbit_world, run_child)

TICKS = 2
M, N = 43, 3  # 129 bodies: an odd tail body, and pipelined ranges of 21 worlds start at odd bodies
CHUNK = 21 * N
INTEGRATORS = ("rk4", "semi_implicit")
_I = {"rk4": 0, "semi_implicit": 1}
_BUILD = {"near": near_world, "orbit": orbit_world}
WHEELS = range(1, 9)

# name: (world, effector list of the world's columns; "tq" is the wheel-torque column)
LISTS = {
    "alone": ("near", lambda c: [("wheels", {"torques": c["tq"]})]),
    "after_g": ("near", lambda c: [("gravity", {}), ("wheels", {"torques": c["tq"]})]),
    "wworld": ("near", lambda c: [("wheels", {"torques": c["tq"]}), ("wrench_world", {"wrench": c["wrench_world"]})]),
    "j2": ("orbit", lambda c: [("wheels", {"torques": c["tq"]}), ("j2", {})]),
    "opposed": ("near", lambda c: [("wheels", {"torques": c["tq"]}), ("wrench_world", {"wrench": c["wrench_world"]})]),
}
CASES = [(K, name) for K in WHEELS for name in LISTS if name != "opposed" or K % 2 == 0]


def _world(K, name, n_worlds=M):
    """(start = (pos, vel, ine), effector list, dt) of K wheels on list `name`.  Wheel torques are ~1 rad/s^2 each
    near the origin and ~0.02 rad/s^2 in orbit (near_world / orbit_world's nine-wheel scale); "opposed" wheels are
    [t_1 .. t_K/2, -t_1 .. -t_K/2], whose sum is 0 up to the rounding of its order."""
    fam, spec_of = LISTS[name]
    seed = 600 + 37 * K + 5 * sorted(LISTS).index(name)
    pos, vel, ine, cols, dt = _BUILD[fam](seed, n_worlds, N)
    rng = np.random.default_rng(seed + 2)
    tq = rng.normal(0, 1.0 if fam == "near" else 0.02, (n_worlds, N, 3 * K)) * np.tile(ine[..., :3], K)
    if name == "opposed":
        half = tq[..., :3 * (K // 2)]
        tq = np.concatenate([half, -half], -1)
    return (pos, vel, ine), spec_of({**cols, "tq": np.ascontiguousarray(tq)}), dt


def _norm(a):
    return np.sqrt(np.sum(a * a, -1))


def wheel_scales(spec, pos, vel, ine):
    """(A, B, C) of tests.util.body_scales, with the wheel fold scaled by its wheels one by one: B gets
    sum_k |tau_k .* I^-1| and C gets sum_k |tau_k| (util's |sum_k tau_k| vanishes for opposed wheels)."""
    A, B, C = (np.zeros(ine.shape[:2]) for _ in range(3))
    inv_i = 1.0 / ine[..., :3]
    for i, term in body_terms(spec):
        kind, kw = spec[i]
        if term == "wheels":
            tq = kw["torques"]
            wheels = [tq[..., 3 * k:3 * k + 3] for k in range(tq.shape[-1] // 3)]
            lin, ang, tau = 0.0, sum(_norm(t * inv_i) for t in wheels), sum(_norm(t) for t in wheels)
        else:
            lin, ang = body_term_accels(kind, kw, term, pos, vel, ine)
            tau = _norm(kw["wrench"][..., :3]) if term == "world_torque" else 0.0
        A, B, C = A + lin, B + ang, C + tau
    return A, B, C


def _oracle(O, start, spec, integ, dt, ticks=TICKS):
    w = O.World(*start)
    (w.rk4 if integ == "rk4" else w.semi_implicit)(dt, ticks, body_effectors(O, spec)[0],
                                                   threads=max(1, min(O.max_threads(), os.cpu_count() or 1)))
    return w.pos.copy(), w.vel.copy(), w.accel.copy(), w.force.copy()


def expected_kernel(K, name, integ, math):
    """The tick kernel of a list: FAST compiles three wheels first beside J2 or a world wrench (signatures 192 and
    384, one body per thread at this size); EXACT compiles wheels + world wrench (sequence 0x89) at any count."""
    if math == "fast":
        sig = {"j2": 192, "wworld": 384}.get(name) if K == 3 else None
        if sig is None:
            return f"body_fast_kernel<{_I[integ]}, 128, 4, false>"
        return f"body_fast_spec_kernel<{_I[integ]}, {sig}, false, 128, 4, 1>"
    seq = 0x89 if name in ("wworld", "opposed") else 0xFFFFFFFF
    return f"body_exact_kernel<0, 128, 4, false, {seq}>" if integ == "rk4" else f"body_exact_kernel<1, 256, 1, false, {seq}>"


# --------------------------------------------------------------------------- runs on the device (a fresh child)


def _table(ex, start, cols, dt):
    pos, vel, ine = start
    t = {el.component_id("tick"): np.array([0], dtype=np.uint64), FORCE: np.zeros(pos.shape[:2] + (6,)), INERTIA: ine,
         WORLD_POS: pos, WORLD_ACCEL: np.zeros(pos.shape[:2] + (6,)), el.component_id("simulation_time_step"): np.array([dt]),
         WORLD_VEL: vel}
    t.update({el.component_id(k): v for k, v in cols.items()})
    return [t[c] for c in ex.input_ids]


def _state(ex):
    return np.concatenate([ex.download(c) for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)], -1)


def _run_all(out, args):
    """Child: every case of one math mode through the three feeds.  The set_state run records the kernels it
    launched (an attempt counts only when the profiler saw every launch the library counted)."""
    math = args["math"]
    res = {}
    for K, name in CASES:
        start, spec, dt = _world(K, name)
        _, ge, cols = body_effectors(None, spec)
        for integ in INTEGRATORS:
            key = f"{K}-{name}-{integ}"
            for attempt in range(4):
                ex = el.B200Exec(N, M, dt, None, ge, integ, math)
                ex.set_state(*start, **cols)
                n0 = ex.timings()["kernel_launches"]
                _, names = launched_kernels(lambda: ex.step(TICKS, sync=True), settle=0.05 * 5 ** attempt)
                names = [n for n in names if not n.startswith(("Memcpy", "Memset"))]
                launches = ex.timings()["kernel_launches"] - n0
                if len(names) == launches or attempt == 3:
                    break
                ex.close()
            res[f"{key}_names"] = np.array(names, dtype=str)
            res[f"{key}_ok"] = len(names) == launches
            res[f"{key}_step"] = _state(ex)
            ex.close()
            for feed, chunk in (("small", 0), ("pipelined", CHUNK)):
                with el.B200Exec(N, M, dt, None, ge, integ, math, invoke_chunk_bodies=chunk) as ex:
                    outs = dict(zip(ex.output_ids, ex.invoke_batch(_table(ex, start, cols, dt), TICKS)))
                    res[f"{key}_{feed}"] = np.concatenate([outs[c] for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)], -1)
    np.savez(out, **res)


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """{math: results of _run_all}, each from a fresh child process."""
    d = tmp_path_factory.mktemp("wheel_counts")
    out = {}
    for math in ("exact", "fast"):
        with run_child("tests.test_wheel_counts:_run_all", str(d / f"{math}.npz"), {"math": math}) as z:
            out[math] = {k: z[k] for k in z.files}
    return out


def _split(a):
    return a[..., :7], a[..., 7:13], a[..., 13:19], a[..., 19:25]


@pytest.mark.gpu
@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("K,name", CASES)
@pytest.mark.parametrize("math", ["exact", "fast"])
def test_wheel_fold_matches_the_oracle(oracle, runs, math, K, name, integ):
    O = oracle
    res = runs[math]
    key = f"{K}-{name}-{integ}"
    start, spec, dt = _world(K, name)
    want = _oracle(O, start, spec, integ, dt)
    assert bool(res[f"{key}_ok"]), f"{math} {key}: the profiler lost launch records in every attempt"
    assert_route(list(res[f"{key}_names"]), [expected_kernel(K, name, integ, math)], f"{math} {key}")
    sc = wheel_scales(spec, *start)
    for feed in ("step", "small", "pipelined"):
        got = _split(res[f"{key}_{feed}"])
        what = f"{math} {key} {feed}"
        if math == "exact":
            for q, x, y in zip(("pos", "vel", "accel", "force"), got, want):
                assert np.array_equal(x, y), f"{what} {q}: max abs diff {np.max(np.abs(x - y))}"
        else:
            assert_body_close(got, want, start, dt, TICKS, sc, what=what)


# --------------------------------------------------------------------------- CPU: the bound is sensitive and not tight


def _with_torques(spec, tq):
    return [(k, {**kw, "torques": tq}) if k == "wheels" else (k, kw) for k, kw in spec]


def _rejects(got, want, start, dt, sc):
    try:
        assert_body_close(got, want, start, dt, TICKS, sc)
    except AssertionError:
        return True
    return False


@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("K,name", CASES)
def test_wheel_bound_is_sensitive(oracle, K, name, integ):
    """One wheel scaled by 1 + 1e-8 (the first, and the last) and the last wheel dropped must fail the bound; the
    wheels folded in reverse order must pass it."""
    O = oracle
    start, spec, dt = _world(K, name)
    sc = wheel_scales(spec, *start)
    want = _oracle(O, start, spec, integ, dt)
    assert not _rejects(want, want, start, dt, sc)
    tq = next(kw["torques"] for k, kw in spec if k == "wheels")
    for j in sorted({0, K - 1}):
        t = tq.copy()
        t[..., 3 * j:3 * j + 3] *= 1.0 + 1e-8
        got = _oracle(O, start, _with_torques(spec, t), integ, dt)
        assert _rejects(got, want, start, dt, sc), f"{K} {name} {integ}: wheel {j} scaled by 1 + 1e-8 passes"
    dropped = tq.copy()
    dropped[..., 3 * (K - 1):] = 0.0
    got = _oracle(O, start, _with_torques(spec, dropped), integ, dt)
    assert _rejects(got, want, start, dt, sc), f"{K} {name} {integ}: the last wheel dropped passes"
    rev = np.ascontiguousarray(tq.reshape(tq.shape[:-1] + (K, 3))[..., ::-1, :].reshape(tq.shape))
    got = _oracle(O, start, _with_torques(spec, rev), integ, dt)
    assert_body_close(got, want, start, dt, TICKS, sc, what=f"{K} {name} {integ}: wheels in reverse order")


def test_opposed_wheels_cancel():
    """The opposed lists' torque sums vanish to rounding, so only a per-wheel scale can bound them."""
    for K in (2, 4, 6, 8):
        start, spec, _ = _world(K, "opposed")
        tq = spec[0][1]["torques"]
        total = sum(tq[..., 3 * k:3 * k + 3] for k in range(K))
        per_wheel = sum(_norm(tq[..., 3 * k:3 * k + 3]) for k in range(K))
        assert np.all(_norm(total) <= 1e-14 * per_wheel) and np.all(per_wheel > 0)
