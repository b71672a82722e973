"""The FAST free-body tick keeps one byte per 64-body segment that says whether every mass of the segment is regular:
where the only force is a +0 gravity and Force is not formed, the mass enters only as (0 m + 0) rcp_nr(m), which is +0
for a regular m as for m = 1, so those warps leave the mass plane in HBM.  Skipping it must give the same bits as
reading it, for every class of mass, and every path that writes Inertia must make the handle forget what it knew."""

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200.executor import FORCE, INERTIA, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from tests.util import random_world

pytestmark = pytest.mark.gpu

M = 120001  # more than one wave of body pairs: the double2 kernel, whose last pair has one body
TICKS = 4
DT = 0.01
SEG = 64  # bodies per warp of pairs = per summary byte

# every class of mass, with what (0 m + 0) rcp_nr(m) makes of it on the device: +0 (regular: a warp may use m = 1),
# -0 (negative) or NaN; a subnormal m is flushed to 0 by rcp.approx.ftz, so the Newton steps end in NaN
MASSES = [(0.0, "nan"), (-0.0, "nan"), (-1.5, "-0"), (np.finfo(np.float64).tiny, "+0"), (5e-324 * 7, "nan"),
          (np.finfo(np.float64).max, "+0"), (np.inf, "nan"), (np.nan, "nan")]
SUBNORMAL = MASSES[4][0]


def _world(seed, M=M, N=1):
    """Segments cycle through four kinds: one body of every mass class (and -0 velocities) in lanes 0..15; every body
    of one class (cycling through the classes), half of them with -0 velocities; healthy with -0 velocities; healthy.
    Returns (pos, vel, ine, neg_zero): neg_zero marks the bodies whose six velocity components start at -0."""
    pos, vel, ine = random_world(seed, M, N)
    n = M * N
    i = np.arange(n)
    seg, lane = i // SEG, i % SEG
    m = ine.reshape(n, 7)[:, 6]
    mixed, whole = seg % 4 == 0, seg % 4 == 1
    for k, (v, _) in enumerate(MASSES):
        m[mixed & (lane == k)] = v
        m[whole & ((seg // 4) % len(MASSES) == k)] = v
    neg_zero = (mixed & (lane < 16)) | (whole & (lane % 2 == 0)) | ((seg % 4 == 2) & (lane % 5 == 0))
    neg_zero[-1] = True  # the pair of the odd tail
    vel.reshape(n, 6)[neg_zero] = -0.0
    return pos, vel, ine, neg_zero.reshape(M, N)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _download(ex):
    return [ex.download(c) for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)]


def _assert_same_bits(got, want, what):
    for name, a, b in zip(("pos", "vel", "accel", "force", "trajectory"), got, want):
        assert np.array_equal(_bits(a), _bits(b)), f"{what}: {name} differs"


@pytest.mark.parametrize("integrator", ["rk4", "semi_implicit"])
def test_one_tick_launches_match_a_fused_launch(oracle, integrator):
    """Launch 1 learns the summary, launches 2 and 3 use it, launch 4 writes Force; one launch of all four ticks reads
    every mass.  Both must agree bit for bit, the classes must be the ones the kernel's expression gives, and the
    healthy bodies must follow the oracle."""
    pos, vel, ine, neg_zero = _world(2026)
    runs = []
    for fused in (1, TICKS):
        with el.B200Exec(1, M, DT, None, [], integrator, "fast", max_fused_ticks=fused) as ex:
            ex.set_state(pos, vel, ine)
            ex.step(TICKS, sync=True)
            runs.append(_download(ex))
    got, fused = runs
    _assert_same_bits(got, fused, f"{integrator}: one tick per launch vs one launch")

    # the class of every mass, read off the device: a -0 linear velocity stays -0 under a -0 acceleration, turns +0
    # under a +0 one and NaN under a NaN one
    m = ine[..., 6]
    lin = fused[1][..., 3:]
    for v, cls in MASSES:
        at = neg_zero & ((m == v) if not np.isnan(v) else np.isnan(m))
        if v == 0.0:
            at &= np.signbit(m) == np.signbit(v)
        assert at.any(), v
        if cls == "nan":
            assert np.isnan(lin[at]).all(), f"{integrator}: m = {v!r}"
        else:
            assert np.array_equal(_bits(lin[at]), _bits(np.full(lin[at].shape, 0.0 if cls == "+0" else -0.0))), \
                f"{integrator}: m = {v!r} should give {cls}"

    w = oracle.World(pos, vel, ine)
    if integrator == "rk4":
        w.rk4(DT, TICKS, [], threads=4)
    else:
        w.semi_implicit(DT, TICKS, [], threads=4)
    healthy = np.isfinite(m) & (m >= np.finfo(np.float64).tiny)
    for what, a, b in zip(("pos", "vel", "accel", "force"), got, (w.pos, w.vel, w.accel, w.force)):
        a, b = a[healthy], b[healthy]
        err = float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))
        assert err <= TICKS * 1e-12, f"{integrator} {what}: rel err {err:.3e}"
    # FAST arithmetic differs from the oracle on two classes, with or without the summary: it flushes a subnormal mass,
    # and it forms the gravity term g m even for g = 0, so an infinite mass gives 0 inf = NaN where the oracle's
    # 0 / inf is 0
    odd = ~healthy & (m != SUBNORMAL) & ~np.isinf(m)
    for what, a, b in zip(("pos", "vel"), got, (w.pos, w.vel)):
        assert np.array_equal(np.isfinite(a[odd]), np.isfinite(b[odd])), f"{integrator} {what}"


def _flip_masses(ine, N):
    """Masses for a second phase: the degenerate segments turn healthy, and the healthy segments that start with -0
    velocities gain a NaN and a negative mass (lanes 5 and 10, both -0 lanes)."""
    rng = np.random.default_rng(99)
    out = ine.copy()
    n = out.shape[0] * N
    m = out.reshape(n, 7)[:, 6]
    i = np.arange(n)
    seg, lane = i // SEG, i % SEG
    bad = seg % 4 <= 1
    m[bad] = rng.uniform(0.5, 50, int(bad.sum()))
    m[(seg % 4 == 2) & (lane == 5)] = np.nan
    m[(seg % 4 == 2) & (lane == 10)] = -2.0
    return out


def _table(ex, state, ine):
    """invoke_batch inputs; a None entry is a column that is not dirty (the device copy stands)."""
    pos, vel = state if state is not None else (None, None)
    t = {el.component_id("tick"): None, FORCE: None, INERTIA: ine, WORLD_POS: pos, WORLD_ACCEL: None,
         el.component_id("simulation_time_step"): None, WORLD_VEL: vel}
    return [t[c] for c in ex.input_ids]


def _outputs(ex, outs):
    o = dict(zip(ex.output_ids, outs))
    return [o[c] for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)]


# (path, worlds, entities, bodies per invoke range): the pipelined case runs ranges of 104 928 bodies (the double2
# kernel) over N = 3 entities, so ranges 1 and 3 start half way into a segment and ranges 0 and 2 on a segment
# boundary; the last range is too small for body pairs.  The packed case (<= 1024 bodies) runs one body per thread.
PATHS = [("upload", M, 1, 0), ("packed", 1000, 1, 0), ("pipelined", 140905, 3, 104928)]


@pytest.mark.parametrize("path,Mw,N,chunk", PATHS, ids=[p[0] for p in PATHS])
def test_inertia_writes_invalidate_the_summary(path, Mw, N, chunk):
    """Populate the summary, overwrite Inertia through one write path so that regular segments turn degenerate and
    degenerate ones regular, and step with one tick per launch: the states after every tick must be bit-identical to
    a fresh handle's that reads every mass.  A following batch with a NULL Inertia input keeps using the summary."""
    pos, vel, ine, neg_zero = _world(7, Mw, N)
    ine2 = _flip_masses(ine, N)
    kw = dict(trajectory_every=1, trajectory_capacity=9, invoke_chunk_bodies=chunk)
    with el.B200Exec(N, Mw, DT, None, [], "rk4", "fast", max_fused_ticks=1, **kw) as ex, \
         el.B200Exec(N, Mw, DT, None, [], "rk4", "fast", max_fused_ticks=8, **kw) as ref:
        ex.set_state(pos, vel, ine)
        ex.step(3, sync=True)  # launch 1 populates the summary, launch 2 uses it
        mid = (ex.download(WORLD_POS), ex.download(WORLD_VEL))
        mid[1][neg_zero] = -0.0
        if path == "upload":
            results = []
            for h in (ex, ref):
                h.set_state(mid[0], mid[1], ine2)
                h.step(3, sync=True)
                results.append(_download(h))
            got, want = results
        else:
            got = _outputs(ex, ex.invoke_batch(_table(ex, mid, ine2), 3))
            want = _outputs(ref, ref.invoke_batch(_table(ref, mid, ine2), 3))
        _assert_same_bits(got + [ex.trajectory()[3:6]], want + [ref.trajectory()[0:3]], f"{path}: after the Inertia write")
        if path == "upload":
            return
        got = _outputs(ex, ex.invoke_batch(_table(ex, None, None), 3))
        want = _outputs(ref, ref.invoke_batch(_table(ref, None, None), 3))
        _assert_same_bits(got + [ex.trajectory()[6:9]], want + [ref.trajectory()[3:6]], f"{path}: NULL Inertia input")


def test_raw_inertia_pointer_retires_the_summary():
    """Masses written through b200_sixdof_device_plane bypass the handle: the next tick must read them."""
    import torch

    pos, vel, ine = random_world(5, M, 1)
    with el.B200Exec(1, M, DT, None, [], "rk4", "fast", max_fused_ticks=1, trajectory_every=1, trajectory_capacity=8) as ex:
        ex.set_state(pos, vel, ine)
        ex.step(3, sync=True)  # every full segment is regular and known to be
        ptr = ex.device_plane(INERTIA, 6)

        class Plane:
            __cuda_array_interface__ = {"shape": (M,), "typestr": "<f8", "data": (ptr, False), "version": 3}

        j = 10 * SEG + 17
        torch.as_tensor(Plane(), device="cuda")[j] = 0.0
        torch.cuda.synchronize()
        ex.step(2, sync=True)  # launch 1 forms no Force: only the mass plane tells it about the zero mass
        after_one = ex.trajectory()[3]
    assert np.isnan(after_one[j, 0, 10:13]).all()
    others = np.arange(M) != j
    assert np.isfinite(after_one[others]).all()
