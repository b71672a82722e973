"""Ensemble statistics over the world axis (b200_sixdof_trajectory_stats / _state_stats / b200_stats_merge, Exec's
ensemble mode) against an exact reference: the mean is math.fsum(x) / n, m2 the fsum of the squared deviations from
it, over the finite values only.

Bounds (every comparison below): count and min / max equal; mean within 1e-13 max|x|; std = sqrt(m2 / n) within
1e-8 std + 32 eps max|x| — the absolute term is the spread a mean rounded to a few ulps of max|x| can resolve (it
matters only for groups whose worlds agree to the last bits).  test_bounds_are_sensitive shows the one-pass
E[x^2] - E[x]^2 formula violates the std bound on data with |mean| / std = 1e6, where the library must keep it."""

import math

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from tests.ensemble_util import FREE, ROCKET, handle, need_gpu, rocket_world, run_gloo, sampled_state, split

EPS = np.finfo(np.float64).eps
NAN = float("nan")


# --------------------------------------------------------------------------- reference and bounds


def ref_group(x):
    """(count, mean, m2, min, max) of the finite values of a 1-D array, exact up to the final roundings."""
    f = np.asarray(x, dtype=np.float64)
    f = f[np.isfinite(f)]
    n = f.size
    if n == 0:
        return (0.0, NAN, NAN, NAN, NAN)
    mean = math.fsum(f.tolist()) / n
    m2 = math.fsum(((f - mean) ** 2).tolist())
    return (float(n), mean, m2, float(np.min(f)), float(np.max(f)))


def ref_table(x):
    """x [worlds, ...] -> [..., 5]: ref_group over the world axis of every trailing index."""
    x = np.asarray(x, dtype=np.float64)
    flat = x.reshape(x.shape[0], -1)
    out = np.array([ref_group(flat[:, g]) for g in range(flat.shape[1])]).reshape(x.shape[1:] + (5,))
    return out


def std_of(t):
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.sqrt(t[..., 2] / t[..., 0])


def check_table(got, want, scale, what=""):
    """got / want [..., 5]; scale = max|x| over the finite values of each group ([...])."""
    assert got.shape == want.shape, what
    assert np.array_equal(got[..., 0], want[..., 0]), f"{what}: counts differ"
    empty = want[..., 0] == 0
    assert np.all(np.isnan(got[empty][..., 1:])), f"{what}: a group without finite values is not NaN"
    g, w, s = got[~empty], want[~empty], scale[~empty]
    assert np.array_equal(g[:, 3], w[:, 3]) and np.array_equal(g[:, 4], w[:, 4]), f"{what}: min / max differ"
    mean_err = np.abs(g[:, 1] - w[:, 1])
    assert np.all(mean_err <= 1e-13 * s), f"{what}: mean off by {np.max(mean_err / np.maximum(s, 1e-300)):.3e} max|x|"
    sg, sw = std_of(g), std_of(w)
    bound = 1e-8 * sw + 32 * EPS * s
    err = np.abs(sg - sw)
    assert np.all(err <= bound), f"{what}: std off by {np.max(err / np.maximum(bound, 1e-300)):.3g} x the bound"


def finite_scale(x):
    """max|x| over the finite values along the world axis (0 where none)."""
    a = np.abs(np.asarray(x, dtype=np.float64))
    return np.max(np.where(np.isfinite(a), a, 0.0), axis=0)


# --------------------------------------------------------------------------- CPU: b200_stats_merge


@pytest.mark.parametrize("seed", range(6))
def test_merge_matches_exact_sums(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(10_000, 1_000_001)) if seed < 5 else 1_000_000
    k = int(rng.integers(1, 17))
    groups = np.stack([rng.normal(3.0, 2.0, n), rng.uniform(-1e3, 5e3, n), 7.0e5 + rng.exponential(1.0, n)], axis=1)
    parts = split(rng, n, k)
    if k > 2:
        parts.insert(1, parts[0][:0])  # an empty part in the middle
    tables = [ref_table(groups[idx]) if len(idx) else np.tile([0.0, NAN, NAN, NAN, NAN], (3, 1)) for idx in parts]
    got = el.merge_stats(tables)
    check_table(got, ref_table(groups), finite_scale(groups), f"{k} parts")
    # min / max are np.min / np.max themselves, bit for bit
    assert np.array_equal(got[:, 3], np.min(groups, 0)) and np.array_equal(got[:, 4], np.max(groups, 0))
    assert got.tobytes() == el.merge_stats(tables).tobytes()  # identical calls, identical bits


def test_bounds_are_sensitive():
    """|mean| / std = 1e6 (orbital positions with metre-level dispersion): the merge keeps the bounds, the one-pass
    formula E[x^2] - E[x]^2 misses the std bound by orders of magnitude on the same data."""
    rng = np.random.default_rng(7)
    n = 200_000
    x = 6.4e6 + rng.normal(0.0, 6.4, n)
    assert 0.9e6 <= abs(np.mean(x)) / np.std(x) <= 1.1e6
    parts = split(rng, n, 9)
    tables = [ref_table(x[idx][:, None]) for idx in parts]
    want = ref_table(x[:, None])
    got = el.merge_stats(tables)
    check_table(got, want, finite_scale(x[:, None]), "merge")
    naive = np.sqrt(max(np.mean(x * x) - np.mean(x) ** 2, 0.0))
    sw = float(std_of(want)[0])
    assert abs(naive - sw) > 1e-8 * sw + 32 * EPS * np.max(np.abs(x)), "the data is not hard enough to tell the formulas apart"


def test_non_finite_worlds_are_excluded_and_counted():
    rng = np.random.default_rng(3)
    x = rng.normal(0.0, 1.0, (1000, 4))
    x[[3, 17, 500], 0] = [np.nan, np.inf, -np.inf]
    x[:, 2] = np.nan  # nothing finite in this group
    x[::2, 3] = np.inf
    parts = split(rng, 1000, 5)
    tables = [ref_table(x[idx]) if len(idx) else np.tile([0.0, NAN, NAN, NAN, NAN], (4, 1)) for idx in parts]
    got = el.merge_stats(tables)
    want = ref_table(x)
    assert list(got[:, 0]) == [997.0, 1000.0, 0.0, 500.0]
    assert np.all(np.isnan(got[2, 1:]))
    check_table(got, want, finite_scale(x), "non-finite")


def test_merge_rejects_bad_tables():
    with pytest.raises(_lib.B200ValueError):
        el.merge_stats([np.zeros((3, 5)), np.zeros((4, 5))])
    with pytest.raises(_lib.B200ValueError):
        el.merge_stats([np.zeros((3, 4))])
    with pytest.raises(_lib.B200Error):
        el.merge_stats([np.full((2, 5), -1.0)])  # a negative count


def _rank_table(rank):
    rng = np.random.default_rng(100 + rank)
    x = 1.0e4 * (rank + 1) + rng.normal(0.0, 3.0, (500 + 37 * rank, 6, 4))
    return ref_table(x)


def _gather_worker(rank, ws):
    from elodin_b200.sharding import gather_ensemble

    return gather_ensemble(_rank_table(rank))


def test_gather_ensemble_two_gloo_ranks():
    ws = 2
    got = run_gloo(_gather_worker, ws)
    want = el.merge_stats([_rank_table(r) for r in range(ws)])  # rank order
    assert got[0].shape == (6, 4, 5)
    assert got[0].tobytes() == want.tobytes() and got[1].tobytes() == want.tobytes()


# --------------------------------------------------------------------------- GPU


SHAPES = [(1, 1), (7, 3), ((1 << 16) + 3, 1), (5, 1024), (100, 300)]


def _ring_ref(traj):
    """traj [S, M, N, W] -> reference [S, N, W, 5] and scales [S, N, W]."""
    x = np.moveaxis(traj, 1, 0)  # [M, S, N, W]
    return ref_table(x), finite_scale(x)


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("kind", [FREE, ROCKET])
@pytest.mark.parametrize("width", [13, 25])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_trajectory_stats_match_the_ring(shape, width, kind, math_mode):
    need_gpu()
    M, N = shape
    with handle(kind, M, N, math_mode, width=width, capacity=3)[0] as ex:
        ex.step(3)
        traj = ex.trajectory()
        got = ex.trajectory_stats()
        launches = ex.timings()["kernel_launches"]
        again = ex.trajectory_stats()
        assert ex.timings()["kernel_launches"] > launches  # the reduction runs in this library's kernels
    assert got.shape == (3, N, width, 5)
    want, scale = _ring_ref(traj)
    check_table(got, want, scale, f"{shape} {kind} {math_mode} W={width}")
    assert got.tobytes() == again.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_state_stats_match_the_columns(shape, math_mode):
    need_gpu()
    M, N = shape
    with handle(ROCKET, M, N, math_mode, capacity=1)[0] as ex:
        ex.step(2)
        got = ex.state_stats()
        cols = sampled_state(ex)
    assert got.shape == (N, 25, 5)
    check_table(got, ref_table(cols), finite_scale(cols), f"{shape} {math_mode}")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [((1 << 16) + 3, 1), (7, 3), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_state_stats_keep_the_bounds_at_orbital_offsets(shape):
    """The kernel on |mean| / std = 1e6 data (orbital positions, metre-level dispersion), where E[x^2] - E[x]^2
    breaks the std bound."""
    need_gpu()
    M, N = shape
    rng = np.random.default_rng(11)
    from tests.util import near_world

    pos, vel, ine, cols, dt = near_world(5, M, N)
    pos[..., 4:] = np.array([6.4e6, -3.1e6, 2.2e6]) + rng.normal(0.0, 6.4, (M, N, 3))
    vel[..., 3:] = 7.6e3 + rng.normal(0.0, 7.6e-3, (M, N, 3))
    with handle(FREE, M, N, "fast", state=(pos, vel, ine, cols, dt))[0] as ex:
        got = ex.state_stats()
        state = sampled_state(ex)
    check_table(got, ref_table(state), finite_scale(state), f"orbital {shape}")
    if M > 1000:
        x = state[:, 0, 4]
        naive = np.sqrt(max(np.mean(x * x) - np.mean(x) ** 2, 0.0))
        sw = float(std_of(ref_table(x[:, None]))[0])
        assert abs(naive - sw) > 1e-8 * sw + 32 * EPS * np.max(np.abs(x))


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("shape", [(7, 3), ((1 << 16) + 3, 1), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_non_finite_worlds_are_dropped_from_the_count(shape, math_mode):
    need_gpu()
    M, N = shape
    from tests.util import near_world

    pos, vel, ine, cols, dt = near_world(2, M, N)
    bad = [1, M // 2, M - 2]
    pos[bad[0], 0, 4] = np.nan
    vel[bad[1], N - 1, 3] = np.inf
    pos[bad[2], 0, 5] = -np.inf
    with handle(ROCKET, M, N, math_mode, capacity=2, state=(pos, vel, ine, cols, dt))[0] as ex:
        s0 = ex.state_stats()
        state0 = sampled_state(ex)
        ex.step(2)
        traj = ex.trajectory()
        got = ex.trajectory_stats()
    assert s0[0, 4, 0] == M - 1 and s0[N - 1, 7 + 3, 0] == M - 1 and s0[0, 5, 0] == M - 1
    check_table(s0, ref_table(state0), finite_scale(state0), "uploaded state")
    want, scale = _ring_ref(traj)
    check_table(got, want, scale, "after two ticks")
    assert np.all(got[..., 0] <= M) and np.min(got[..., 0]) < M  # the broken worlds stay out of the count


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(7, 3), ((1 << 16) + 3, 1), (5, 1024), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_a_sample_has_the_same_bits_in_any_ring(shape):
    need_gpu()
    M, N = shape
    S = 64 if M * N < 100_000 else 8
    big, state = handle(ROCKET, M, N, "fast", capacity=S)
    one, _ = handle(ROCKET, M, N, "fast", capacity=1, state=state)
    with big, one:
        big.step(S)
        many = big.trajectory_stats()
        assert many.tobytes() == big.trajectory_stats().tobytes()
        for s in range(S):
            one.trajectory_reset()
            one.step(1)
            single = one.trajectory_stats()
            assert single.shape[0] == 1
            assert single[0].tobytes() == many[s].tobytes(), f"sample {s}"


@pytest.mark.gpu
def test_two_handles_merged_match_one():
    need_gpu()
    from tests.util import near_world

    M, N = 20_001, 2
    pos, vel, ine, cols, dt = near_world(9, M, N)
    half = M // 2
    part = lambda a, lo, hi: np.ascontiguousarray(a[lo:hi])
    sub = lambda lo, hi: (part(pos, lo, hi), part(vel, lo, hi), part(ine, lo, hi),
                          {k: part(v, lo, hi) for k, v in cols.items()}, dt)
    whole, _ = handle(ROCKET, M, N, "fast", capacity=3, state=(pos, vel, ine, cols, dt))
    a, _ = handle(ROCKET, half, N, "fast", capacity=3, state=sub(0, half))
    b, _ = handle(ROCKET, M - half, N, "fast", capacity=3, state=sub(half, M))
    with whole, a, b:
        for ex in (whole, a, b):
            ex.step(3)
        want = whole.trajectory_stats()
        traj = whole.trajectory()
        got = el.merge_stats([a.trajectory_stats(), b.trajectory_stats()])
    check_table(got, want, _ring_ref(traj)[1], "two handles")


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
def test_exec_ensemble_mode_against_the_default_mode(math_mode):
    need_gpu()
    M, ticks = 300, 23
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=24.0, math=math_mode, n_worlds=M, world_params=params)
    ref = w.build(sys_, **kw)
    ref.run(ticks)
    runs = {}
    for name, ring, host in (("ring1", 1, False), ("ring16", 16, False), ("host", 3, True), ("default_ring", None, False)):
        s = (sys_ | el.host_system(lambda ctx: None)) if host else sys_
        ex = w.build(s, ensemble=True, ensemble_ring=ring, **kw)
        ex.run(ticks)
        runs[name] = ex
    ens = runs["ring1"]
    for pair in ("rocket.world_pos", "rocket.world_vel", "rocket.world_accel", "rocket.force", "ball.world_pos", "ball.force"):
        hist = ref.history_worlds(pair)  # [rows, M, width]
        got = ens.ensemble(pair)
        assert got["mean"].shape == hist.shape[:1] + hist.shape[2:] == (6, hist.shape[2])
        table = np.stack([got["count"], got["mean"], got["std"] ** 2 * got["count"], got["min"], got["max"]], -1)
        worlds = np.moveaxis(hist, 1, 0)  # [M, rows, width]
        check_table(table, ref_table(worlds), finite_scale(worlds), pair)
        for name, ex in runs.items():
            other = ex.ensemble(pair)
            for k in got:
                assert other[k].tobytes() == got[k].tobytes(), f"{pair} {k}: {name} differs from ring1"
    for name, ex in runs.items():
        for cname in ("world_pos", "world_vel", "world_accel", "force"):
            cid = el.component_id(cname)
            assert np.array_equal(ex.world.columns[cid].buffer, ref.world.columns[cid].buffer), f"{name}: final {cname}"
        assert ex.tick == ref.tick == ticks
    with pytest.raises(_lib.B200Error, match="ensemble"):
        ens.history("rocket.world_pos")
    with pytest.raises(_lib.B200Error, match="ensemble"):
        ens.history_worlds("rocket.world_pos")
    with pytest.raises(_lib.B200Error, match="ensemble"):
        ens.attach_db("/nonexistent/db")
    with pytest.raises(_lib.B200ValueError, match="rocket.inertia") as e:
        ens.ensemble("rocket.inertia")
    assert e.value.code == _lib.ERR_COMPONENT_NOT_FOUND
    with pytest.raises(_lib.B200ValueError, match="rocket.thrust"):
        ens.ensemble("rocket.thrust")
