"""World-sharded quantiles (b200_sixdof_sharded_quantiles_begin / _round / _end, sharding.gather_quantiles): R handles
hold consecutive slices of one campaign and reduce their quantile tables together, in rounds whose u32 words are summed
over the ranks.  The table must have the bits of the unsharded entry on one handle holding every world, for any rank
count and split, the sign of zero included."""

import os

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib, sharding
from tests.ensemble_util import ROCKET, handle, need_gpu, no_device, run_gloo  # noqa: F401
from tests.test_ensemble_quantiles import ref_quantiles, same_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = (0.0, 1e-3, 1 / 3, 0.5, 0.9, 0.999, 1.0)
LEVELS16 = tuple(np.linspace(0.0, 1.0, 16))
DBL_MAX = np.finfo(np.float64).max
HIST_WORDS = (1 << 14) + 2 * 32  # u32 words of one triple in a histogram round: 2^14 counters, 32 u64 keys


# --------------------------------------------------------------------------- helpers


def state_handle(x):
    """A handle whose state planes are x [M, E, 25] (the B200_TRAJ_FULL layout)."""
    M, E, _ = x.shape
    ine = np.broadcast_to(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 7))
    ex = el.B200Exec(E, M, 0.01, None, [], "rk4", "exact")
    ex.set_state(x[..., :7], x[..., 7:13], ine, accel=x[..., 13:19], force=x[..., 19:25])
    return ex


def cut(M, bounds):
    """[(a, b)] of the consecutive rank ranges ending at the sorted `bounds` (the last one ends at M)."""
    edges = [0] + list(bounds) + [M]
    return list(zip(edges[:-1], edges[1:]))


def cut_groups(sizes, a, b):
    """The global group sizes cut to the worlds [a, b)."""
    out, g0 = [], 0
    for s in sizes:
        out.append(max(0, min(g0 + s, b) - max(g0, a)))
        g0 += s
    return out


def drive(exs, q, source="state", groups=False):
    """The rounds of every handle in lockstep, the partials summed (u32, wrapping) with numpy.  Returns (the tables,
    the round sizes, begin's bound)."""
    bound = [ex.sharded_quantiles_begin(q, source, groups) for ex in exs]
    assert len(set(bound)) == 1, bound
    bufs = [np.zeros(max(bound[0] // 4, 1), np.uint32) for _ in exs]
    sizes, n, red = [], 0, None
    while True:
        got = [ex.sharded_quantiles_round(red, n, b) for ex, b in zip(exs, bufs)]
        assert len(set(got)) == 1, got  # every rank makes the same rounds
        n = got[0]
        assert n <= bound[0] and n % 4 == 0
        sizes.append(n)
        if n == 0:
            break
        red = bufs[0][: n // 4].copy()
        for b in bufs[1:]:
            red += b[: n // 4]
    return [ex.sharded_quantiles_end() for ex in exs], sizes, bound[0]


def rounds_per_slice(sizes):
    """The round sizes split at each count round (a count round is one u32 per triple: below one histogram triple)."""
    out = []
    for n in sizes[:-1]:
        if n < HIST_WORDS * 4:
            out.append(0)
        else:
            assert n % (HIST_WORDS * 4) == 0
        out[-1] += 1
    return out


def check_rounds(sizes):
    per = rounds_per_slice(sizes)
    assert all(1 <= r <= 8 for r in per), per
    return per


def degenerate(M, E, seed=3):
    """[M, E, 25] planes: all-equal, heavy ties, signed zeros, subnormals, +-DBL_MAX, NaN / +-inf, every binade."""
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (M, E, 25))
    x[..., 0] = 1.25
    x[..., 1] = rng.choice([1.0, 2.0, 3.0], (M, E))
    x[..., 2] = rng.choice([0.0, -0.0, 5e-324, -5e-324, 2.2e-308], (M, E))
    x[..., 3] = rng.choice([DBL_MAX, -DBL_MAX], (M, E))
    x[..., 4][rng.random((M, E)) < 0.1] = np.nan
    x[..., 4][rng.random((M, E)) < 0.05] = np.inf
    x[..., 4][rng.random((M, E)) < 0.05] = -np.inf
    x[..., 5] = np.nan
    x[..., 6] = rng.choice([0.0, -0.0], (M, E))
    x[..., 7] = np.ldexp(rng.random((M, E)), rng.integers(-1074, 1023, (M, E))) * rng.choice([-1, 1], (M, E))
    x[..., 8] = 6.9e6 + rng.normal(0.0, 1.0, (M, E))
    x[..., 9] = np.where(rng.random((M, E)) < 1e-3, -3.0, 2.0)
    return x


def sharded_state(x, bounds, q, groups=None):
    """The sharded state quantiles of x over the ranks of `bounds` (grouped when `groups` is the global sizes)."""
    exs = [state_handle(np.ascontiguousarray(x[a:b])) for a, b in cut(x.shape[0], bounds)]
    if groups is not None:
        for ex, (a, b) in zip(exs, cut(x.shape[0], bounds)):
            ex.set_world_groups(cut_groups(groups, a, b))
    return drive(exs, q, "state", groups is not None)


def one_state(x, q, groups=None):
    ex = state_handle(x)
    if groups is None:
        return ex.state_quantiles(q)
    ex.set_world_groups(groups)
    return ex.state_group_quantiles(q)


# --------------------------------------------------------------------------- CPU


def test_sharded_symbols_are_bound_and_declared():
    header = open(os.path.join(ROOT, "include", "b200_sixdof.h")).read()
    for name in ("b200_sixdof_sharded_quantiles_begin", "b200_sixdof_sharded_quantiles_round",
                 "b200_sixdof_sharded_quantiles_end"):
        assert name in _lib.SYMBOLS and name + "(" in header
    for src, k in _lib.QUANTILE_SOURCES.items():
        assert f"B200_QUANTILE_{'RING' if src == 'ring' else src.upper()} = {k}" in header


def test_gather_quantiles_refuses_a_bad_source_before_any_call():
    class Boom:
        def __getattr__(self, name):
            raise AssertionError("the executor must not be reached")

    with pytest.raises(ValueError, match="quantile source"):
        sharding.gather_quantiles(Boom(), LEVELS, source="samples")


def test_build_refuses_a_process_group_without_the_options_it_serves(no_device):
    from tests.ensemble_util import two_body_world

    w = two_body_world()
    with pytest.raises(_lib.B200Error, match="process_group: need World.build"):  # the mode first
        w.build(el.six_dof(), n_worlds=4, process_group=object())
    with pytest.raises(_lib.B200Error, match="process_group makes the quantile tables collective"):
        w.build(el.six_dof(), n_worlds=4, ensemble=True, process_group=object())
    with pytest.raises(ValueError, match="quantile level"):  # the option's own values before the group is used
        w.build(el.six_dof(), n_worlds=4, ensemble=True, quantiles=[2.0], process_group=object())


class _ArgumentsOnly:
    """An executor stand-in for the argument exchange of gather_quantiles: its begin succeeds with no round to make."""

    n_worlds = 10

    def sharded_quantiles_shape(self, q, source="ring", groups=False):
        return (1, 25, np.atleast_1d(q).size)

    def sharded_quantiles_begin(self, q, source="ring", groups=False):
        return 0


def _bad_argument_worker(rank, ws, kind):
    """Rank 1 passes an argument it cannot use; every rank must raise, none may wait on the others."""
    args = {"source": ("state", "samples"), "levels": (LEVELS, ("a", "b"))}[kind]
    try:
        if kind == "source":
            sharding.gather_quantiles(_ArgumentsOnly(), LEVELS, args[rank])
        else:
            sharding.gather_quantiles(_ArgumentsOnly(), args[rank], "state")
    except Exception as e:  # noqa: BLE001 - the error is the result
        return type(e).__name__
    return None


@pytest.mark.parametrize("kind", ["source", "levels"])
def test_an_argument_one_rank_cannot_use_raises_on_every_rank(kind):
    assert run_gloo(_bad_argument_worker, 2, kind) == ["ValueError", "ValueError"]


# --------------------------------------------------------------------------- GPU: simulated ranks


@pytest.mark.gpu
@pytest.mark.parametrize("R", [1, 2, 3, 5])
def test_state_quantiles_over_ranks_equal_one_handle(R):
    need_gpu()
    M, E = 20011, 2
    x = degenerate(M, E)
    rng = np.random.default_rng(R)
    bounds = sorted(rng.choice(np.arange(1, M), R - 1, replace=False).tolist())  # ragged
    tabs, sizes, _ = sharded_state(x, bounds, LEVELS)
    want = one_state(x, LEVELS)
    assert same_bits(want, ref_quantiles(x, LEVELS))
    for t in tabs:
        assert same_bits(t, want)
    check_rounds(sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("q", [(0.0,), (1.0,), (0.5, 0.5, 0.25, 0.25), LEVELS16], ids=["0", "1", "dup", "16"])
def test_levels(q):
    need_gpu()
    x = degenerate(9001, 1, seed=5)
    tabs, sizes, _ = sharded_state(x, [3000, 3001], q)
    for t in tabs:
        assert same_bits(t, one_state(x, q))
    check_rounds(sizes)


GROUPS = {
    # global groups of <= 256, <= 8192 and > 8192 worlds, cut by the ranks onto other routes, one empty everywhere
    "routes": ([200, 0, 5000, 9500, 300], [150, 5300, 5301, 12000]),
    "empty on a rank": ([10, 8300, 9000], [5, 6, 8310]),
    "one rank": ([100, 9000], []),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(GROUPS))
def test_grouped_state_quantiles_over_ranks(case):
    need_gpu()
    sizes, bounds = GROUPS[case]
    M = sum(sizes)
    x = degenerate(M, 1, seed=7)
    tabs, sizes_r, _ = sharded_state(x, bounds, LEVELS, groups=sizes)
    want = one_state(x, LEVELS, groups=sizes)
    o = np.cumsum([0] + sizes)
    for g in range(len(sizes)):
        assert same_bits(want[g], ref_quantiles(x[o[g]:o[g + 1]], LEVELS)), g
    for t in tabs:
        assert same_bits(t, want)
    check_rounds(sizes_r)


@pytest.mark.gpu
def test_split_invariance():
    """Permuting the worlds over the ranks, or moving the rank boundaries, changes no bit and no round size."""
    need_gpu()
    M = 12345
    x = degenerate(M, 1, seed=11)
    want = one_state(x, LEVELS16)
    perm = np.random.default_rng(0).permutation(M)
    seen = []
    for xx, bounds in ((x, []), (x, [4000, 8000]), (x, [1, 12000]), (x[perm], [6000, 6100]),
                       (x[::-1], [100, 200, 300])):
        tabs, sizes, bound = sharded_state(np.ascontiguousarray(xx), bounds, LEVELS16)
        for t in tabs:
            assert same_bits(t, want)
        check_rounds(sizes)
        assert max(sizes) <= bound
        seen.append((sizes, bound))
    assert all(s == seen[0] for s in seen), seen  # the same round sizes and bound for every split


@pytest.mark.gpu
def test_more_than_one_slice():
    """E = 60: a slice holds 22 of the 25 (group, plane) rows, so the call runs two slices in its rounds."""
    need_gpu()
    x = degenerate(3001, 60, seed=13)
    tabs, sizes, bound = sharded_state(x, [1500], LEVELS)
    want = one_state(x, LEVELS)
    for t in tabs:
        assert same_bits(t, want)
    per = check_rounds(sizes)
    assert len(per) == 2
    assert bound == 22 * 60 * HIST_WORDS * 4


@pytest.mark.gpu
def test_adversarial_neighbours_finish_within_the_round_bound():
    """Keys a last bit apart around every one of 16 levels, interleaved over the ranks: every rank refines to ranges
    of one key, within 8 rounds, exactly."""
    need_gpu()
    M = 16 * 1024 + 17
    x = np.empty(M)
    x[0] = 1.0
    for k in range(1, M):
        x[k] = np.nextafter(x[k - 1], 2.0)
    x = x[np.random.default_rng(2).permutation(M)]
    planes = np.broadcast_to(x[:, None, None], (M, 1, 25)).copy()
    planes[:, 0, 1] = -x
    planes[:, 0, 2] = np.where(np.arange(M) % 2, 0.0, -0.0)
    for bounds in ([M // 2], [1000, 2000, 9000]):
        tabs, sizes, _ = sharded_state(planes, bounds, LEVELS16)
        want = one_state(planes, LEVELS16)
        assert same_bits(want, ref_quantiles(planes, LEVELS16))
        for t in tabs:
            assert same_bits(t, want)
        check_rounds(sizes)


def _rocket_ranks(M, bounds, capacity=4, ticks=3, seed=1):
    from tests.util import near_world

    pos, vel, ine, cols, dt = near_world(seed, M, 2)
    one = handle(ROCKET, M, 2, "exact", capacity=capacity, state=(pos, vel, ine, cols, dt))[0]
    exs = [handle(ROCKET, b - a, 2, "exact", capacity=capacity,
                  state=(pos[a:b], vel[a:b], ine[a:b], {k: v[a:b] for k, v in cols.items()}, dt))[0]
           for a, b in cut(M, bounds)]
    for ex in [one] + exs:
        ex.step(ticks)
    return one, exs


@pytest.mark.gpu
@pytest.mark.parametrize("grouped", [False, True])
def test_ring_and_outcome_quantiles_over_ranks(grouped):
    need_gpu()
    M, bounds, sizes = 20000, [7000, 7001, 15000], [3000, 9000, 0, 8000]
    one, exs = _rocket_ranks(M, bounds)
    vals = np.random.default_rng(3).normal(0.0, 1.0, (M, 2))
    vals[::7, 0] = np.nan
    vals[:, 1] = np.round(vals[:, 1])
    spans = cut(M, bounds)
    one.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, vals[:, k]) for k in range(2)])
    for ex, (a, b) in zip(exs, spans):
        ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, vals[a:b, k]) for k in range(2)])
    if grouped:
        one.set_world_groups(sizes)
        for ex, (a, b) in zip(exs, spans):
            ex.set_world_groups(cut_groups(sizes, a, b))
    ring = one.trajectory_group_quantiles(LEVELS) if grouped else one.trajectory_quantiles(LEVELS)
    outc = one.outcome_group_quantiles(LEVELS) if grouped else one.outcome_quantiles(LEVELS)
    tabs, sizes_r, _ = drive(exs, LEVELS, "ring", grouped)
    for t in tabs:
        assert same_bits(t, ring)
    check_rounds(sizes_r)
    tabs, sizes_r, _ = drive(exs, LEVELS, "outcomes", grouped)
    for t in tabs:
        assert same_bits(t, outc)
    check_rounds(sizes_r)
    if not grouped:
        assert same_bits(outc, ref_quantiles(vals, LEVELS))
        assert exs[0].quantile_reads() >= 1.0


@pytest.mark.gpu
def test_a_summary_fold_between_rounds_ends_an_outcome_call():
    """The outcome planes are computed from the run summaries: a fold between rounds changes them, so the next round
    of an outcome call is refused; a ring or state call is not affected by it."""
    need_gpu()
    x = degenerate(10000, 1, seed=19)
    ex = state_handle(x)
    ex.summary_begin(True)
    ex.summary_add_state()
    ex.set_outcomes([(_lib.OUTCOME_EXTREMA, 1, 6, 0)])  # the run maximum of world_pos[6]
    part = np.zeros(ex.sharded_quantiles_begin(LEVELS, "outcomes") // 4, np.uint32)
    n = ex.sharded_quantiles_round(None, 0, part)
    ex.summary_add_state()
    with pytest.raises(_lib.B200Error) as e:
        ex.sharded_quantiles_round(part, n, part)
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    part = np.zeros(ex.sharded_quantiles_begin(LEVELS, "state") // 4, np.uint32)
    n = ex.sharded_quantiles_round(None, 0, part)
    ex.summary_add_state()
    while n:
        n = ex.sharded_quantiles_round(part, n, part)
    assert same_bits(ex.sharded_quantiles_end(), ex.state_quantiles(LEVELS))
    tabs, _, _ = drive([ex], LEVELS, "outcomes")
    assert same_bits(tabs[0], ex.outcome_quantiles(LEVELS))


@pytest.mark.gpu
def test_protocol_errors_leave_the_handle_usable():
    need_gpu()
    x = degenerate(10000, 1, seed=17)
    exs = [state_handle(np.ascontiguousarray(x[a:b])) for a, b in cut(10000, [4000])]
    ex = exs[0]
    buf = np.zeros(1 << 20, np.uint32)

    def code(call):
        with pytest.raises(_lib.B200Error) as e:
            call()
        return e.value.code

    # round and end without a begin
    assert code(lambda: ex.sharded_quantiles_round(None, 0, buf)) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_quantiles_end()) == _lib.ERR_INVALID_ARGUMENT
    # bad levels, no groups when grouped
    assert code(lambda: ex.sharded_quantiles_begin((0.5, 1.5))) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_quantiles_begin((0.5,), "state", groups=True)) == _lib.ERR_INVALID_ARGUMENT
    # a wrong reduced_bytes and an end before the last round leave the call as it was
    bound = ex.sharded_quantiles_begin(LEVELS, "state")
    part = np.zeros(bound // 4, np.uint32)
    n = ex.sharded_quantiles_round(None, 0, part)
    assert n > 0
    assert code(lambda: ex.sharded_quantiles_round(part, n + 4, part)) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_quantiles_round(part, n, part[:1])) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_quantiles_end()) == _lib.ERR_INVALID_ARGUMENT
    # a step between rounds discards the call
    ex.step(1)
    assert code(lambda: ex.sharded_quantiles_round(part, n, part)) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_quantiles_round(None, 0, part)) == _lib.ERR_INVALID_ARGUMENT
    # the handles still reduce, sharded and not, and another reduction between rounds leaves a call valid
    b = [e.sharded_quantiles_begin(LEVELS, "state") for e in exs][0]
    bufs = [np.zeros(b // 4, np.uint32) for _ in exs]
    n, red = 0, None
    while True:
        got = [e.sharded_quantiles_round(red, n, q) for e, q in zip(exs, bufs)]
        for e in exs:
            e.state_quantiles((0.5,))
            e.state_stats()
        n = got[0]
        if n == 0:
            break
        red = bufs[0][: n // 4] + bufs[1][: n // 4]
    assert code(lambda: exs[0].sharded_quantiles_round(None, 0, bufs[0])) == _lib.ERR_INVALID_ARGUMENT  # after the last
    exs_all = state_handle(np.concatenate([sampled(e) for e in exs]))
    want = exs_all.state_quantiles(LEVELS)
    for e in exs:
        assert same_bits(e.sharded_quantiles_end(), want)


def sampled(ex):
    from tests.ensemble_util import sampled_state

    return sampled_state(ex)


# --------------------------------------------------------------------------- GPU: two gloo processes on one GPU

GLOO_M, GLOO_SIZES = 20001, [5000, 9500, 200, 5301]


def _gloo_data():
    from tests.util import near_world

    pos, vel, ine, cols, dt = near_world(21, GLOO_M, 2)
    vals = np.random.default_rng(22).normal(0.0, 1.0, (GLOO_M, 2))
    return (pos, vel, ine, cols, dt), vals


def _gloo_exec(a, b, sizes):
    (pos, vel, ine, cols, dt), vals = _gloo_data()
    ex = handle(ROCKET, b - a, 2, "exact", capacity=3,
                state=(pos[a:b], vel[a:b], ine[a:b], {k: v[a:b] for k, v in cols.items()}, dt))[0]
    ex.step(2)
    ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, vals[a:b, k]) for k in range(2)])
    ex.set_world_groups(sizes)
    return ex


def _gather_worker(rank, ws):
    a, b = sharding.shard_worlds(GLOO_M, rank, ws)
    ex = _gloo_exec(a, b, sharding.shard_groups(GLOO_SIZES, rank, ws))
    return {src: sharding.gather_quantiles(ex, LEVELS, src, groups=True) for src in ("ring", "state", "outcomes")}


def _mismatch_worker(rank, ws):
    a, b = sharding.shard_worlds(GLOO_M, rank, ws)
    ex = _gloo_exec(a, b, sharding.shard_groups(GLOO_SIZES, rank, ws))
    out = []
    for q in (LEVELS if rank == 0 else LEVELS[:-1], (0.5,) if rank == 0 else (1.5,)):
        try:
            sharding.gather_quantiles(ex, q, "state")
            out.append(None)
        except Exception as e:  # noqa: BLE001 - the error is the result
            out.append(type(e).__name__)
    # the handle still works after both refusals
    out.append(sharding.gather_quantiles(ex, (0.5,), "state").shape)
    return out


@pytest.mark.gpu
def test_gather_quantiles_over_two_gloo_processes():
    need_gpu()
    got = run_gloo(_gather_worker, 2)
    one = _gloo_exec(0, GLOO_M, GLOO_SIZES)
    want = {"ring": one.trajectory_group_quantiles(LEVELS), "state": one.state_group_quantiles(LEVELS),
            "outcomes": one.outcome_group_quantiles(LEVELS)}
    for r in got:
        for src, t in want.items():
            assert same_bits(r[src], t), src


@pytest.mark.gpu
def test_mismatched_levels_raise_on_every_rank():
    need_gpu()
    got = run_gloo(_mismatch_worker, 2)
    assert got[0][0] == got[1][0] == "ValueError"
    assert got[0][1] is not None and got[1][1] is not None  # rank 1's bad level: its begin fails, both raise
    assert got[0][2] == got[1][2]


CAMPAIGN_M, CAMPAIGN_GROUPS, CAMPAIGN_TICKS = 20000, [9000, 2000, 9000], 16


def _campaign(a, b, groups, process_group=None):
    from tests.ensemble_util import rocket_world

    w, sys_, params = rocket_world(CAMPAIGN_M)
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=24.0, n_worlds=b - a,
                 world_params={k: v[a:b] for k, v in params.items()}, ensemble=True, quantiles=LEVELS, groups=groups,
                 outcomes=[el.Outcome("z", "rocket.world_pos", 6)], process_group=process_group)
    ex.run(CAMPAIGN_TICKS)
    return {"quantiles": ex.quantiles("rocket.world_pos"), "group_quantiles": ex.quantiles("rocket.world_pos", groups=True),
            "outcome": ex.outcome_quantiles(LEVELS), "group_outcome": ex.outcome_quantiles(LEVELS, groups=True)}


def _campaign_worker(rank, ws):
    import torch.distributed as dist

    a, b = sharding.shard_worlds(CAMPAIGN_M, rank, ws)
    return _campaign(a, b, sharding.shard_groups(CAMPAIGN_GROUPS, rank, ws), dist.group.WORLD)


@pytest.mark.gpu
def test_world_build_with_a_process_group_equals_one_process():
    need_gpu()
    got = run_gloo(_campaign_worker, 2)
    want = _campaign(0, CAMPAIGN_M, CAMPAIGN_GROUPS)
    for r in got:
        for name, t in want.items():
            assert same_bits(r[name], t), name


@pytest.mark.gpu
def test_gather_quantiles_over_a_one_rank_nccl_group():
    """The NCCL route: the round words live in a CUDA buffer that the all-reduce and the handle's stream share."""
    need_gpu()
    import torch.distributed as dist

    if not dist.is_nccl_available() or dist.is_initialized():
        pytest.skip("needs NCCL and no process group in this process")
    x = degenerate(20011, 2, seed=23)
    ex = state_handle(x)
    ex.set_world_groups([9000, 11011])
    dist.init_process_group("nccl", rank=0, world_size=1, store=dist.HashStore())
    try:
        got = {g: sharding.gather_quantiles(ex, LEVELS, "state", groups=g) for g in (False, True)}
    finally:
        dist.destroy_process_group()
    assert same_bits(got[False], ex.state_quantiles(LEVELS))
    assert same_bits(got[True], ex.state_group_quantiles(LEVELS))
