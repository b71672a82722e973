"""World-sharded ranks (b200_sixdof_sharded_ranks_begin / _round / _end, sharding.gather_ranks,
gather_rank_correlation and the Exec-level collectives outcome_ranks, outcome_rank_correlation and outcome_sensitivity):
R handles hold consecutive slices of one campaign and rank their outcomes together, in rounds whose u32 words are summed
over the ranks.  Every rank's rank rows must be the rows of its worlds in the unsharded entry on one handle holding every
world, bit for bit, for any rank count and split; rho is the merged covariance of the ranks' rank planes.

The CPU tests check the bindings and prototypes, the refusals made before any backend call, and that an argument one
rank cannot use raises on every rank over two gloo processes.  The GPU tests drive simulated ranks in lockstep in one
process (the partials summed with numpy) over adversarial planes, group sizes at every route edge, several scratch
slices and a split key exchange, and check the rounds and the reads against the restated protocol of
test_sharded_rank_shapes (sharded_plan), the rho and PRCC contracts and the protocol's refusals; two gloo processes on
one GPU then run a whole campaign through World.build(..., process_group=)."""

import os
import re
import warnings

import numpy as np
import pytest
import scipy.stats

import elodin_b200 as el
from elodin_b200 import _lib, sharding
from elodin_b200.executor import merge_covariance, partial_rank_correlation, rank_correlation
from tests.ensemble_util import need_gpu, run_gloo
from tests.test_outcome_rank_correlation import _adversarial, _only_values, ref_ranks, same
from tests.test_sharded_rank_shapes import Split, sharded_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = 32 << 20  # include/b200_sixdof.h: the largest round of a sharded rank call, in bytes


# --------------------------------------------------------------------------- helpers


def cut(M, bounds):
    edges = [0] + list(bounds) + [M]
    return list(zip(edges[:-1], edges[1:]))


def drive(exs, planes, groups=False, between=None):
    """The rounds of every handle in lockstep, the partials summed (u32, wrapping) with numpy; `between(k)` runs after
    round k.  Returns ([(ranks, covariance records)] per rank, the round sizes, begin's bound)."""
    R = len(exs)
    bound = [ex.sharded_ranks_begin(planes, groups, r, R) for r, ex in enumerate(exs)]
    assert len(set(bound)) == 1 and bound[0] == CAP, bound
    bufs = [np.zeros(bound[0] // 4, np.uint32) for _ in exs]
    sizes, n, red = [], 0, None
    while True:
        got = [ex.sharded_ranks_round(red, n, b) for ex, b in zip(exs, bufs)]
        assert len(set(got)) == 1, got  # every rank makes the same rounds
        if between is not None:
            between(len(sizes))
        n = got[0]
        assert n <= bound[0] and n % 4 == 0
        sizes.append(n)
        if n == 0:
            break
        red = bufs[0][: n // 4].copy()
        for b in bufs[1:]:
            red += b[: n // 4]
    return [ex.sharded_ranks_end() for ex in exs], sizes, bound[0]


def sharded(values, bounds, planes, sizes=None):
    """The sharded ranks of values [M, p] over the ranks of `bounds` (grouped when `sizes` holds the global groups)."""
    M = values.shape[0]
    spans = cut(M, bounds)
    exs = []
    for a, b in spans:
        exs.append(_only_values(np.ascontiguousarray(values[a:b]), "fast",
                                None if sizes is None else sharding_cut(sizes, a, b)))
    out, rounds, bound = drive(exs, planes, sizes is not None)
    return exs, spans, out, rounds


def sharding_cut(sizes, a, b):
    out, g0 = [], 0
    for s in sizes:
        out.append(max(0, min(g0 + s, b) - max(g0, a)))
        g0 += s
    return out


def restated(values, planes, spans, sizes=None):
    """The restated protocol of the call over the ranks of `spans` (sharded_plan); its plans keep in bounds."""
    P = sharded_plan(values, sizes, planes, Split(len(spans), dict(enumerate(spans))))
    assert P["errors"] == [], P["errors"]
    return P


def check_reads(exs, P, sizes, p):
    tasks = len(sizes or [0]) * p
    for ex in exs:
        assert round(ex.rank_reads() * tasks) == P["reads"] and ex.rank_reads() == P["reads"] / tasks


def rho_of(covs, p):
    return rank_correlation(merge_covariance(covs), p)


# --------------------------------------------------------------------------- CPU


def test_sharded_rank_symbols_are_bound_and_declared():
    h = open(os.path.join(ROOT, "include", "b200_sixdof.h")).read()
    for name, args in (("b200_sixdof_sharded_ranks_begin", 7), ("b200_sixdof_sharded_ranks_round", 6),
                       ("b200_sixdof_sharded_ranks_end", 5)):
        m = re.search(name + r"\(([^)]*)\)", h)
        assert m and len(m.group(1).split(",")) == args, name
        assert name in _lib.SYMBOLS
        assert len(getattr(_lib.lib(), name).argtypes) == args
    assert "32 MiB" in h  # CAP above


class _Boom:
    def __getattr__(self, name):
        raise AssertionError("the executor must not be reached")


def test_gather_functions_refuse_bad_planes_before_any_call():
    for fn in (sharding.gather_ranks, sharding.gather_rank_correlation):
        for planes in ([], [0, 0], [-1], ["a"]):
            with pytest.raises(ValueError):
                fn(_Boom(), planes)
    with pytest.raises(ValueError, match="2 or more"):  # a correlation needs two planes, as the unsharded call
        sharding.gather_rank_correlation(_Boom(), [3])


def test_exec_collectives_refuse_before_any_backend_call(monkeypatch):
    from tests.test_host_logic import _FakeBackend
    from tests.test_outcome_rank_correlation import OUTS, _exec

    ex = _exec(monkeypatch, outcomes=OUTS)
    n0 = len(_FakeBackend.calls)
    with pytest.raises(_lib.B200Error, match="build the Exec with World.build") as e:  # not world-sharded
        sharding.outcome_sensitivity(ex, ["gain"], ["apogee"])
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    ex._pg = object()
    cases = [
        (lambda: sharding.outcome_sensitivity(ex, [], ["apogee"]), ValueError, "non-empty and disjoint"),
        (lambda: sharding.outcome_sensitivity(ex, ["gain", "t"], "t"), ValueError, "non-empty and disjoint"),
        (lambda: sharding.outcome_sensitivity(ex, ["gain"] * 2, ["t"]), ValueError, "distinct outcome names"),
        (lambda: sharding.outcome_sensitivity(ex, ["gain"], ["nosuch"]), _lib.B200ValueError, "outcome not found"),
        (lambda: sharding.outcome_sensitivity(ex, ["gain"], ["t"], groups=True), _lib.B200Error, r"groups=True"),
        (lambda: sharding.outcome_ranks(ex, ["apogee", "apogee"]), ValueError, "distinct outcome names"),
        (lambda: sharding.outcome_rank_correlation(ex, ["gain"]), ValueError, "2 or more distinct"),
        (lambda: sharding.outcome_rank_correlation(ex, ["gain", "x"]), _lib.B200ValueError, "outcome not found"),
    ]
    for call, exc, match in cases:
        with pytest.raises(exc, match=match):
            call()
    assert len(_FakeBackend.calls) == n0
    # the Exec methods still refuse a world-sharded Exec, and point at the collectives
    with pytest.raises(_lib.B200Error, match=r"not supported.*sharding\.outcome_sensitivity"):
        ex.outcome_sensitivity(["gain"], ["apogee"])
    assert len(_FakeBackend.calls) == n0


class _ArgumentsOnly:
    """An executor stand-in for the argument exchange of gather_ranks: its begin succeeds with no round to make."""

    n_worlds, world_groups, n_outcomes = 10, 1, 3

    def sharded_ranks_begin(self, planes, groups, rank, n_ranks):
        return 0


def _bad_argument_worker(rank, ws, kind):
    """Rank 1 passes planes it cannot use (or a different selection); every rank must raise, none may wait."""
    planes = {"repeated": ([0, 1], [1, 1]), "different": ([0, 1], [0, 2])}[kind][rank]
    try:
        sharding.gather_ranks(_ArgumentsOnly(), planes)
    except Exception as e:  # noqa: BLE001 - the error is the result
        return type(e).__name__
    return None


@pytest.mark.parametrize("kind", ["repeated", "different"])
def test_an_argument_one_rank_cannot_use_raises_on_every_rank(kind):
    assert run_gloo(_bad_argument_worker, 2, kind) == ["ValueError", "ValueError"]


# --------------------------------------------------------------------------- GPU: simulated ranks


def _check(values, bounds, planes, sizes=None, math="fast"):
    """Ranks over the ranks of `bounds` equal one handle's rows and scipy; the rho contract; returns the rounds."""
    exs, spans, out, rounds = sharded(values, bounds, planes, sizes)
    one = _only_values(values, math, sizes)
    want = one.outcome_group_ranks(planes) if sizes is not None else one.outcome_ranks(planes)
    assert same(want, ref_ranks(values[:, planes], sizes))
    for (a, b), (r, _) in zip(spans, out):
        assert same(r, want[a:b]), (a, b)
    P = restated(values, planes, spans, sizes)
    assert rounds == P["rounds"], rounds
    check_reads(exs, P, sizes, len(planes))
    return exs, spans, out, rounds, one


def _check_rho(values, planes, exs, spans, out, one, sizes=None):
    p = len(planes)
    covs = [c for _, c in out]
    got = rho_of(covs, p)
    # the restatement: handles holding each rank's campaign midranks as VALUES outcomes
    rest = []
    for (a, b), (r, _) in zip(spans, out):
        h = _only_values(r, "fast", None if sizes is None else sharding_cut(sizes, a, b))
        rest.append(h.outcome_group_covariance(list(range(p))) if sizes is not None else
                    h.outcome_covariance(list(range(p)))[None])
    assert same(got, rho_of(rest, p))
    direct = one.outcome_group_rank_correlation(planes) if sizes is not None else one.outcome_rank_correlation(planes)[None]
    if len(exs) == 1:
        assert same(got, direct)
    assert np.allclose(got, direct, atol=1e-12, rtol=0, equal_nan=True)
    o = 0
    for g, n in enumerate([values.shape[0]] if sizes is None else sizes):
        x = values[o:o + n][:, planes]
        x = x[np.all(np.isfinite(x), axis=1)]
        o += n
        assert got[g, 0] == x.shape[0]
        if x.shape[0] < 2:
            continue
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            st = np.atleast_2d(scipy.stats.spearmanr(x).statistic)
        want = np.array([[1.0, st[0, 0]], [st[0, 0], 1.0]]) if p == 2 else st
        for j in range(p):
            if np.all(x[:, j] == x[0, j]):
                want[j, :] = want[:, j] = np.nan
        assert np.allclose(got[g, 1:].reshape(p, p), want, atol=1e-12, rtol=0, equal_nan=True), g
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("R", [1, 2, 3, 5])
def test_ranks_over_ranks_equal_one_handle(R):
    need_gpu()
    M = 3 * 8192 + 4099
    values = _adversarial(M, seed=R)
    rng = np.random.default_rng(R)
    bounds = sorted(rng.choice(np.arange(1, M), R - 1, replace=False).tolist())
    planes = list(range(8))
    exs, spans, out, rounds, one = _check(values, bounds, planes)
    _check_rho(values, [0, 1, 3, 4, 6], *sharded(values, bounds, [0, 1, 3, 4, 6])[:3], one)
    for j in planes:  # each plane alone: its own finite worlds; the read bound on every plane
        e, _, o, r = sharded(values, bounds, [j])
        for (a, b), (rk, _) in zip(spans, o):
            assert same(rk, ref_ranks(values[:, [j]])[a:b]), j
        P = restated(values, [j], spans)
        assert r == P["rounds"], (j, r)
        check_reads(e, P, None, 1)


@pytest.mark.gpu
def test_uneven_splits_and_a_rank_without_complete_worlds():
    need_gpu()
    M = 2 * 8192 + 3
    values = _adversarial(M, seed=9)
    values[100:2100, 0] = np.nan  # rank 1's worlds: none complete
    for bounds in ([1, 100, 2100], [M - 1], [5000, 5001, 5002]):
        exs, spans, out, rounds, one = _check(values, bounds, [0, 2, 3, 5])
        _check_rho(values, [0, 2, 3, 5], exs, spans, out, one)


@pytest.mark.gpu
def test_grouped_route_edges_over_ranks():
    """Global groups of 0, 1, 2, 256, 257, 8192, 8193 and 2^20 + 5 worlds, cut so that some are empty on some ranks."""
    need_gpu()
    sizes = [0, 1, 2, 256, 257, 8192, 8193, (1 << 20) + 5]
    M = sum(sizes)
    values = _adversarial(M, seed=3)
    o = np.cumsum([0] + sizes)
    bounds = [int(o[4]) + 100, int(o[6]) + 5000, int(o[7]) + 4]
    planes = list(range(8))
    exs, spans, out, rounds, one = _check(values, bounds, planes, sizes)
    assert len(restated(values, planes, spans, sizes)["slices"]) >= 2  # the 2^20 + 5 group's 8 tasks need two
    _check_rho(values, [0, 1, 2, 4, 6], *sharded(values, bounds, [0, 1, 2, 4, 6], sizes)[:3], one, sizes)


@pytest.mark.gpu
def test_several_scratch_slices():
    """25 planes x 64 groups of 8193 worlds: more tasks than one 256 MiB slice holds, on 2 ranks."""
    need_gpu()
    sizes = [8193] * 64
    rng = np.random.default_rng(9)
    values = rng.normal(0, 1, (sum(sizes), 25))
    values[:, 7] = np.round(values[:, 7] * 3)
    values[rng.random(values.shape) < 0.0005] = np.nan
    order = list(range(25))[::-1]
    exs, spans, out, rounds, one = _check(values, [sum(sizes) // 3], order, sizes)
    # every group has at most 8192 complete worlds: one bucket per task, so each slice makes no histogram exchange and
    # the offsets and the keys of each window of its keys
    P = restated(values, order, spans, sizes)
    assert len(P["slices"]) >= 2 and P["hist"] == [] and len(rounds) == 1 + 2 * len(P["windows"]) + 1


@pytest.mark.gpu
def test_a_split_key_exchange_and_the_scratch_bound():
    """One group of 6 * 10^6 continuous worlds on 4 ranks: its keys (8 bytes per bucket world) take more than one
    window, no round reaches the cap, and the device memory a rank's call takes stays within a window's exchange, the
    histograms of the ranges that exist and 64 bytes per world of its own, not a multiple of the group's global size;
    the call frees it at its end."""
    need_gpu()
    import torch

    M, R = 6_000_000, 4
    values = np.random.default_rng(5).normal(0, 1, (M, 1))
    spans = cut(M, [M * k // R for k in range(1, R)])
    exs = [_only_values(np.ascontiguousarray(values[a:b]), "fast") for a, b in spans]
    torch.cuda.init()
    bound = [ex.sharded_ranks_begin([0], False, r, R) for r, ex in enumerate(exs)][0]
    torch.cuda.synchronize()
    base = torch.cuda.mem_get_info()[0]
    least = base
    bufs = [np.zeros(bound // 4, np.uint32) for _ in exs]
    rounds, n, red = [], 0, None
    while True:
        got = [ex.sharded_ranks_round(red, n, b) for ex, b in zip(exs, bufs)]
        least = min(least, torch.cuda.mem_get_info()[0])
        n = got[0]
        assert len(set(got)) == 1
        rounds.append(n)
        if n == 0:
            break
        red = sum(b[: n // 4] for b in bufs[1:]) + bufs[0][: n // 4]
    out = [ex.sharded_ranks_end() for ex in exs]
    want = ref_ranks(values)
    for (a, b), (r, _) in zip(spans, out):
        assert same(r, want[a:b])
    P = restated(values, [0], spans)
    assert rounds == P["rounds"] and max(rounds) < CAP and len(P["windows"]) >= 2, rounds  # a level, two windows
    check_reads(exs, P, None, 1)
    used = base - least
    per_rank = CAP + (16 << 20) + 64 * (M // R)
    assert used <= R * per_rank, (used, R * per_rank)
    assert used < R * 40 * M  # a plan sized by the global count would take this much
    # freed at the end: what stays is the handles' shared staging buffer, which the end's ranks went through
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] >= base - (8 * M + R * (2 << 20) + (8 << 20))


@pytest.mark.gpu
def test_prcc_from_the_merged_rho():
    need_gpu()
    M = 30000
    rng = np.random.default_rng(2)
    x = rng.normal(size=(M, 3))
    y = x @ np.array([1.0, -0.5, 0.1]) + rng.normal(scale=0.3, size=M)
    values = np.column_stack([x, np.round(y, 1)])
    exs, spans, out, rounds, one = _check(values, [7000, 20000], [0, 1, 2, 3])
    R = rho_of([c for _, c in out], 4)[0, 1:].reshape(4, 4)
    prcc = partial_rank_correlation(R)
    direct = one.outcome_rank_correlation([0, 1, 2, 3])[1:].reshape(4, 4)
    assert np.allclose(prcc, partial_rank_correlation(direct), atol=1e-10)
    assert prcc[0] > 0.9 and prcc[1] < -0.7


@pytest.mark.gpu
def test_protocol_errors_leave_the_handle_usable():
    need_gpu()
    M = 20000
    values = _adversarial(M, seed=17)
    planes = [0, 1, 4]
    exs = [_only_values(np.ascontiguousarray(values[a:b]), "fast") for a, b in cut(M, [8000])]
    ex = exs[0]
    buf = np.zeros(CAP // 4, np.uint32)

    def code(call):
        with pytest.raises(_lib.B200Error) as e:
            call()
        return e.value.code

    assert code(lambda: ex.sharded_ranks_round(None, 0, buf)) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_ranks_end()) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_ranks_begin([0, 0], False, 0, 2)) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_ranks_begin([9], False, 0, 2)) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_ranks_begin([0], True, 0, 2)) == _lib.ERR_INVALID_ARGUMENT  # no groups
    assert code(lambda: ex.sharded_ranks_begin([0], False, 2, 2)) == _lib.ERR_INVALID_ARGUMENT  # rank >= n_ranks
    # a wrong reduced_bytes, a small partial and an end before the last round leave the call as it was
    ex.sharded_ranks_begin(planes, False, 0, 1)
    n = ex.sharded_ranks_round(None, 0, buf)
    assert n > 0
    assert code(lambda: ex.sharded_ranks_round(buf, n + 4, buf)) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_ranks_round(buf, n, buf[:1])) == _lib.ERR_INVALID_ARGUMENT
    assert code(lambda: ex.sharded_ranks_end()) == _lib.ERR_INVALID_ARGUMENT
    while n:
        n = ex.sharded_ranks_round(buf, n, buf)
    assert same(ex.sharded_ranks_end()[0], ex.outcome_ranks(planes))
    # a rows change (a step, new outcomes) or an unsharded rank call between rounds discards the call
    for change in (lambda: ex.step(1), lambda: ex.set_world_groups([8000]), lambda: ex.outcome_ranks([0]),
                   lambda: ex.outcome_rank_correlation([0, 1])):
        ex.sharded_ranks_begin(planes, False, 0, 1)
        n = ex.sharded_ranks_round(None, 0, buf)
        change()
        assert code(lambda: ex.sharded_ranks_round(buf, n, buf)) == _lib.ERR_INVALID_ARGUMENT
        assert code(lambda: ex.sharded_ranks_round(None, 0, buf)) == _lib.ERR_INVALID_ARGUMENT
    ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, np.ascontiguousarray(values[:8000, j])) for j in range(8)])
    # another reduction between rounds leaves the call valid; both handles still rank together
    def other(k):
        for e in exs:
            e.outcome_quantiles((0.5,))
            e.outcome_covariance([0, 1])
            e.outcome_top_worlds([0], 3, True)

    out, _, _ = drive(exs, planes, between=other)
    want = ref_ranks(values[:, planes])
    assert same(out[0][0], want[:8000]) and same(out[1][0], want[8000:])


# --------------------------------------------------------------------------- GPU: two gloo processes on one GPU

CAMPAIGN_M, CAMPAIGN_GROUPS, CAMPAIGN_TICKS = 20000, [9000, 2000, 9000], 16


def _campaign(a, b, groups, process_group=None):
    from tests.ensemble_util import rocket_world

    w, sys_, params = rocket_world(CAMPAIGN_M)
    p = {k: v[a:b] for k, v in params.items()}
    outcomes = [el.Outcome.values("thrust", p["thrust"][:, 0, 0]), el.Outcome.values("wind", p["wind"][:, 0, 0]),
                el.Outcome.values("mass", p["inertia"][:, 0, 6]), el.Outcome("z", "rocket.world_pos", 6),
                el.Outcome("x", "rocket.world_pos", 4)]
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=24.0, n_worlds=b - a, world_params=p, ensemble=True,
                 groups=groups, outcomes=outcomes, process_group=process_group)
    ex.run(CAMPAIGN_TICKS)
    inputs, outputs = ["thrust", "wind", "mass"], ["z", "x"]
    if process_group is None:
        return {"sens": ex.outcome_sensitivity(inputs, outputs), "gsens": ex.outcome_sensitivity(inputs, outputs, True),
                "ranks": ex.outcome_ranks(["z", "mass"], groups=True)}
    return {"sens": sharding.outcome_sensitivity(ex, inputs, outputs),
            "gsens": sharding.outcome_sensitivity(ex, inputs, outputs, groups=True),
            "ranks": sharding.outcome_ranks(ex, ["z", "mass"], groups=True),
            "corr": sharding.outcome_rank_correlation(ex, ["z", "mass", "x"])}


def _campaign_worker(rank, ws):
    import torch.distributed as dist

    a, b = sharding.shard_worlds(CAMPAIGN_M, rank, ws)
    return _campaign(a, b, sharding.shard_groups(CAMPAIGN_GROUPS, rank, ws), dist.group.WORLD)


@pytest.mark.gpu
def test_outcome_sensitivity_over_two_gloo_processes_equals_one_process():
    need_gpu()
    got = run_gloo(_campaign_worker, 2)
    want = _campaign(0, CAMPAIGN_M, CAMPAIGN_GROUPS)
    for r in got:
        for key in ("sens", "gsens"):
            for f in ("count", "rho", "prcc"):
                assert np.allclose(r[key][f], want[key][f], atol=1e-12, rtol=0, equal_nan=True), (key, f)
            assert r[key]["inputs"] == want[key]["inputs"] and r[key]["outputs"] == want[key]["outputs"]
        assert same(r["sens"]["rho"], got[0]["sens"]["rho"]) and same(r["sens"]["prcc"], got[0]["sens"]["prcc"])
        assert r["corr"]["names"] == ["z", "mass", "x"] and r["corr"]["rho"].shape == (3, 3)
    for name in ("z", "mass"):
        assert same(np.concatenate([r["ranks"][name] for r in got]), want["ranks"][name]), name
