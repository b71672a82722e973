"""Worst worlds of a Monte-Carlo batch (b200_sixdof_outcome_[group_]top_worlds, topk_kernels.cu): per group and
selected outcome, the first k finite worlds in IEEE totalOrder (descending for largest), ties by ascending world index.

The CPU tests check every Exec.outcome_top_worlds refusal before the backend is reached, the constants and prototypes
against the header, the numpy restatement of the order on hand cases, the host merge of per-rank records over random
splits, the collective over a 2-rank gloo group, and that an Exec which never asks for worst worlds makes the backend
calls it made before.  The GPU tests, in both math modes, hold every record to the numpy restatement bit for bit and
index for index: on a rocket campaign, on adversarial planes at every route edge (group sizes, slices of the scratch,
ties across the compaction cap, signed zeros and non-finite values), per group against a handle over the group,
merged over simulated ranks against one handle, through retained rows and a re-run of the flagged worlds, and through
the C ABI's refusals, destinations and a caller stream."""

import ctypes
import os
import re

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200.executor import merge_top_worlds
from elodin_b200.sharding import shard_groups, shard_sizes
from tests.ensemble_util import need_gpu, rocket_world, run_gloo, split, two_body_world
from tests.test_ensemble_outcomes import _OutcomeFake, _values_handle, campaign
from tests.test_host_logic import _FakeBackend

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("exact", "fast")
O = el.Outcome
READ_BOUND = 10  # include/b200_sixdof.h: at most 10 reads of the planes on any data


# --------------------------------------------------------------------------- the numpy restatement of the order


def ref_top(x, k, largest, offset=0):
    """[1 + 2k] record of values x (world w = offset + index): the finite worlds ordered by the totalOrder key
    (complemented for largest), ties by world, the first k; NaN / -1 past the count."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    world = np.arange(x.size, dtype=np.int64) + offset
    fin = np.isfinite(x)
    u = x[fin].view(np.uint64)
    key = np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))
    if largest:
        key = ~key
    order = np.lexsort((world[fin], key))[:k]
    rec = np.full(1 + 2 * k, np.nan)
    rec[0] = fin.sum()
    rec[1 + k:] = -1.0
    rec[1:1 + order.size] = x[fin][order]
    rec[1 + k:1 + k + order.size] = world[fin][order]
    return rec


def bits(x):
    x = np.array(x, dtype=np.float64)
    x[np.isnan(x)] = np.nan
    return x.view(np.uint64)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


def test_reference_order_on_hand_cases():
    nan, inf, big, tiny = np.nan, np.inf, np.finfo(np.float64).max, 5e-324
    x = np.array([0.0, -0.0, nan, inf, -inf, big, -big, tiny, -tiny, 1.0])
    r = ref_top(x, 10, False)
    assert r[0] == 7
    assert list(r[11:18]) == [6, 8, 1, 0, 7, 9, 5] and list(r[18:]) == [-1, -1, -1]
    assert same(r[1:8], [-big, -tiny, -0.0, 0.0, tiny, 1.0, big]) and np.all(np.isnan(r[8:11]))
    r = ref_top(x, 3, True)
    assert list(r[4:]) == [5, 9, 7] and same(r[1:4], [big, 1.0, tiny])
    assert list(ref_top(x, 7, True)[8:])[-2:] == [8, 6]
    r = ref_top(np.array([-0.0, 0.0, -0.0, 0.0]), 4, True)  # +0 above -0, ties by world
    assert list(r[5:]) == [1, 3, 0, 2]
    r = ref_top(np.full(6, 2.5), 4, True)  # ties across the plane: the lowest worlds, either direction
    assert list(r[5:]) == [0, 1, 2, 3] and list(ref_top(np.full(6, 2.5), 4, False)[5:]) == [0, 1, 2, 3]
    r = ref_top(np.array([nan, 3.0, inf, 1.0]), 2, False)  # exactly k finite
    assert r[0] == 2 and list(r[3:]) == [3, 1]
    r = ref_top(np.array([nan, inf, -inf]), 2, True)  # none finite
    assert r[0] == 0 and np.all(np.isnan(r[1:3])) and list(r[3:]) == [-1, -1]
    assert list(ref_top(np.array([1.0, 2.0]), 1, True, offset=10)[2:]) == [11]


def test_host_merge_over_random_splits():
    rng = np.random.default_rng(5)
    for trial in range(40):
        n = int(rng.integers(0, 300))
        x = np.round(rng.normal(0, 2, n))  # many ties, which straddle the ranks
        x[rng.random(n) < 0.1] = np.nan
        x[rng.random(n) < 0.05] = -0.0
        k = int(rng.integers(1, 40))
        largest = bool(trial % 2)
        parts = split(rng, n, int(rng.integers(1, 6)))  # empty ranks included
        tables = [ref_top(x[p], k, largest)[None] for p in parts]
        offsets = [int(p[0]) if p.size else sum(q.size for q in parts[:i]) for i, p in enumerate(parts)]
        got = merge_top_worlds(tables, offsets, largest)
        assert same(got[0], ref_top(x, k, largest)), trial
    with pytest.raises(ValueError, match="2 tables and 1 offsets"):
        merge_top_worlds([np.zeros(3), np.zeros(3)], [0], True)
    with pytest.raises(_lib.B200ValueError):
        merge_top_worlds([np.zeros(4)], [0], True)


def test_header_constants_and_prototypes():
    h = open(os.path.join(ROOT, "include", "b200_sixdof.h")).read()
    assert int(re.search(r"#define B200_MAX_TOP_WORLDS (\d+)u", h).group(1)) == _lib.MAX_TOP_WORLDS == 1024
    for name, args in (("b200_sixdof_outcome_top_worlds", 7), ("b200_sixdof_outcome_group_top_worlds", 7),
                       ("b200_sixdof_top_worlds_reads", 1)):
        m = re.search(name + r"\(([^)]*)\)", h)
        assert m and len(m.group(1).split(",")) == args, name
        assert name in _lib.SYMBOLS, name
    src = open(os.path.join(ROOT, "elodin_b200", "_lib.py")).read()
    assert "L.b200_sixdof_outcome_top_worlds.argtypes = [vp, C.POINTER(u32), u32, u32, C.c_int, vp, u64]" in src
    assert "L.b200_sixdof_outcome_group_top_worlds.argtypes = [vp, C.POINTER(u32), u32, u32, C.c_int, vp, u64]" in src
    assert "L.b200_sixdof_top_worlds_reads.restype = C.c_double" in src


# --------------------------------------------------------------------------- CPU: Exec through a fake backend


class _TopFake(_OutcomeFake):
    """The outcome fake with the worst-worlds calls logged and records whose worlds name their slot."""

    def _top(self, name, planes, k, largest, G=None):
        self._log(name, list(planes), k, largest)
        rec = np.full((len(planes), 1 + 2 * k), np.nan)
        rec[:, 0] = 7.0
        rec[:, 1:1 + k] = np.arange(k) + 0.5
        rec[:, 1 + k:] = np.arange(k)
        return rec if G is None else np.broadcast_to(rec, (G,) + rec.shape).copy()

    def outcome_top_worlds(self, planes, k, largest):
        return self._top("outcome_top_worlds", planes, k, largest)

    def outcome_group_top_worlds(self, planes, k, largest):
        return self._top("outcome_group_top_worlds", planes, k, largest, self.n_groups)


def _exec(monkeypatch, **kw):
    from elodin_b200 import world as W

    monkeypatch.setattr(W, "B200Exec", _TopFake)
    _FakeBackend.calls = []
    args = dict(simulation_rate=120.0, telemetry_rate=40.0, n_worlds=5, ensemble=True, ensemble_ring=2, extrema=True,
                thresholds=[el.Threshold("rocket.world_pos", 6, below=0.0)])
    args.update(kw)
    ex = two_body_world().build(el.six_dof(), **args)
    ex.run(7)
    return ex


OUTS = [O("apogee", "rocket.world_pos", 6, "max"), O.threshold("t", 0, "tick"), O.values("gain", np.arange(5.0))]


def test_refusals_before_any_backend_call(monkeypatch):
    ex = _exec(monkeypatch, outcomes=OUTS)
    n0 = len(_FakeBackend.calls)
    for kw, exc, match in (
        (dict(k=0), ValueError, r"k = 0, an int in \[1, 1024\]"),
        (dict(k=1025), ValueError, "k = 1025"),
        (dict(k=2.0), ValueError, "k = 2.0"),
        (dict(k=True), ValueError, "k = True"),
        (dict(k="3"), ValueError, "k = '3'"),
        (dict(k=3, largest=1), TypeError, "largest = 1, a bool"),
        (dict(k=3, largest=None), TypeError, "largest = None"),
        (dict(k=3, names=["apogee", "apogee"]), ValueError, "distinct outcome names"),
        (dict(k=3, names=[]), ValueError, "distinct outcome names"),
        (dict(k=3, names=["nosuch"]), _lib.B200ValueError, "outcome not found: 'nosuch'"),
        (dict(k=3, groups=True), _lib.B200Error, r"outcome_top_worlds\(groups=True\).*groups=\[...\]"),
    ):
        with pytest.raises(exc, match=match):
            ex.outcome_top_worlds(**kw)
    assert len(_FakeBackend.calls) == n0
    plain = _exec(monkeypatch)
    with pytest.raises(_lib.B200Error, match=r"outcome_top_worlds\(\): build the Exec with .*outcomes=\[...\]"):
        plain.outcome_top_worlds(3)


def test_an_exec_that_never_asks_makes_the_same_calls(monkeypatch):
    """The worst-worlds entry adds no backend call of its own to an Exec's run; asking adds exactly one."""
    _exec(monkeypatch, outcomes=OUTS, groups=[2, 3])
    before = list(_FakeBackend.calls)
    assert not any("top_worlds" in c[0] for c in before)
    from tests.test_ensemble_outcomes import _calls

    _, with_outcomes = _calls(monkeypatch, outcomes=OUTS)
    assert not any("top_worlds" in c[0] for c in with_outcomes)
    ex = _exec(monkeypatch, outcomes=OUTS, groups=[2, 3])
    assert _FakeBackend.calls == before
    got = ex.outcome_top_worlds(4, names=["gain", "apogee"], largest=False)
    assert _FakeBackend.calls == before + [("outcome_top_worlds", [2, 0], 4, False)]
    assert got["names"] == ["gain", "apogee"] and np.array_equal(got["count"], [7.0, 7.0])
    assert got["world"].dtype == np.int64 and np.array_equal(got["world"], np.tile(np.arange(4), (2, 1)))
    assert np.array_equal(got["value"], np.tile(np.arange(4) + 0.5, (2, 1)))
    g = ex.outcome_top_worlds(2, groups=True)
    assert _FakeBackend.calls[-1] == ("outcome_group_top_worlds", [0, 1, 2], 2, True)
    assert g["count"].shape == (2, 3) and g["world"].shape == (2, 3, 2)


# --------------------------------------------------------------------------- CPU: the collective over gloo


class _RankExec:
    """A rank's executor as gather_top_worlds sees it: its own worlds' values and the restatement's records."""

    def __init__(self, values, sizes=None):
        self.values, self.sizes, self.n_worlds = values, sizes, values.shape[0]

    def outcome_top_worlds(self, planes, k, largest):
        if not 1 <= k <= _lib.MAX_TOP_WORLDS:
            raise _lib.B200Error(_lib.ERR_INVALID_ARGUMENT, f"top worlds k = {k}")
        return np.stack([ref_top(self.values[:, p], k, largest) for p in planes])

    def outcome_group_top_worlds(self, planes, k, largest):
        out, o = [], 0
        for n in self.sizes:
            out.append(np.stack([ref_top(self.values[o:o + n, p], k, largest, o) for p in planes]))
            o += n
        return np.stack(out)


def _gloo_worker(rank, ws, values, ks, sizes):
    from elodin_b200.sharding import gather_top_worlds, shard_worlds

    w0, w1 = shard_worlds(values.shape[0], rank, ws)
    ex = _RankExec(values[w0:w1], shard_groups(sizes, rank, ws))
    got = [gather_top_worlds(ex, [2, 0], 5, True), gather_top_worlds(ex, [1], 3, False, groups=True)]
    try:
        gather_top_worlds(ex, [0], ks[rank], True)
        got.append(None)
    except (ValueError, _lib.B200Error) as e:
        got.append(type(e).__name__ + ": " + str(e))
    try:
        gather_top_worlds(ex, [0], 2000 if rank == 1 else 2, True)
        got.append(None)
    except (ValueError, _lib.B200Error) as e:
        got.append(type(e).__name__ + ": " + str(e))
    return got


def test_gather_over_two_gloo_ranks():
    rng = np.random.default_rng(2)
    values = np.round(rng.normal(0, 3, (23, 3)))
    values[rng.random((23, 3)) < 0.1] = np.nan
    sizes = [5, 0, 10, 8]
    got = run_gloo(_gloo_worker, 2, values, [4, 5], sizes)
    want0 = np.stack([ref_top(values[:, p], 5, True) for p in (2, 0)])
    o = np.concatenate([[0], np.cumsum(sizes)])
    want1 = np.stack([ref_top(values[o[g]:o[g + 1], 1], 3, False, o[g])[None] for g in range(4)])
    for rank, (a, b, differ, failed) in enumerate(got):
        assert same(a, want0) and same(b, want1), rank
        assert differ and "rank 1 differs from rank 0" in differ, rank  # raised on both ranks, no hang
        assert failed and "top worlds k = 2000" in failed or "rank 1 failed" in failed, rank


# --------------------------------------------------------------------------- GPU


def _check(got, values, k, largest, sizes=None):
    """Every record of a table [p, 1 + 2k] (or [G, p, 1 + 2k] over `sizes`) against the restatement."""
    if sizes is None:
        for j in range(values.shape[1]):
            assert same(got[j], ref_top(values[:, j], k, largest)), (j, k, largest)
        return
    o = 0
    for g, n in enumerate(sizes):
        for j in range(values.shape[1]):
            assert same(got[g, j], ref_top(values[o:o + n, j], k, largest, o)), (g, j, k, largest)
        o += n


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_rocket_campaign_records_equal_the_restatement(math):
    need_gpu()
    M = 300
    sizes = [100, 37, 163]
    ex, _, _ = campaign(M, math, "resident", groups=sizes)
    v = ex.outcome_values()
    names = ex.outcomes
    vals = np.stack([v[n] for n in names], axis=1)
    be = ex.backend
    planes = list(range(len(names)))
    counts = np.isfinite(vals).sum(0)
    ks = sorted({1, 7, 1024} | {int(c) + d for c in counts for d in (-1, 0, 1) if 1 <= int(c) + d <= 1024})
    for k in ks:
        for largest in (False, True):
            _check(be.outcome_top_worlds(planes, k, largest), vals, k, largest)
    for k in (1, 7, 36, 37, 38, 1024):
        for largest in (False, True):
            _check(be.outcome_group_top_worlds(planes, k, largest), vals, k, largest, sizes)
    assert be.top_worlds_reads() == 1.0  # small groups: one read
    got = ex.outcome_top_worlds(16, names=["apogee", "t_hit"], largest=True)
    assert same(got["value"][0], ref_top(v["apogee"], 16, True)[1:17])
    assert np.array_equal(got["world"][1], ref_top(v["t_hit"], 16, True)[17:].astype(np.int64))


def _adversarial(M, seed):
    """[M, 6] planes: continuous, rounded (ties), all equal, mixed signed zeros and non-finite values, a tie block of
    20000 worlds at 1.0 with 500 worlds above it spread over the plane, and few distinct values (dwell-like counts)."""
    rng = np.random.default_rng(seed)
    v = np.empty((M, 6))
    v[:, 0] = rng.normal(0, 1, M)
    v[:, 1] = np.round(rng.normal(0, 30, M))
    v[:, 2] = 3.25
    z = rng.integers(0, 5, M)
    v[:, 3] = np.choose(z, [0.0, -0.0, np.nan, np.inf, -np.inf])
    v[:, 3][rng.random(M) < 0.01] = 7.0
    v[:, 4] = rng.uniform(-1.0, 0.999, M)
    tie = rng.permutation(M)[: min(M, 20000)]
    v[tie, 4] = 1.0
    above = rng.permutation(M)[: min(M, 500)]
    v[above, 4] = rng.uniform(1.5, 2.0, above.size)
    v[:, 5] = rng.integers(0, 4, M).astype(np.float64)
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_route_edges_and_adversarial_planes(math):
    need_gpu()
    sizes = [0, 1, 255, 256, 257, 8191, 8192, 8193, (1 << 20) + 1]
    M = sum(sizes)
    values = _adversarial(M, seed=1)
    ex = _values_handle(values, math, groups=sizes)
    planes = list(range(values.shape[1]))
    for k, largest in ((1, True), (16, False), (1024, True), (1024, False), (700, True)):
        got = ex.outcome_group_top_worlds(planes, k, largest)
        _check(got, values, k, largest, sizes)
        assert 1.0 <= ex.top_worlds_reads() <= READ_BOUND
    # ungrouped over the 2^20 + 1 worlds alone: the bound on every plane, 3 reads on a uniform one
    big = values[-sizes[-1]:]
    one = _values_handle(big, math)
    for j in range(big.shape[1]):
        for k, largest in ((1024, True), (1024, False), (5, True)):
            _check(one.outcome_top_worlds([j], k, largest), big[:, [j]], k, largest)
            assert one.top_worlds_reads() <= READ_BOUND, (j, k)
    u = np.random.default_rng(3).uniform(0.0, 1.0, (big.shape[0], 1))
    uni = _values_handle(u, math)
    for k, largest in ((16, True), (1024, False), (1024, True)):
        _check(uni.outcome_top_worlds([0], k, largest), u, k, largest)
        assert uni.top_worlds_reads() <= 3.0, k
    eq = _values_handle(np.full((big.shape[0], 1), -2.0), math)  # all equal: the lowest world indices
    got = eq.outcome_top_worlds([0], 1024, True)
    assert np.array_equal(got[0, 1025:], np.arange(1024)) and eq.top_worlds_reads() <= READ_BOUND


@pytest.mark.gpu
def test_two_scratch_slices():
    """25 planes x 64 groups of 8193 worlds: more large tasks than one 256 MiB slice of the scratch holds."""
    need_gpu()
    sizes = [8193] * 64
    rng = np.random.default_rng(9)
    values = rng.normal(0, 1, (sum(sizes), 25))
    values[:, 7] = np.round(values[:, 7] * 3)
    values[rng.random(values.shape) < 0.02] = np.nan
    ex = _values_handle(values, "fast", groups=sizes)
    got = ex.outcome_group_top_worlds(list(range(25))[::-1], 33, True)
    _check(got, values[:, ::-1], 33, True, sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_group_records_equal_a_handle_over_the_group(math):
    need_gpu()
    sizes = [0, 300, 57, 8643, 9000]
    values = _adversarial(sum(sizes), seed=4)
    ex = _values_handle(values, math, E=3, groups=sizes)
    got = ex.outcome_group_top_worlds([5, 0, 4], 50, False)
    o = 0
    for g, n in enumerate(sizes):
        if n:
            sub = _values_handle(values[o:o + n], math, E=2).outcome_top_worlds([5, 0, 4], 50, False)
            sub[:, 51:][sub[:, 51:] >= 0] += o
            assert same(got[g], sub), g
        else:
            assert np.all(got[g, :, 0] == 0) and np.all(got[g, :, 51:] == -1)
        o += n


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_sharded_ranks_merge_into_the_whole(math):
    need_gpu()
    rng = np.random.default_rng(6)
    M = 20000
    values = _adversarial(M, seed=6)
    sizes = [3000, 0, 9000, 8000]
    whole = _values_handle(values, math, groups=sizes)
    planes = [4, 1, 3]
    want = whole.outcome_top_worlds(planes, 64, True)
    want_g = whole.outcome_group_top_worlds(planes, 20, False)
    for parts in (shard_sizes(M, 2), shard_sizes(M, 3), [int(p.size) for p in split(rng, M, 4)]):
        offs = np.concatenate([[0], np.cumsum(parts)[:-1]])
        hs = [_values_handle(values[o:o + n], math) for o, n in zip(offs, parts) if n]
        live = [o for o, n in zip(offs, parts) if n]
        got = merge_top_worlds([h.outcome_top_worlds(planes, 64, True) for h in hs], live, True)
        assert same(got, want), parts
        tabs = []
        for r, (o, n) in enumerate(zip(offs, parts)):
            if n:
                h = _values_handle(values[o:o + n], math, groups=shard_groups(sizes, r, len(parts)) if len(parts) in (2, 3)
                                   else _cut(sizes, o, n))
                tabs.append(h.outcome_group_top_worlds(planes, 20, False))
        assert same(merge_top_worlds(tabs, live, False), want_g), parts


def _cut(sizes, o, n):
    """The global group sizes cut to the world range [o, o + n) (shard_groups for an arbitrary split)."""
    out, g0 = [], 0
    for s in sizes:
        out.append(max(0, min(g0 + s, o + n) - max(g0, o)))
        g0 += s
    return out


def _loop_campaign(M, math, retain=None, params=None):
    w, sys_, p = rocket_world(M)
    params = p if params is None else params
    outs = [O("apogee", "rocket.world_pos", 6, "max"), O.threshold("t_down", 0, "tick")]
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=40.0, n_worlds=M, math=math, world_params=params,
                 ensemble=True, extrema=True, thresholds=[el.Threshold("rocket.world_pos", 6, below=1.0)],
                 outcomes=outs, retain=retain)
    ex.run(90)
    return ex, p


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_flagged_worlds_replay_through_retain_and_a_rerun(math):
    need_gpu()
    M = 2000
    ex, params = _loop_campaign(M, math)
    top = ex.outcome_top_worlds(8, largest=True)
    low = ex.outcome_top_worlds(8, names=["t_down"], largest=False)
    v = ex.outcome_values()
    assert same(top["value"][0], ref_top(v["apogee"], 8, True)[1:9])
    flagged = sorted(set(top["world"][0].tolist()) | set(low["world"][0][low["world"][0] >= 0].tolist()))
    re_ex, _ = _loop_campaign(M, math, retain=flagged)
    z = re_ex.history_worlds("rocket.world_pos")[..., 6]  # [rows, k]
    tpr = re_ex.ticks_per_telemetry
    for slot, w in enumerate(flagged):
        col = z[:, slot]
        fin = col[np.isfinite(col)]
        assert same(fin.max(), v["apogee"][w]), w
        below = np.nonzero(col < 1.0)[0]
        assert same(below[0] * tpr if below.size else np.nan, v["t_down"][w]), w
    if math == "exact":  # a campaign of just the flagged worlds' parameters gives them their values bit for bit
        sub = {k: np.ascontiguousarray(a[flagged]) for k, a in params.items()}
        ex2, _ = _loop_campaign(len(flagged), math, params=sub)
        v2 = ex2.outcome_values()
        assert same(v2["apogee"], v["apogee"][flagged]) and same(v2["t_down"], v["t_down"][flagged])


def _refused(call, code, match):
    with pytest.raises(_lib.B200Error, match=match) as e:
        call()
    assert e.value.code == code


@pytest.mark.gpu
def test_abi_refusals_destinations_and_a_caller_stream():
    need_gpu()
    import torch

    M = 9000
    values = _adversarial(M, seed=8)[:, :3]
    ex = el.B200Exec(1, M, 0.01, None, [], "rk4", "exact")
    INV = _lib.ERR_INVALID_ARGUMENT
    _refused(lambda: ex.outcome_top_worlds([0], 3, True), INV, "no outcomes: call b200_sixdof_set_outcomes first")
    ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, values[:, j]) for j in range(3)])
    L, h = ex._L, ex._h
    out = np.empty(64)
    u32p = ctypes.POINTER(ctypes.c_uint32)

    def call(planes, n_p, k, largest, nbytes, grouped=False):
        fn = L.b200_sixdof_outcome_group_top_worlds if grouped else L.b200_sixdof_outcome_top_worlds
        arr = None if planes is None else (ctypes.c_uint32 * max(len(planes), 1))(*planes)
        return lambda: _lib.check(fn(h, ctypes.cast(arr, u32p) if arr is not None else None, n_p, k, largest,
                                     ctypes.c_void_p(out.ctypes.data), nbytes))

    _refused(call(None, 1, 3, 1, 56), INV, "null top-worlds planes")
    _refused(call([0], 0, 3, 1, 56), INV, "0 top-worlds planes: 1 to 3")
    _refused(call([0, 1, 2, 0], 4, 3, 1, 56), INV, "4 top-worlds planes: 1 to 3")
    _refused(call([3], 1, 3, 1, 56), INV, "top-worlds plane 0 is 3: the outcome has 3 planes")
    _refused(call([1, 1], 2, 3, 1, 56), INV, "top-worlds plane 1 listed twice")
    _refused(call([0], 1, 0, 1, 56), INV, "top worlds k = 0: 1 to 1024")
    _refused(call([0], 1, 1025, 1, 56), INV, "top worlds k = 1025")
    _refused(call([0], 1, 3, 2, 56), INV, "top worlds largest = 2: 0 or 1")
    _refused(call([0], 1, 3, 1, 48), _lib.ERR_VALUE_SIZE_MISMATCH, "outcome top worlds are 56 bytes, got 48")
    _refused(call([0], 1, 3, 1, 56, grouped=True), INV, "grouped outcome top worlds: call b200_sixdof_set_world_groups")
    call([0], 1, 3, 1, 56)()
    assert same(out[:7], ref_top(values[:, 0], 3, True))
    # a summary that drops what an outcome names: refused, naming the outcome
    ex2 = el.B200Exec(1, 50, 0.01, None, [], "rk4", "exact")
    ex2.summary_begin(True, [(0, 6, False, 0.0)])
    ex2.set_outcomes([(_lib.OUTCOME_THRESHOLD, 0, 0)])
    ex2.summary_begin(True)
    _refused(lambda: ex2.outcome_top_worlds([0], 3, True), INV, "outcome 0: threshold 0, the summary in force has 0")
    # host and device destinations, and a caller-owned stream: the same records
    sizes = [100, 8900]
    ex.set_world_groups(sizes)
    want = ex.outcome_group_top_worlds([2, 0], 300, False)
    _check(want, values[:, [2, 0]], 300, False, sizes)
    dev = torch.empty(want.size, dtype=torch.float64, device="cuda")
    ex._reduce("group_top_worlds", "outcome", ex._selection([2, 0]) + (300, 0), want.shape, dev.data_ptr())
    torch.cuda.synchronize()
    assert same(dev.cpu().numpy().reshape(want.shape), want)
    s = torch.cuda.Stream()
    ex.set_stream(s.cuda_stream)
    with torch.cuda.stream(s):
        dev2 = torch.full((want.size,), 5.0, dtype=torch.float64, device="cuda")
        ex._reduce("group_top_worlds", "outcome", ex._selection([2, 0]) + (300, 0), want.shape, dev2.data_ptr())
        back = dev2.cpu()  # ordered after the entry on the caller's stream
    assert same(back.numpy().reshape(want.shape), want)
    assert same(ex.outcome_group_top_worlds([2, 0], 300, False), want)
    ex.set_stream(None)
