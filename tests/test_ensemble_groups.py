"""Grouped ensembles: the statistics and histograms of every contiguous world range (one sweep point of a campaign) in
one call.  The defining property: group g's record has the bits of the ungrouped call on a handle that holds exactly
the group's worlds.  CPU: World.build's groups= validation, monte_carlo.plan_groups, sharding.shard_groups and the
merge of grouped tables.  GPU: the grouped entries against per-group handles and numpy, and Exec's grouped tables
against one Exec per group."""

import ctypes
import json
import os

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200 import monte_carlo as mc
from elodin_b200.sharding import shard_groups, shard_worlds
from tests.ensemble_util import need_gpu, no_device, rocket_world, run_gloo, two_body_world  # noqa: F401
from tests.test_ensemble_histograms import SPECS, catalogue, check_conservation, ref_row, state_handle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("exact", "fast")


def stats_wc(E):
    """stats_kernels.cu stats_shape, restated: the worlds of a chunk while a group has at most 64 chunks of the least
    size (kMinPerThread = 8 values per lane), and the size of a group of exactly 64 such chunks."""
    J = 256 // E if E <= 256 else 1
    return 8 * J, 64 * 8 * J


# --------------------------------------------------------------------------- CPU: World.build, plans, shards, merge


def test_build_validates_groups_before_the_device(no_device):
    w, sys_ = two_body_world(), el.six_dof()
    with pytest.raises(ValueError, match="ensemble=True"):
        w.build(sys_, n_worlds=4, groups=[2, 2])
    with pytest.raises(ValueError, match="sum to 5, not to n_worlds = 4"):
        w.build(sys_, n_worlds=4, ensemble=True, groups=[2, 3])
    with pytest.raises(ValueError, match="negative"):
        w.build(sys_, n_worlds=4, ensemble=True, groups=[5, -1])
    for bad in ([2.0, 2], [True, 3], ["2", 2]):
        with pytest.raises(TypeError, match="not an integer"):
            w.build(sys_, n_worlds=4, ensemble=True, groups=bad)
    for bad in ("22", 4, {2: 2}):
        with pytest.raises(TypeError):
            w.build(sys_, n_worlds=4, ensemble=True, groups=bad)
    with pytest.raises(ValueError, match="0 groups: 1 to 1024"):
        w.build(sys_, n_worlds=4, ensemble=True, groups=[])
    with pytest.raises(ValueError, match="1025 groups: 1 to 1024"):
        w.build(sys_, n_worlds=1025, ensemble=True, groups=[1] * 1025)
    with pytest.raises(AssertionError, match="before the handle"):  # a valid setting reaches the device
        w.build(sys_, n_worlds=1024, ensemble=True, groups=np.ones(1024, dtype=np.int64))


def _mixed_dists():
    with open(os.path.join(ROOT, "tests", "golden", "mc_plans.json")) as f:
        spec = json.load(f)["mixed_dists"]["spec"]
    import tomllib

    return mc.materialize(tomllib.loads(spec))


def test_plan_groups_on_the_golden_mixed_dists_plan(tmp_path):
    rows = _mixed_dists()
    assert len(rows) == 102
    same, sizes, keys = mc.plan_groups(rows, ["param.gain"])
    assert same == rows and sizes == [51, 51] and keys == [{"param.gain": 0.5}, {"param.gain": 1.0}]
    same, sizes, keys = mc.plan_groups(rows, ["param.gain", "meta.label"])
    assert same == rows and sizes == [17] * 6
    assert keys == [{"param.gain": g, "meta.label": lab} for g in (0.5, 1.0) for lab in "xyz"]
    got, sizes, keys = mc.plan_groups(rows, ["meta.label"])
    assert sizes == [34, 34, 34] and keys == [{"meta.label": lab} for lab in "xyz"]
    assert sorted(r["run_id"] for r in got) == sorted(r["run_id"] for r in rows)  # every row once, whole
    by_id = {r["run_id"]: r for r in rows}
    assert all(r is by_id[r["run_id"]] for r in got)
    for g, lab in enumerate("xyz"):
        part = got[34 * g:34 * (g + 1)]
        assert all(r["meta.label"] == lab for r in part)
        assert [r["seed"] for r in part] == sorted(r["seed"] for r in part)  # plan order inside the group
    # read_plan rows: the same grouping, keys named as in the plan
    path = tmp_path / "plan.csv"
    mc.write_plan(rows, path)
    read = mc.read_plan(path)
    got_r, sizes_r, keys_r = mc.plan_groups(read, ["meta.label"])
    assert sizes_r == sizes and keys_r == keys and [r["run_id"] for r in got_r] == [r["run_id"] for r in got]
    for bad in (["param.nope"], ["gain"], ["meta.label", "meta.x"]):
        with pytest.raises(ValueError, match=bad[-1].replace(".", r"\.")):
            mc.plan_groups(rows, bad)


@pytest.mark.parametrize("seed", range(6))
def test_shard_groups_cut_the_global_groups(seed):
    rng = np.random.default_rng(seed)
    G = int(rng.integers(1, 12))
    sizes = [int(x) if rng.random() > 0.3 else 0 for x in rng.integers(0, 40, G)]
    n = sum(sizes)
    for ws in range(1, 6):
        parts = [shard_groups(sizes, r, ws) for r in range(ws)]
        for r, p in enumerate(parts):
            w0, w1 = shard_worlds(n, r, ws)
            assert len(p) == G and min(p) >= 0 and sum(p) == w1 - w0
        assert [sum(col) for col in zip(*parts)] == sizes


def _stats_part(rng, G, empty):
    t = np.empty((G, 5))
    for g in range(G):
        x = rng.normal(size=int(rng.integers(1, 50))) * 10.0 ** rng.integers(-3, 4)
        t[g] = (0.0, np.nan, np.nan, np.nan, np.nan) if empty[g] else (
            x.size, x.mean(), ((x - x.mean()) ** 2).sum(), x.min(), x.max())
    return t


def test_merge_of_grouped_tables_skips_empty_parts():
    rng = np.random.default_rng(3)
    G, P = 40, 4
    empty = rng.random((P, G)) < 0.4
    empty[:, 0] = True  # a group no part holds
    parts = [_stats_part(rng, G, empty[p]) for p in range(P)]
    got = el.merge_stats(parts)
    for g in range(G):
        full = [p[g:g + 1] for k, p in enumerate(parts) if not empty[k, g]]
        want = el.merge_stats(full)[0] if full else np.array([0.0, np.nan, np.nan, np.nan, np.nan])
        assert got[g].tobytes() == want.tobytes(), g


# --------------------------------------------------------------------------- GPU: the grouped entries


def states(M, E, seed):
    """x [M, E, 25]: normal draws with a few NaN and inf, per-world offsets so that groups differ."""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(M, E, 25)) * rng.uniform(0.5, 3.0, (M, 1, 1)) + rng.normal(size=(M, 1, 1)) * 100
    x[rng.random((M, E, 25)) < 0.01] = np.nan
    x[rng.random((M, E, 25)) < 0.002] = np.inf
    return x


def ring_handle(x, mode, width):
    """A free-body handle over the state x with a ring of two samples after two ticks."""
    M, E, _ = x.shape
    ex = state_handle(x, mode, trajectory_every=1, trajectory_capacity=2, trajectory_full=width == 25)
    ex.step(2)
    return ex


def offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(int)


def group_sizes(E):
    wc, wide = stats_wc(E)
    return [0, 1, 7, wc - 1, wc, wc + 1, 0, wide, 3]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("E", [1, 3, 300])
def test_group_stats_equal_one_handle_per_group(E, mode):
    need_gpu()
    sizes = group_sizes(E)
    o = offsets(sizes)
    x = states(int(o[-1]), E, seed=E)
    for width in (13, 25):
        with ring_handle(x, mode, width) as ex:
            ex.set_world_groups(sizes)
            assert ex.world_groups == len(sizes)
            st, tr = ex.state_group_stats(), ex.trajectory_group_stats()
            traj = ex.trajectory()
            assert st.shape == (len(sizes), E, 25, 5) and tr.shape == (2, len(sizes), E, width, 5)
            for g, n in enumerate(sizes):
                if n == 0:
                    assert np.all(st[g, ..., 0] == 0) and np.all(np.isnan(st[g, ..., 1:]))
                    assert np.all(tr[:, g, ..., 0] == 0) and np.all(np.isnan(tr[:, g, ..., 1:]))
                    continue
                with ring_handle(np.ascontiguousarray(x[o[g]:o[g + 1]]), mode, width) as one:
                    assert np.array_equal(one.trajectory(), traj[:, o[g]:o[g + 1]], equal_nan=True)  # the same samples
                    assert np.array_equal(st[g], one.state_stats(), equal_nan=True), (g, n)
                    assert np.array_equal(tr[:, g], one.trajectory_stats(), equal_nan=True), (g, n, width)


@pytest.mark.gpu
def test_g1_and_g2_groups():
    need_gpu()
    E = 3
    x = states(5000, E, seed=11)
    with state_handle(x, "exact") as ex:
        all_ = ex.state_stats()
        ex.set_world_groups([5000])
        assert np.array_equal(ex.state_group_stats()[0], all_, equal_nan=True)  # G = 1: the ungrouped table
        ex.set_world_groups([1234, 3766])
        two = ex.state_group_stats()
        for g, (a, b) in enumerate(((0, 1234), (1234, 5000))):
            with state_handle(np.ascontiguousarray(x[a:b]), "exact") as one:
                assert np.array_equal(two[g], one.state_stats(), equal_nan=True)


@pytest.mark.gpu
def test_1024_groups():
    need_gpu()
    rng = np.random.default_rng(5)
    sizes = [int(s) if rng.random() > 0.1 else 0 for s in rng.integers(0, 60, 1024)]
    sizes[100] = 2600  # one group of several chunks among many of one
    o = offsets(sizes)
    E = 3
    x = states(int(o[-1]), E, seed=6)
    with state_handle(x, "exact") as ex:
        ex.set_world_groups(sizes)
        st = ex.state_group_stats()
    for g, n in enumerate(sizes):
        if n == 0:
            assert np.all(st[g, ..., 0] == 0) and np.all(np.isnan(st[g, ..., 1:])), g
            continue
        v = x[o[g]:o[g + 1]]
        f = np.isfinite(v)
        assert np.array_equal(st[g, ..., 0], f.sum(0).astype(float)), g
        with np.errstate(invalid="ignore"):
            mn = np.where(f.any(0), np.min(np.where(f, v, np.inf), 0), np.nan)
            mx = np.where(f.any(0), np.max(np.where(f, v, -np.inf), 0), np.nan)
        assert np.array_equal(st[g, ..., 3], mn, equal_nan=True) and np.array_equal(st[g, ..., 4], mx, equal_nan=True)
    for g in list(range(0, 1024, 64)) + [100]:
        if sizes[g] == 0:
            continue
        with state_handle(np.ascontiguousarray(x[o[g]:o[g + 1]]), "exact") as one:
            assert np.array_equal(st[g], one.state_stats(), equal_nan=True), g


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_group_histograms_equal_numpy_per_group(mode):
    need_gpu()
    specs = SPECS[:2] + SPECS[4:6]
    sizes = [0, 1, 5000, 7, 0, 12000, 1025]
    o = offsets(sizes)
    x = catalogue(specs, int(o[-1]), 3, seed=8)
    with state_handle(x, mode, trajectory_every=1, trajectory_capacity=1, trajectory_full=True) as ex:
        ungrouped = ex.state_histograms(specs)
        ex.set_world_groups(sizes)
        got = ex.state_group_histograms(specs)
        ex.step(1)
        tr = ex.trajectory_group_histograms(specs)
        tr_all = ex.trajectory_histograms(specs)
        traj = ex.trajectory()
    assert got.shape == (len(sizes), ungrouped.shape[0])
    for g in range(len(sizes)):
        assert got[g].tobytes() == ref_row(x[o[g]:o[g + 1]], specs).tobytes(), g
        assert tr[0, g].tobytes() == ref_row(traj[0, o[g]:o[g + 1]], specs).tobytes(), g
        check_conservation(got[g], specs, sizes[g])
    assert got.sum(0).tobytes() == ungrouped.tobytes() and tr[0].sum(0).tobytes() == tr_all[0].tobytes()


@pytest.mark.gpu
def test_ungrouped_entries_do_not_change_with_groups():
    need_gpu()
    x = states(6000, 2, seed=9)
    specs = SPECS[4:5]
    with ring_handle(x, "exact", 25) as a, ring_handle(x, "exact", 25) as b:
        b.set_world_groups([100, 0, 5900])
        assert np.array_equal(a.state_stats(), b.state_stats(), equal_nan=True)
        assert np.array_equal(a.trajectory_stats(), b.trajectory_stats(), equal_nan=True)
        assert a.state_histograms(specs).tobytes() == b.state_histograms(specs).tobytes()
        assert a.trajectory_histograms(specs).tobytes() == b.trajectory_histograms(specs).tobytes()
        b.set_world_groups([])
        assert b.world_groups == 0


@pytest.mark.gpu
def test_grouped_entry_errors_and_launches():
    need_gpu()
    x = states(3000, 2, seed=10)
    u64p = ctypes.POINTER(ctypes.c_uint64)
    with state_handle(x, "exact") as ex:
        L, h = ex._L, ex._h
        buf = np.empty(10 ** 6)
        for fn in (L.b200_sixdof_state_group_stats, L.b200_sixdof_trajectory_group_stats):
            assert fn(h, buf.ctypes.data, 8) == _lib.ERR_INVALID_ARGUMENT  # no groups set
        specs, _ = ex._hist_specs(SPECS[:1])
        assert L.b200_sixdof_state_group_histograms(h, *specs, buf.ctypes.data, 8) == _lib.ERR_INVALID_ARGUMENT
        for sizes, n in (([1000, 1999], 2), ([3001], 1), ([1] * 1025, 1025)):
            a = np.asarray(sizes, dtype=np.uint64)
            assert L.b200_sixdof_set_world_groups(h, a.ctypes.data_as(u64p), n) == _lib.ERR_INVALID_ARGUMENT
        assert L.b200_sixdof_set_world_groups(h, None, 3) == _lib.ERR_INVALID_ARGUMENT
        assert ex.world_groups == 0
        ex.set_world_groups([1000, 0, 2000])
        want = 3 * 2 * 25 * 5 * 8
        assert L.b200_sixdof_state_group_stats(h, buf.ctypes.data, want - 8) == _lib.ERR_VALUE_SIZE_MISMATCH
        rec = 3 + SPECS[0][2]
        assert L.b200_sixdof_state_group_histograms(h, *specs, buf.ctypes.data, 3 * rec * 8 + 8) == _lib.ERR_VALUE_SIZE_MISMATCH
        n0 = ex.timings()["kernel_launches"]
        ex.state_group_stats()                    # groups of 1000 and 2000 worlds, 2 entities: several chunks
        n1 = ex.timings()["kernel_launches"]
        ex.state_group_histograms(SPECS[:1])
        n2 = ex.timings()["kernel_launches"]
    assert n1 - n0 == 2 and n2 - n1 == 1


# --------------------------------------------------------------------------- GPU: Exec


def _group_params(params, a, b):
    return {k: np.ascontiguousarray(v[a:b]) for k, v in params.items()}


HISTS = lambda: [el.Histogram("rocket.world_pos", 6, range=(-5.0, 40.0), bins=64),  # noqa: E731
                 el.Histogram("rocket.world_vel", (3, 5), range=((-30.0, 30.0), (-30.0, 30.0)), bins=(16, 8))]


@pytest.mark.gpu
@pytest.mark.parametrize("host_cb", [False, True])
def test_exec_grouped_tables_equal_one_exec_per_group(host_cb):
    need_gpu()
    M, sizes = 4096, [1000, 2500, 596]
    o = offsets(sizes)
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=12.0, math="exact", ensemble=True)
    post = (lambda tick, ctx: None) if host_cb else None
    ex = w.build(sys_, n_worlds=M, world_params=params, histograms=HISTS(), groups=sizes, **kw)
    ex.run(50, post_step=post)
    plain = w.build(sys_, n_worlds=M, world_params=params, histograms=HISTS(), **kw)
    plain.run(50, post_step=post)
    assert ex.groups == sizes
    for pair in ("rocket.world_pos", "ball.world_vel", "rocket.force"):
        a, b = ex.ensemble(pair), plain.ensemble(pair)
        for k in a:
            assert np.array_equal(a[k], b[k], equal_nan=True), (pair, k)
    for g in range(len(sizes)):
        one = w.build(sys_, n_worlds=sizes[g], world_params=_group_params(params, o[g], o[g + 1]), histograms=HISTS(), **kw)
        one.run(50, post_step=post)
        for pair in ("rocket.world_pos", "ball.world_vel", "rocket.world_accel"):
            got, want = ex.ensemble(pair, groups=True), one.ensemble(pair)
            for k in got:
                assert got[k].shape[:2] == (6, len(sizes))
                assert np.array_equal(got[k][:, g], want[k], equal_nan=True), (g, pair, k)
        for i in range(2):
            got, want = ex.histogram(i, groups=True), one.histogram(i)
            for k in want:
                if k != "edges":
                    assert np.array_equal(got[k][:, g], want[k]), (g, i, k)
    with pytest.raises(_lib.B200Error, match="groups"):
        plain.ensemble("rocket.world_pos", groups=True)


# --------------------------------------------------------------------------- GPU: two gloo ranks


def _sharded_worker(rank, ws, sizes, M):
    from elodin_b200.sharding import gather_ensemble, gather_histograms, shard_groups, shard_worlds

    w0, w1 = shard_worlds(M, rank, ws)
    x = states(M, 2, seed=12)[w0:w1]
    with ring_handle(np.ascontiguousarray(x), "exact", 25) as ex:
        ex.set_world_groups(shard_groups(sizes, rank, ws))
        return gather_ensemble(ex.trajectory_group_stats()), gather_histograms(ex.trajectory_group_histograms(SPECS[4:5]))


@pytest.mark.gpu
def test_two_gloo_ranks_gather_grouped_tables():
    need_gpu()
    M, sizes = 20_001, [3000, 0, 9000, 4000, 4001]  # the shard boundary at 10 001 splits group 2
    got = run_gloo(_sharded_worker, 2, sizes, M)
    with ring_handle(states(M, 2, seed=12), "exact", 25) as ex:
        ex.set_world_groups(sizes)
        want, want_h = ex.trajectory_group_stats(), ex.trajectory_group_histograms(SPECS[4:5])
    for stats, hist in got:
        assert hist.tobytes() == want_h.tobytes()
        for g in (0, 1, 3, 4):
            assert np.array_equal(stats[:, g], want[:, g], equal_nan=True), g
        split = stats[:, 2]
        assert np.array_equal(split[..., 0], want[:, 2, ..., 0])
        assert np.array_equal(split[..., 3:], want[:, 2, ..., 3:], equal_nan=True)
        scale = np.abs(want[:, 2, ..., 1]) + np.sqrt(want[:, 2, ..., 2] / want[:, 2, ..., 0]) + 1.0
        assert np.all(np.abs(split[..., 1] - want[:, 2, ..., 1]) <= 1e-12 * scale)
        assert np.allclose(split[..., 2], want[:, 2, ..., 2], rtol=1e-11, atol=0)


# --------------------------------------------------------------------------- edge cases: plans, empty worlds, slices


def test_plan_groups_edge_cases():
    assert mc.plan_groups([], ["param.gain"]) == ([], [], [])
    nan = float("nan")
    rows = [{"run_id": f"r{i}", "seed": i + 1, "param.gain": v} for i, v in enumerate([nan, 1.0, float("nan"), 1.0, nan])]
    got, sizes, keys = mc.plan_groups(rows, ["param.gain"])  # every NaN one value, as every 1.0 is
    assert sizes == [3, 2] and [r["run_id"] for r in got] == ["r0", "r2", "r4", "r1", "r3"]
    assert np.isnan(keys[0]["param.gain"]) and keys[1] == {"param.gain": 1.0}


@pytest.mark.gpu
def test_zero_entity_handle_takes_groups():
    need_gpu()
    with el.B200Exec(0, 4, 0.01, None, [], "rk4", "exact", trajectory_every=1, trajectory_capacity=2,
                     trajectory_full=True) as ex:
        ex.step(2)
        ex.set_world_groups([3, 0, 1])
        assert ex.world_groups == 3
        assert ex.state_group_stats().shape == (3, 0, 25, 5)
        assert ex.trajectory_group_stats().shape == (2, 3, 0, 25, 5)
        assert ex.state_stats().shape == (0, 25, 5)
        with pytest.raises(_lib.B200Error) as e:  # no entity row 0 to histogram
            ex.state_group_histograms(SPECS[:1])
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        with pytest.raises(_lib.B200Error) as e:
            ex.set_world_groups([3])
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT and ex.world_groups == 3


@pytest.mark.gpu
def test_sliced_partials_equal_one_slice():
    """E = 300 and 16 samples of 25 planes: the ring's partials (58 chunks ungrouped, 67 over the groups) take more than
    256 MiB, so the ring's tables run in two slices of planes; each sample equals the state's table (one slice) taken
    at its tick, bit for bit."""
    need_gpu()
    sizes, E, S = [0, 512, 3, 0], 300, 16
    x = states(sum(sizes), E, seed=13)
    with state_handle(x, "exact", trajectory_every=1, trajectory_capacity=S, trajectory_full=True) as ex:
        ex.set_world_groups(sizes)
        one, grouped = [], []
        for _ in range(S):
            ex.step(1)
            one.append(ex.state_stats())
            grouped.append(ex.state_group_stats())
        got, n1 = _launches(ex, ex.trajectory_stats)
        got_g, n2 = _launches(ex, ex.trajectory_group_stats)
        _, n_one = _launches(ex, ex.state_stats)
    assert n1 == 4 and n2 == 4 and n_one == 2  # two slices of a chunk and a merge launch, against one slice
    assert np.array_equal(got, np.stack(one), equal_nan=True)
    assert np.array_equal(got_g, np.stack(grouped), equal_nan=True)


def _launches(ex, call):
    n0 = ex.timings()["kernel_launches"]
    got = call()
    return got, ex.timings()["kernel_launches"] - n0
