"""Grouped quantiles and covariance: the percentile envelopes and joint spreads of every contiguous world range (one
sweep point of a campaign) in one call.  The defining property: group g's record has the bits of the ungrouped entry
on a handle that holds exactly the group's worlds.  CPU: World.build's validation of groups= with quantiles= /
covariance=, the accessors' refusals, and a restatement of the covariance group table and its slices.  GPU: the
grouped entries against per-group handles, numpy and the exact references, at every route and chunking edge, the
invariants of the one-group case, Exec on both run routes, and two gloo ranks."""

import ctypes

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200.sharding import shard_groups, shard_worlds
from elodin_b200.world import Exec
from tests.ensemble_util import need_gpu, no_device, rocket_world, run_gloo, two_body_world  # noqa: F401
from tests.test_ensemble_covariance import check_table, ref_table, scales
from tests.test_ensemble_histograms import state_handle
from tests.test_ensemble_quantiles import _degenerate, ref_quantiles
from tests.test_ensemble_shapes import SLICE_GROUPS, cdiv, cov_chunks, cov_launches

MODES = ("exact", "fast")
LEVELS = (0.0, 1e-3, 0.01, 1 / 3, 0.5, 0.99, 1.0)
CAP = 256 << 20  # the scratch bound of a covariance slice
WARP_MAX, SMALL_MAX = 256, 8192


def offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(int)


# --------------------------------------------------------------------------- restatements of the launch contract


def cov_group_table(sizes, E):
    """cov_kernels.cu cov_group_table: (Wc, C, k0) per group; an empty group is one chunk of no worlds."""
    out, k0 = [], 0
    for n in sizes:
        Wc, C = cov_chunks(n, E) if n else (0, 1)
        out.append((Wc, C, k0))
        k0 += C
    return out


def cov_slices(sizes, E, p, samples=1):
    """cov_kernels.cu cov_slices: [(g0, g1, s0, ns)], consecutive groups while one sample's partials of their chunks fit
    in 256 MiB, then as many samples as fit (every sample where no group of the slice has more than one chunk)."""
    t = cov_group_table(sizes, E)
    per_chunk = E * (1 + p + p * p) * 8
    out, g0 = [], 0
    while g0 < len(t):
        g1, chunks = g0 + 1, t[g0][1]
        while g1 < len(t) and (chunks + t[g1][1]) * per_chunk <= CAP:
            chunks += t[g1][1]
            g1 += 1
        merge = any(t[g][1] > 1 for g in range(g0, g1))
        ns = max(1, CAP // (chunks * per_chunk)) if merge else samples
        out += [(g0, g1, s0, min(ns, samples - s0), merge) for s0 in range(0, samples, ns)]
        g0 = g1
    return out


def cov_group_launches(sizes, E, p, samples=1):
    return sum(2 if merge else 1 for *_, merge in cov_slices(sizes, E, p, samples))


def quantile_group_launches(sizes, E, planes=25):
    """quantile_kernels.cu launch_quantiles: one launch per sort route with groups, 18 per radix slice of (group,
    plane) rows (whole rows, or entity ranges of one row)."""
    warp = any(n <= WARP_MAX for n in sizes)
    block = any(WARP_MAX < n <= SMALL_MAX for n in sizes)
    rows = sum(n > SMALL_MAX for n in sizes) * planes
    slices = 0
    if rows:
        slices = cdiv(rows, max(1, SLICE_GROUPS // E)) if E <= SLICE_GROUPS else rows * cdiv(E, SLICE_GROUPS)
    return warp + block + 18 * slices


# --------------------------------------------------------------------------- CPU


def test_build_validates_grouped_quantiles_and_covariance_before_the_device(no_device):
    w, sys_ = two_body_world(), el.six_dof()
    kw = dict(n_worlds=4, ensemble=True)
    with pytest.raises(ValueError, match="not in \\[0, 1\\]"):
        w.build(sys_, groups=[2, 2], quantiles=[0.5, 1.5], **kw)
    with pytest.raises(ValueError, match="twice"):
        w.build(sys_, groups=[2, 2], covariance=[("world_pos", (4, 4))], **kw)
    with pytest.raises(ValueError, match="sum to 5"):
        w.build(sys_, groups=[2, 3], quantiles=[0.5], covariance=["world_pos"], **kw)
    with pytest.raises(ValueError, match="ensemble=True"):
        w.build(sys_, n_worlds=4, groups=[2, 2])
    with pytest.raises(AssertionError, match="before the handle"):  # a valid setting reaches the device
        w.build(sys_, groups=[0, 4], quantiles=[0.01, 0.99], covariance=[("world_pos", (4, 5, 6))], **kw)


def _bare_exec(kinds):
    ex = Exec.__new__(Exec)
    ex._ens_rows = {k: [] for k in kinds}
    ex._cov_labels = ["world_pos[4]"]
    return ex


def test_accessors_refuse_without_groups():
    ex = _bare_exec(["stats", "quantiles", "covariance", "histograms"])
    with pytest.raises(_lib.B200Error, match=r"quantiles\(groups=True\): build the Exec with World.build\(\.\.\., "
                                             r"ensemble=True, quantiles=\[\.\.\.\], groups=\[\.\.\.\]\)") as e:
        ex.quantiles("rocket.world_pos", groups=True)
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    with pytest.raises(_lib.B200Error, match=r"covariance\(groups=True\): build the Exec with World.build\(\.\.\., "
                                             r"ensemble=True, covariance=\[\.\.\.\], groups=\[\.\.\.\]\)") as e:
        ex.covariance("rocket", groups=True)
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT


def test_covariance_group_table_on_hand_worked_splits():
    # 63 / 64 / 65 worlds at E = 1: one chunk up to 64 worlds (kMinWorlds), then two of 33; an empty group is one chunk
    assert cov_group_table([0, 63, 64, 65, 0], 1) == [(0, 1, 0), (63, 1, 1), (64, 1, 2), (33, 2, 3), (0, 1, 5)]
    # the chunk count saturates at kChunkTasks = 528 for E = 1 (528 * 64 worlds); one world more takes chunks of 65
    assert cov_group_table([528 * 64 - 1, 528 * 64, 528 * 64 + 1], 1) == [(64, 528, 0), (64, 528, 528), (65, 520, 1056)]
    # E = 32 is one entity tile, E = 33 two: half the chunks
    assert cov_group_table([67584], 32) == [(128, 528, 0)] and cov_group_table([67584], 33) == [(256, 264, 0)]
    # G = 1 is the ungrouped call: its launches and slices of whole samples
    for M, E, p, S in ((5, 1, 3, 1), (1 << 16, 1, 25, 1), (1 << 16, 1, 25, 40), (100, 300, 6, 16), (1 << 20, 2, 25, 300)):
        assert cov_group_launches([M], E, p, S) == cov_launches(M, E, p, S), (M, E, p, S)
    # 1024 groups of 33 792 worlds at p = 25: 2.8 GB of partials for one sample, run as 97 groups a slice
    sizes = [528 * 64] * 1024
    per_group = 528 * (1 + 25 + 625) * 8
    assert per_group * 1024 > 2.8e9
    sl = cov_slices(sizes, 1, 25)
    assert [(g0, g1) for g0, g1, *_ in sl] == [(g, min(g + 97, 1024)) for g in range(0, 1024, 97)]
    assert all((g1 - g0) * per_group <= CAP for g0, g1, *_ in sl) and 98 * per_group > CAP
    assert cov_group_launches(sizes, 1, 25) == 22
    # one-chunk groups need no scratch: one slice of every sample, one launch
    assert cov_slices([10, 0, 64], 1, 25, 7) == [(0, 3, 0, 7, False)] and cov_group_launches([10, 0, 64], 1, 25, 7) == 1


def test_quantile_route_launches_restated():
    assert quantile_group_launches([0, 1, 2, 255, 256], 3) == 1
    assert quantile_group_launches([257, 8192], 3) == 1
    assert quantile_group_launches([0, 300, 9000], 3) == 2 + 18
    assert quantile_group_launches([8193], 1) == 18
    assert quantile_group_launches([8193] * 55, 1) == 18 * 2  # 1375 (group, plane) rows: two slices


# --------------------------------------------------------------------------- GPU helpers


def catalogue(sizes, E, seed):
    """x [M, E, 25]: the degenerate catalogue of the shape tests per entity (ties, +-0, subnormals, NaN / +-inf, a plane
    without a finite world, orbital offsets, +-DBL_MAX), with per-world offsets on some planes so that groups differ,
    and one non-empty group whose plane 6 is all non-finite."""
    M = int(sum(sizes))
    x = np.stack([_degenerate(M, seed=seed + e) for e in range(E)], axis=1)
    rng = np.random.default_rng(seed)
    x[:, :, 3] += np.repeat(np.arange(len(sizes), dtype=float), sizes)[:, None] * 0.25
    o = offsets(sizes)
    big = [g for g, n in enumerate(sizes) if n > 0]
    if big:
        g = big[len(big) // 2]
        x[o[g]:o[g + 1], :, 6] = rng.choice([np.nan, np.inf, -np.inf], (sizes[g], E))
    return np.ascontiguousarray(x)


def numpy_quantiles(v, q):
    """np.quantile over the finite values of v [n] (NaN where none)."""
    f = v[np.isfinite(v)]
    with np.errstate(over="ignore", invalid="ignore"):  # numpy's lerp between -DBL_MAX and DBL_MAX
        return np.quantile(f, q) if f.size else np.full(len(q), np.nan)


def _launches(ex, call):
    n0 = ex.timings()["kernel_launches"]
    got = call()
    return got, ex.timings()["kernel_launches"] - n0


# --------------------------------------------------------------------------- GPU: quantiles

QUANTILE_CASES = {
    "sort edges": ([0, 1, 2, 255, 256, 257, 0], 3),
    "radix edge": ([8192, 0, 8193], 1),
    "three routes": ([0, 3, 300, 9000, 1], 3),
}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(QUANTILE_CASES))
def test_group_quantiles_equal_one_handle_per_group(case, mode):
    need_gpu()
    sizes, E = QUANTILE_CASES[case]
    o = offsets(sizes)
    x = catalogue(sizes, E, seed=len(case))
    with state_handle(x, mode, trajectory_every=1, trajectory_capacity=1, trajectory_full=True) as ex:
        ungrouped = ex.state_quantiles(LEVELS)
        ex.set_world_groups(sizes)
        st, n = _launches(ex, lambda: ex.state_group_quantiles(LEVELS))
        assert n == quantile_group_launches(sizes, E)
        assert np.array_equal(ex.state_quantiles(LEVELS), ungrouped, equal_nan=True)  # groups change no ungrouped table
        ex.step(1)
        tr = ex.trajectory_group_quantiles(LEVELS)
        traj = ex.trajectory()
    assert st.shape == (len(sizes), E, 25, len(LEVELS)) and tr.shape == (1, len(sizes), E, 25, len(LEVELS))
    for g, n in enumerate(sizes):
        v = x[o[g]:o[g + 1]]
        assert np.array_equal(st[g], ref_quantiles(v, LEVELS), equal_nan=True), (g, n)  # bit for bit, +-0 included
        assert st[g].tobytes() == ref_quantiles(v, LEVELS).tobytes(), (g, n)
        for e in range(E):
            for i in range(25):
                assert np.array_equal(st[g, e, i], numpy_quantiles(v[:, e, i], LEVELS), equal_nan=True), (g, e, i)
        if n == 0:
            assert np.all(np.isnan(st[g])) and np.all(np.isnan(tr[:, g]))
            continue
        with state_handle(np.ascontiguousarray(v), mode, trajectory_every=1, trajectory_capacity=1,
                          trajectory_full=True) as one:
            assert st[g].tobytes() == one.state_quantiles(LEVELS).tobytes(), (g, n)
            one.step(1)
            assert np.array_equal(one.trajectory(), traj[:, o[g]:o[g + 1]], equal_nan=True)  # the same samples
            assert tr[:, g].tobytes() == one.trajectory_quantiles(LEVELS).tobytes(), (g, n)


@pytest.mark.gpu
def test_1024_quantile_groups():
    need_gpu()
    rng = np.random.default_rng(7)
    sizes = [int(s) if rng.random() > 0.1 else 0 for s in rng.integers(0, 40, 1024)]
    sizes[0], sizes[500], sizes[1023] = 0, 9000, 0  # empty first and last groups, one radix group among them
    o, E = offsets(sizes), 1
    x = catalogue(sizes, E, seed=8)
    with state_handle(x, "exact") as ex:
        ex.set_world_groups(sizes)
        st, n = _launches(ex, lambda: ex.state_group_quantiles(LEVELS[:3]))
        reads = ex.quantile_reads()
    assert n == quantile_group_launches(sizes, E) == 1 + 18
    assert 1.0 < reads < 1.5  # one read per small triple, 3 to 8 for the radix group's 25
    for g in range(1024):
        assert st[g].tobytes() == ref_quantiles(x[o[g]:o[g + 1]], LEVELS[:3]).tobytes(), g


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_radix_triples_in_two_slices(mode):
    """E = 30: a slice holds 45 (group, plane) rows, so the two radix groups' 50 rows run in two slices."""
    need_gpu()
    sizes, E = [5, 8193, 9000], 30
    o = offsets(sizes)
    x = catalogue(sizes, E, seed=9)
    with state_handle(x, mode) as ex:
        ex.set_world_groups(sizes)
        st, n = _launches(ex, lambda: ex.state_group_quantiles(LEVELS))
    assert n == quantile_group_launches(sizes, E) == 1 + 2 * 18
    for g in range(3):
        v = np.ascontiguousarray(x[o[g]:o[g + 1]])
        assert st[g].tobytes() == ref_quantiles(v, LEVELS).tobytes(), g
        with state_handle(v, mode) as one:
            assert st[g].tobytes() == one.state_quantiles(LEVELS).tobytes(), g


# --------------------------------------------------------------------------- GPU: covariance

SELECTIONS = {1: (6,), 3: (4, 5, 6), 6: (0, 4, 5, 6, 10, 11), 25: (24,) + tuple(range(24))}
COV_CASES = {
    "chunk edges": ([0, 63, 64, 65, 0], 1),
    "saturation": ([528 * 64 - 1, 528 * 64, 528 * 64 + 1], 1),
    "E=32": ([0, 100, 5000], 32),
    "E=33": ([7, 0, 5000], 33),
}


def cov_states(sizes, E, seed):
    """x [M, E, 25]: normal draws per group around a group offset, with NaN / inf in a few values (listwise deletion
    inside a group) and one group at an orbital offset."""
    rng = np.random.default_rng(seed)
    M = int(sum(sizes))
    x = rng.normal(size=(M, E, 25)) * rng.uniform(0.5, 3.0, (M, 1, 1))
    x += np.repeat(np.arange(len(sizes), dtype=float) * 10.0, sizes)[:, None, None]
    x[rng.random((M, E, 25)) < 0.01] = np.nan
    x[rng.random((M, E, 25)) < 0.003] = -np.inf
    o = offsets(sizes)
    g = int(np.argmax(sizes))
    x[o[g]:o[g + 1], :, 4:7] += 6.9e6
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(COV_CASES))
def test_group_covariance_equal_one_handle_per_group(case, mode):
    need_gpu()
    sizes, E = COV_CASES[case]
    o = offsets(sizes)
    x = cov_states(sizes, E, seed=len(case))
    tabs, trs = {}, {}
    with state_handle(x, mode, trajectory_every=1, trajectory_capacity=1, trajectory_full=True) as ex:
        ungrouped = {p: ex.state_covariance(sel) for p, sel in SELECTIONS.items()}
        ex.set_world_groups(sizes)
        for p, sel in SELECTIONS.items():
            tabs[p], n = _launches(ex, lambda: ex.state_group_covariance(sel))
            assert n == cov_group_launches(sizes, E, p), p
            assert np.array_equal(ex.state_covariance(sel), ungrouped[p], equal_nan=True)
        perm = ex.state_group_covariance(SELECTIONS[3][::-1])
        ex.step(1)
        trs = {p: ex.trajectory_group_covariance(sel) for p, sel in SELECTIONS.items()}
    for p, t in tabs.items():
        assert t.shape == (len(sizes), E, 1 + p + p * p)
    # permuting the selection permutes every group's table bit for bit
    M3 = tabs[3][..., 4:].reshape(len(sizes), E, 3, 3)
    Mp = perm[..., 4:].reshape(len(sizes), E, 3, 3)
    assert Mp.tobytes() == M3[..., ::-1, ::-1].copy().tobytes()
    assert perm[..., :1].tobytes() == tabs[3][..., :1].tobytes()
    assert perm[..., 1:4].tobytes() == tabs[3][..., 1:4][..., ::-1].copy().tobytes()
    for g, n in enumerate(sizes):
        v = x[o[g]:o[g + 1]]
        for p, sel in SELECTIONS.items():
            if n == 0:
                assert np.all(tabs[p][g, :, 0] == 0) and np.all(np.isnan(tabs[p][g, :, 1:]))
                assert np.all(trs[p][:, g, :, 0] == 0) and np.all(np.isnan(trs[p][:, g, :, 1:]))
            elif p <= 6 and n * E <= 200_000:
                check_table(tabs[p][g], ref_table(v, sel), scales(v, sel), f"group {g}, p = {p}")
        if n == 0:
            continue
        with state_handle(np.ascontiguousarray(v), mode, trajectory_every=1, trajectory_capacity=1,
                          trajectory_full=True) as one:
            for p, sel in SELECTIONS.items():
                assert tabs[p][g].tobytes() == one.state_covariance(sel).tobytes(), (g, p)
            one.step(1)
            for p, sel in SELECTIONS.items():
                assert trs[p][:, g].tobytes() == one.trajectory_covariance(sel).tobytes(), (g, p)


@pytest.mark.gpu
def test_covariance_groups_in_two_slices():
    """100 groups of 33 792 worlds at p = 25: each group has 528 chunks, 2.75 MB of partials, so the call runs as a slice
    of 97 groups and one of 3; each group equals the call where it is one group of three (one slice)."""
    need_gpu()
    G, n = 100, 528 * 64
    sizes = [n] * G
    rng = np.random.default_rng(21)
    x = rng.normal(size=(G * n, 1, 25))
    x += np.repeat(np.arange(G, dtype=float), n)[:, None, None]
    x[rng.random(x.shape) < 1e-3] = np.nan
    sel = SELECTIONS[25]
    with state_handle(x, "exact") as ex:
        ex.set_world_groups(sizes)
        got, launches = _launches(ex, lambda: ex.state_group_covariance(sel))
        assert launches == cov_group_launches(sizes, 1, 25) == 4
        for g in (0, 1, 96, 97, 99):
            ex.set_world_groups([g * n, n, (G - 1 - g) * n])  # the group in the middle (after an empty one for g = 0)
            one, launches = _launches(ex, lambda: ex.state_group_covariance(sel))
            assert launches == 2
            assert got[g].tobytes() == one[1].tobytes(), g


# --------------------------------------------------------------------------- GPU: invariants and refusals


@pytest.mark.gpu
@pytest.mark.parametrize("M", [200, 5000, 20000])
def test_one_group_is_the_ungrouped_table(M):
    need_gpu()
    x = cov_states([M], 2, seed=M)
    with state_handle(x, "exact", trajectory_every=1, trajectory_capacity=2, trajectory_full=True) as ex:
        ex.step(2)
        ex.set_world_groups([M])
        for ring in (False, True):
            kind = "trajectory" if ring else "state"
            a = getattr(ex, f"{kind}_quantiles")(LEVELS)
            b = getattr(ex, f"{kind}_group_quantiles")(LEVELS)
            assert b.tobytes() == (a[:, None] if ring else a[None]).tobytes()
            for sel in SELECTIONS.values():
                a = getattr(ex, f"{kind}_covariance")(sel)
                b = getattr(ex, f"{kind}_group_covariance")(sel)
                assert b.tobytes() == (a[:, None] if ring else a[None]).tobytes()


@pytest.mark.gpu
def test_grouped_entries_refuse_in_the_documented_order():
    need_gpu()
    x = cov_states([3000], 2, seed=10)
    dp, u32p = ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_uint32)
    lv = np.array(LEVELS[:3])
    sel = np.array([4, 5, 6], dtype=np.uint32)
    buf = np.empty(10 ** 6)
    with state_handle(x, "exact") as ex:
        L, h = ex._L, ex._h
        q_fns = (L.b200_sixdof_state_group_quantiles, L.b200_sixdof_trajectory_group_quantiles)
        c_fns = (L.b200_sixdof_state_group_covariance, L.b200_sixdof_trajectory_group_covariance)
        for fn in q_fns:
            assert fn(None, lv.ctypes.data_as(dp), 3, buf.ctypes.data, 8) == _lib.ERR_INVALID_ARGUMENT
            # no groups set: refused before the levels and the size
            assert fn(h, lv.ctypes.data_as(dp), 0, buf.ctypes.data, 8) == _lib.ERR_INVALID_ARGUMENT
            assert b"set_world_groups" in _lib.lib().b200_last_error()
        for fn in c_fns:
            assert fn(None, sel.ctypes.data_as(u32p), 3, buf.ctypes.data, 8) == _lib.ERR_INVALID_ARGUMENT
            assert fn(h, sel.ctypes.data_as(u32p), 0, buf.ctypes.data, 8) == _lib.ERR_INVALID_ARGUMENT
            assert b"set_world_groups" in _lib.lib().b200_last_error()
        ex.set_world_groups([1000, 0, 2000])
        want_q = 3 * 2 * 25 * 3 * 8
        fn = L.b200_sixdof_state_group_quantiles
        assert fn(h, lv.ctypes.data_as(dp), 0, buf.ctypes.data, want_q + 8) == _lib.ERR_INVALID_ARGUMENT  # levels first
        bad = np.array([0.5, 1.5, 0.1])
        assert fn(h, bad.ctypes.data_as(dp), 3, buf.ctypes.data, want_q) == _lib.ERR_INVALID_ARGUMENT
        assert fn(h, lv.ctypes.data_as(dp), 3, buf.ctypes.data, want_q - 8) == _lib.ERR_VALUE_SIZE_MISMATCH
        assert fn(h, lv.ctypes.data_as(dp), 3, buf.ctypes.data, want_q) == _lib.OK
        want_c = 3 * 2 * 13 * 8
        fn = L.b200_sixdof_state_group_covariance
        dup = np.array([4, 4, 6], dtype=np.uint32)
        assert fn(h, dup.ctypes.data_as(u32p), 3, buf.ctypes.data, want_c + 8) == _lib.ERR_INVALID_ARGUMENT
        assert fn(h, sel.ctypes.data_as(u32p), 3, buf.ctypes.data, want_c - 8) == _lib.ERR_VALUE_SIZE_MISMATCH
        assert fn(h, sel.ctypes.data_as(u32p), 3, buf.ctypes.data, want_c) == _lib.OK
        # the trajectory entries take the ring's width: no ring, no plane
        fn = L.b200_sixdof_trajectory_group_covariance
        assert fn(h, sel.ctypes.data_as(u32p), 3, buf.ctypes.data, 0) == _lib.ERR_INVALID_ARGUMENT


# --------------------------------------------------------------------------- GPU: Exec


def _group_params(params, a, b):
    return {k: np.ascontiguousarray(v[a:b]) for k, v in params.items()}


COV_SPEC = [("world_pos", (4, 5, 6)), ("world_vel", (3, 4, 5))]
Q = (0.01, 0.5, 0.99)


@pytest.mark.gpu
@pytest.mark.parametrize("host_cb", [False, True])
def test_exec_grouped_quantiles_and_covariance_equal_one_exec_per_group(host_cb):
    need_gpu()
    M, sizes = 4096, [1000, 0, 2500, 596]
    o = offsets(sizes)
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=12.0, math="exact", ensemble=True, quantiles=Q, covariance=COV_SPEC)
    post = (lambda tick, ctx: None) if host_cb else None
    ex = w.build(sys_, n_worlds=M, world_params=params, groups=sizes, **kw)
    ex.run(50, post_step=post)
    plain = w.build(sys_, n_worlds=M, world_params=params, **kw)
    plain.run(50, post_step=post)
    for pair in ("rocket.world_pos", "ball.world_vel"):
        assert np.array_equal(ex.quantiles(pair), plain.quantiles(pair), equal_nan=True)
    for ent in ("rocket", "ball"):
        a, b = ex.covariance(ent), plain.covariance(ent)
        for k in ("count", "mean", "cov"):
            assert np.array_equal(a[k], b[k], equal_nan=True), (ent, k)
    for g, n in enumerate(sizes):
        got_q = ex.quantiles("rocket.world_pos", groups=True)
        assert got_q.shape == (6, len(sizes), len(Q), 7)
        got_c = ex.covariance("rocket", groups=True)
        assert got_c["count"].shape == (6, len(sizes)) and got_c["cov"].shape == (6, len(sizes), 6, 6)
        if n == 0:
            assert np.all(np.isnan(got_q[:, g])) and np.all(got_c["count"][:, g] == 0)
            continue
        one = w.build(sys_, n_worlds=n, world_params=_group_params(params, o[g], o[g + 1]), **kw)
        one.run(50, post_step=post)
        for pair in ("rocket.world_pos", "ball.world_vel", "rocket.force"):
            assert ex.quantiles(pair, groups=True)[:, g].tobytes() == one.quantiles(pair).tobytes(), (g, pair)
        for ent in ("rocket", "ball"):
            got, want = ex.covariance(ent, groups=True), one.covariance(ent)
            assert got["planes"] == want["planes"]
            for k in ("count", "mean", "cov"):
                assert np.array_equal(got[k][:, g], want[k], equal_nan=True), (g, ent, k)
    with pytest.raises(_lib.B200Error, match="groups"):
        plain.quantiles("rocket.world_pos", groups=True)
    with pytest.raises(_lib.B200Error, match="groups"):
        plain.covariance("rocket", groups=True)


# --------------------------------------------------------------------------- GPU: two gloo ranks

GLOO_SIZES, GLOO_M = [3000, 0, 9000, 4000, 4001], 20_001  # the shard boundary at 10 001 splits group 2


def _sharded_worker(rank, ws):
    w0, w1 = shard_worlds(GLOO_M, rank, ws)
    x = cov_states(GLOO_SIZES, 2, seed=12)[w0:w1]
    from elodin_b200.sharding import gather_covariance

    with state_handle(np.ascontiguousarray(x), "exact") as ex:
        ex.set_world_groups(shard_groups(GLOO_SIZES, rank, ws))
        return gather_covariance(ex.state_group_covariance(SELECTIONS[6])), ex.state_group_quantiles(LEVELS)


@pytest.mark.gpu
def test_two_gloo_ranks_merge_grouped_covariance_and_keep_quantiles_per_rank():
    need_gpu()
    sizes, M = GLOO_SIZES, GLOO_M
    sel = SELECTIONS[6]
    got = run_gloo(_sharded_worker, 2)
    x = cov_states(sizes, 2, seed=12)
    o = offsets(sizes)
    with state_handle(x, "exact") as ex:
        ex.set_world_groups(sizes)
        want = ex.state_group_covariance(sel)
    for rank, (cov, quant) in enumerate(got):
        assert cov.tobytes() == got[0][0].tobytes()  # every rank the same bits
        for g in (0, 1, 3, 4):  # held by one rank: the other's n = 0 is the identity of the merge
            assert cov[g].tobytes() == want[g].tobytes(), g
        v = x[o[2]:o[3]]
        check_table(cov[2], ref_table(v, sel), scales(v, sel), "split group")
        w0, w1 = shard_worlds(M, rank, 2)
        local = offsets(shard_groups(sizes, rank, 2)) + w0
        for g in range(len(sizes)):
            assert quant[g].tobytes() == ref_quantiles(x[local[g]:local[g + 1]], LEVELS).tobytes(), (rank, g)
