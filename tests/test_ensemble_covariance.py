"""Ensemble covariance over the world axis (b200_sixdof_trajectory_covariance / _state_covariance /
b200_covariance_merge, Exec.covariance) against an exact reference over the complete worlds (every selected value
finite): mean = math.fsum(x) / n and M_ab = fsum((x_a - mean_a)(x_b - mean_b)).

Bounds, with C = M / n, sigma = the reference's sqrt(C_aa) and s = max|x| over the complete worlds: count equal, mean
within 1e-13 s, |C_ab - C_ref_ab| <= 1e-8 sigma_a sigma_b + 32 eps (s_a sigma_b + sigma_a s_b).
test_bounds_are_sensitive shows the one-pass sum(xy) - sum(x) sum(y) / n formula violates the bound on |mean| / sigma
= 1e6 data with correlation 0.9, where the library keeps it."""

import ctypes
import math

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from tests.ensemble_util import (FREE, ROCKET, handle, need_gpu, no_device, rocket_world, run_gloo,  # noqa: F401
                                 sampled_state, split, two_body_world)

EPS = np.finfo(np.float64).eps
NAN = float("nan")


# --------------------------------------------------------------------------- reference and bounds


def ref_record(X):
    """X [worlds, p] -> the record (n, mean[p], M[p][p]) over the rows whose p values are all finite."""
    X = np.asarray(X, dtype=np.float64)
    p = X.shape[1]
    Y = X[np.isfinite(X).all(1)]
    n = Y.shape[0]
    if n == 0:
        return np.concatenate([[0.0], np.full(p + p * p, NAN)])
    mean = np.array([math.fsum(Y[:, a].tolist()) / n for a in range(p)])
    D = Y - mean
    M = np.empty((p, p))
    for a in range(p):
        for b in range(a, p):
            M[a, b] = M[b, a] = math.fsum((D[:, a] * D[:, b]).tolist())
    return np.concatenate([[float(n)], mean, M.ravel()])


def ref_table(x, planes):
    """x [worlds, ..., 25 or 13] -> [..., 1 + p + p*p] over the selected planes."""
    x = np.asarray(x, dtype=np.float64)[..., list(planes)]
    flat = x.reshape(x.shape[0], -1, x.shape[-1])
    out = np.array([ref_record(flat[:, g]) for g in range(flat.shape[1])])
    return out.reshape(x.shape[1:-1] + (out.shape[-1],))


def scales(x, planes):
    """max|x_a| over the complete worlds of each group: x [worlds, ..., W] -> [..., p]."""
    x = np.asarray(x, dtype=np.float64)[..., list(planes)]
    ok = np.isfinite(x).all(-1, keepdims=True)
    return np.max(np.where(ok, np.abs(x), 0.0), axis=0)


def check_table(got, want, s, what=""):
    """got / want [..., 1 + p + p*p], s [..., p]."""
    assert got.shape == want.shape, what
    p = s.shape[-1]
    g, w, s = got.reshape(-1, got.shape[-1]), want.reshape(-1, want.shape[-1]), s.reshape(-1, p)
    assert np.array_equal(g[:, 0], w[:, 0]), f"{what}: counts differ"
    empty = w[:, 0] == 0
    assert np.all(np.isnan(g[empty][:, 1:])), f"{what}: a group without complete worlds is not NaN"
    g, w, s = g[~empty], w[~empty], s[~empty]
    mean_err = np.abs(g[:, 1:1 + p] - w[:, 1:1 + p])
    assert np.all(mean_err <= 1e-13 * s), f"{what}: mean off by {np.max(mean_err / np.maximum(s, 1e-300)):.3e} max|x|"
    n = w[:, :1, None]
    cg, cw = g[:, 1 + p:].reshape(-1, p, p) / n, w[:, 1 + p:].reshape(-1, p, p) / n
    sig = np.sqrt(np.maximum(np.diagonal(cw, axis1=1, axis2=2), 0.0))
    bound = 1e-8 * sig[:, :, None] * sig[:, None, :] + 32 * EPS * (s[:, :, None] * sig[:, None, :] + sig[:, :, None] * s[:, None, :])
    err = np.abs(cg - cw)
    assert np.all(err <= bound), f"{what}: covariance off by {np.max(err / np.maximum(bound, 1e-300)):.3g} x the bound"


def symmetric_bits(t, p):
    M = t[..., 1 + p:].reshape(t.shape[:-1] + (p, p))
    return M.tobytes() == np.swapaxes(M, -1, -2).copy().tobytes()


def _empty(groups, p):
    return np.tile(np.concatenate([[0.0], np.full(p + p * p, NAN)]), (groups, 1))


# --------------------------------------------------------------------------- CPU: b200_covariance_merge


@pytest.mark.parametrize("seed", range(4))
def test_merge_matches_exact_sums(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2_000, 40_001))
    k = int(rng.integers(2, 12))
    p = 4
    z = rng.normal(size=(n, 2, p))
    x = np.empty((n, 2, p))
    x[:, 0] = 3.0 + z[:, 0] @ np.array([[2.0, 0, 0, 0], [1.0, 1.0, 0, 0], [0, 0.5, 3.0, 0], [0, 0, -1.0, 0.1]])
    x[:, 1] = 7.0e5 + rng.exponential(1.0, (n, p)) * [1.0, 1e3, 1e-3, 5.0]
    parts = split(rng, n, k)
    parts.insert(1, parts[0][:0])                                       # an empty part in the middle
    tables = [ref_table(x[idx], range(p)) if len(idx) else _empty(2, p) for idx in parts]
    got = el.merge_covariance(tables)
    check_table(got, ref_table(x, range(p)), scales(x, range(p)), f"{k} parts")
    assert symmetric_bits(got, p)
    assert got.tobytes() == el.merge_covariance(tables).tobytes()


def test_reference_equals_numpy():
    rng = np.random.default_rng(2)
    x = rng.normal(size=(500, 5)) @ rng.normal(size=(5, 5))
    x[[3, 40], 2] = [np.nan, np.inf]
    r = ref_record(x)
    y = x[np.isfinite(x).all(1)]
    assert r[0] == 498
    np.testing.assert_allclose(r[6:].reshape(5, 5) / r[0], np.cov(y.T, ddof=0), rtol=1e-12, atol=1e-12)


def test_bounds_are_sensitive():
    """|mean| / sigma = 1e6 with correlation 0.9: the merge keeps the bound, the one-pass sum(xy) - sum(x) sum(y) / n
    misses it on the same data."""
    rng = np.random.default_rng(7)
    n = 200_000
    z = rng.normal(size=(n, 2))
    x = np.stack([6.4e6 + 6.4 * z[:, 0], -6.4e6 + 6.4 * (0.9 * z[:, 0] + math.sqrt(1 - 0.81) * z[:, 1])], 1)
    assert 0.9e6 <= abs(np.mean(x[:, 0])) / np.std(x[:, 0]) <= 1.1e6 and abs(np.corrcoef(x.T)[0, 1] - 0.9) < 0.01
    parts = split(rng, n, 9)
    want = ref_table(x, (0, 1))
    got = el.merge_covariance([ref_table(x[idx], (0, 1)) for idx in parts])
    check_table(got, want, scales(x, (0, 1)), "merge")
    naive = want.copy()
    for a in range(2):
        for b in range(2):
            naive[3 + 2 * a + b] = np.sum(x[:, a] * x[:, b]) - np.sum(x[:, a]) * np.sum(x[:, b]) / n
    with pytest.raises(AssertionError, match="covariance off"):
        check_table(naive, want, scales(x, (0, 1)), "one-pass")


def test_non_finite_rows_are_dropped_listwise():
    rng = np.random.default_rng(3)
    x = rng.normal(0.0, 1.0, (1000, 3, 4))
    x[[3, 17, 500], 0, [0, 1, 3]] = [np.nan, np.inf, -np.inf]          # one bad value per row: the whole row goes
    x[:, 1, 2] = np.nan                                                 # no complete world in group 1
    x[::2, 2, 0] = np.inf
    parts = split(rng, 1000, 5)
    tables = [ref_table(x[idx], range(4)) if len(idx) else _empty(3, 4) for idx in parts]
    got = el.merge_covariance(tables)
    assert list(got[:, 0]) == [997.0, 0.0, 500.0]
    assert np.all(np.isnan(got[1, 1:]))
    check_table(got, ref_table(x, range(4)), scales(x, range(4)), "listwise")
    # planes 1..3 of group 2 exclude nothing: the inf of plane 0 is not selected
    assert ref_table(x[:, 2:3], (1, 2, 3))[0, 0] == 1000.0


def test_merge_refusals():
    with pytest.raises(_lib.B200ValueError):
        el.merge_covariance([np.zeros((3, 7)), np.zeros((4, 7))])        # shapes differ
    for bad in (5, 8, 2, 1):                                            # not 1 + p + p*p
        with pytest.raises(_lib.B200ValueError):
            el.merge_covariance([np.zeros((2, bad))])
    with pytest.raises(_lib.B200ValueError):
        el.merge_covariance([])
    for count in (-1.0, NAN):
        t = np.zeros((2, 7))
        t[1, 0] = count
        with pytest.raises(_lib.B200Error) as e:
            el.merge_covariance([np.zeros((2, 7)), t])
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    with pytest.raises(_lib.B200Error) as e:                            # p = 26
        el.merge_covariance([np.zeros((1, 1 + 26 + 26 * 26))])
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    assert el.merge_covariance([np.zeros((1, 3))]).shape == (1, 3)      # p = 1


def _rank_table(rank):
    rng = np.random.default_rng(100 + rank)
    x = 1.0e4 * (rank + 1) + rng.normal(0.0, 3.0, (300 + 37 * rank, 4, 3))
    return ref_table(x, (2, 0, 1))


def _gather_worker(rank, ws):
    from elodin_b200.sharding import gather_covariance

    return gather_covariance(_rank_table(rank))


def test_gather_covariance_two_gloo_ranks():
    ws = 2
    got = run_gloo(_gather_worker, ws)
    want = el.merge_covariance([_rank_table(r) for r in range(ws)])
    assert got[0].shape == (4, 13)
    assert got[0].tobytes() == want.tobytes() and got[1].tobytes() == want.tobytes()


def test_build_validates_covariance_before_the_device(no_device):
    w, sys_ = two_body_world(), el.six_dof()
    for bad in (["world_pos"], ["inertia"], []):                         # the mode is checked before the selection
        with pytest.raises(_lib.B200Error, match="ensemble=True") as e:
            w.build(sys_, covariance=bad)
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    with pytest.raises(_lib.B200ValueError, match="inertia"):
        w.build(sys_, ensemble=True, covariance=["inertia"])
    with pytest.raises(ValueError, match="twice"):
        w.build(sys_, ensemble=True, covariance=["world_pos", ("world_pos", (4,))])
    with pytest.raises(ValueError, match="twice"):
        w.build(sys_, ensemble=True, covariance=[("world_vel", (3, 3))])
    for idx in ((7,), (-1,), (1.0,), (True,)):
        with pytest.raises(ValueError, match="index"):
            w.build(sys_, ensemble=True, covariance=[("world_pos", idx)])
    with pytest.raises(ValueError, match="1 to 25"):
        w.build(sys_, ensemble=True, covariance=[])
    for bad in ("world_pos", [3], [("world_pos",)], [("world_pos", (1,), 2)]):
        with pytest.raises(TypeError):
            w.build(sys_, ensemble=True, covariance=bad)
    with pytest.raises(AssertionError, match="handle is created"):  # all 25 planes
        w.build(sys_, ensemble=True, covariance=["world_pos", "world_vel", "world_accel", "force"])
    with pytest.raises(AssertionError, match="handle is created"):
        w.build(sys_, ensemble=True, covariance=[("world_pos", (6, 4, 5)), ("force", [np.int64(0)])])


def test_covariance_symbols_are_exported():
    L = _lib.lib()
    for name in ("b200_sixdof_trajectory_covariance", "b200_sixdof_state_covariance", "b200_covariance_merge"):
        assert name in _lib.SYMBOLS and hasattr(L, name)
    assert _lib.MAX_COV_PLANES == 25


# --------------------------------------------------------------------------- GPU


SHAPES = [(1, 1), (7, 3), ((1 << 16) + 3, 1), (5, 1024), (100, 300)]
ALL = tuple(range(25))
SELECTIONS = {1: (6,), 3: (4, 5, 6), 13: tuple(range(12, -1, -1)), 25: (24,) + tuple(range(24))}


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("kind", [FREE, ROCKET])
@pytest.mark.parametrize("width", [13, 25])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_trajectory_covariance_matches_the_ring(shape, width, kind, math_mode):
    need_gpu()
    M, N = shape
    with handle(kind, M, N, math_mode, width=width, capacity=2)[0] as ex:
        ex.step(2)
        traj = np.moveaxis(ex.trajectory(), 1, 0)                       # [M, S, N, W]
        for p, sel in SELECTIONS.items():
            if max(sel) >= width:
                continue
            n0 = ex.timings()["kernel_launches"]
            got = ex.trajectory_covariance(sel)
            assert ex.timings()["kernel_launches"] > n0                 # the reduction runs in this library's kernels
            assert got.shape == (2, N, 1 + p + p * p)
            check_table(got, ref_table(traj, sel), scales(traj, sel), f"{shape} {kind} {math_mode} W={width} p={p}")
            assert symmetric_bits(got, p)
            assert got.tobytes() == ex.trajectory_covariance(sel).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(7, 3), ((1 << 16) + 3, 1), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_diagonal_matches_the_statistics_and_permutations_permute_bits(shape):
    need_gpu()
    M, N = shape
    with handle(ROCKET, M, N, "fast", capacity=1)[0] as ex:
        ex.step(2)
        full = ex.state_covariance(ALL)
        stats = ex.state_stats()                                        # [N, 25, 5], every world finite
        state = sampled_state(ex)
        rng = np.random.default_rng(5)
        perm = rng.permutation(25)
        permuted = ex.state_covariance(perm)
        sub = (17, 4, 9)
        subset = ex.state_covariance(sub)
    check_table(full, ref_table(state, ALL), scales(state, ALL), f"state {shape}")
    assert np.array_equal(full[:, 0], stats[:, 0, 0])
    Mf = full[:, 26:].reshape(N, 25, 25)
    m2 = stats[..., 2]
    sig2 = m2 / M
    s = scales(state, ALL)
    err = np.abs(np.diagonal(Mf, axis1=1, axis2=2) / M - sig2)
    assert np.all(err <= 1e-8 * sig2 + 64 * EPS * s * np.sqrt(sig2))
    # permutation and subset invariance, bit for bit
    assert permuted[:, 1:26].tobytes() == full[:, 1:26][:, perm].tobytes()
    assert permuted[:, 26:].reshape(N, 25, 25).tobytes() == Mf[:, perm][:, :, perm].tobytes()
    assert subset[:, 1:4].tobytes() == full[:, 1:26][:, list(sub)].tobytes()
    assert subset[:, 4:].reshape(N, 3, 3).tobytes() == Mf[:, list(sub)][:, :, list(sub)].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("shape", [(7, 3), ((1 << 16) + 3, 1), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_non_finite_worlds_are_dropped_listwise(shape, math_mode):
    need_gpu()
    from tests.util import near_world

    M, N = shape
    pos, vel, ine, cols, dt = near_world(2, M, N)
    pos[1, 0, 4] = np.nan                                               # selected
    vel[M // 2, N - 1, 3] = np.inf                                      # selected
    pos[M - 2, 0, 5] = -np.inf                                          # selected
    pos[M - 1, 0, 0] = np.nan                                           # not selected: excludes nothing
    sel = (4, 5, 6, 10)
    with handle(FREE, M, N, math_mode, capacity=1, state=(pos, vel, ine, cols, dt))[0] as ex:
        got = ex.state_covariance(sel)
        state = sampled_state(ex)
        sub = ex.state_covariance((6, 11))                              # the bad worlds are in neither plane
    if N == 1:
        assert got[0, 0] == M - 3
    else:
        assert got[0, 0] == M - 2 and got[N - 1, 0] == M - 1
    assert np.all(sub[:, 0] == M)
    check_table(got, ref_table(state, sel), scales(state, sel), f"{shape} listwise")
    check_table(sub, ref_table(state, (6, 11)), scales(state, (6, 11)), f"{shape} unselected")
    with handle(FREE, M, N, math_mode, capacity=1,
                 state=(np.full_like(pos, np.nan), vel, ine, cols, dt))[0] as ex:
        empty = ex.state_covariance((4, 10))
    assert np.all(empty[:, 0] == 0) and np.all(np.isnan(empty[:, 1:]))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [((1 << 16) + 3, 1), (7, 3), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_orbital_offsets_keep_the_bound(shape):
    """|mean| / sigma = 1e6 with correlation 0.9 between x and y, where sum(xy) - sum(x) sum(y) / n breaks the bound."""
    need_gpu()
    from tests.util import near_world

    M, N = shape
    rng = np.random.default_rng(11)
    pos, vel, ine, cols, dt = near_world(5, M, N)
    z = rng.normal(size=(M, N, 3))
    pos[..., 4] = 6.4e6 + 6.4 * z[..., 0]
    pos[..., 5] = -3.1e6 + 6.4 * (0.9 * z[..., 0] + math.sqrt(0.19) * z[..., 1])
    pos[..., 6] = 2.2e6 + 6.4 * z[..., 2]
    vel[..., 3:] = 7.6e3 + rng.normal(0.0, 7.6e-3, (M, N, 3))
    sel = (4, 5, 6, 10, 11, 12)
    with handle(FREE, M, N, "fast", capacity=1, state=(pos, vel, ine, cols, dt))[0] as ex:
        got = ex.state_covariance(sel)
        state = sampled_state(ex)
    want = ref_table(state, sel)
    check_table(got, want, scales(state, sel), f"orbital {shape}")
    if M > 1000:
        x = state[:, 0, [4, 5]]
        naive = want[:1].copy()
        naive[0, 1 + 6 + 1] = np.sum(x[:, 0] * x[:, 1]) - np.sum(x[:, 0]) * np.sum(x[:, 1]) / M
        naive[0, 1 + 6 + 6] = naive[0, 1 + 6 + 1]
        with pytest.raises(AssertionError, match="covariance off"):
            check_table(naive, want[:1], scales(state, sel)[:1], "one-pass")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(7, 3), ((1 << 16) + 3, 1), (5, 1024), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_a_sample_has_the_same_bits_in_any_ring(shape):
    """At (1<<16)+3 x 1 the 128-sample call at p = 25 needs two scratch slices (a slice holds 98 groups there)."""
    need_gpu()
    M, N = shape
    S = 128 if M > 1000 and N == 1 else 64
    big, state = handle(ROCKET, M, N, "fast", capacity=S)
    one, _ = handle(ROCKET, M, N, "fast", capacity=1, state=state)
    sel = SELECTIONS[25]
    with big, one:
        big.step(S)
        n0 = big.timings()["kernel_launches"]
        many = big.trajectory_covariance(sel)
        launches = big.timings()["kernel_launches"] - n0
        if M == (1 << 16) + 3:
            assert launches == 4                                        # two slices, each a chunk and a merge launch
        assert many.tobytes() == big.trajectory_covariance(sel).tobytes()
        traj = np.moveaxis(big.trajectory(), 1, 0)
        for s in range(S):
            one.trajectory_reset()
            one.step(1)
            single = one.trajectory_covariance(sel)
            assert single.shape[0] == 1
            assert single[0].tobytes() == many[s].tobytes(), f"sample {s}"
    for s in (0, S // 2, S - 1):
        check_table(many[s], ref_table(traj[:, s], sel), scales(traj[:, s], sel), f"sample {s}")


@pytest.mark.gpu
def test_refusals_and_device_destinations():
    need_gpu()
    import torch

    L = _lib.lib()
    M, N = 20000, 2
    up = ctypes.POINTER(ctypes.c_uint32)
    with handle(ROCKET, M, N, "exact", width=13, capacity=2)[0] as ex:
        ex.step(2)
        good = ex.trajectory_covariance((4, 5, 6, 10))
        for sel in ([], list(range(14)), [4, 5, 4], [13], [24]):        # a 13-plane ring has no accel / force
            a = np.array(sel if sel else [0], dtype=np.uint32)
            rc = L.b200_sixdof_trajectory_covariance(ex._h, a.ctypes.data_as(up), len(sel), good.ctypes.data, 0)
            assert rc == _lib.ERR_INVALID_ARGUMENT, sel
        assert L.b200_sixdof_state_covariance(ex._h, np.array([25], dtype=np.uint32).ctypes.data_as(up), 1,
                                              good.ctypes.data, 0) == _lib.ERR_INVALID_ARGUMENT
        a = np.array(list(range(25)) + [0], dtype=np.uint32)
        assert L.b200_sixdof_state_covariance(ex._h, a.ctypes.data_as(up), 26, good.ctypes.data, 0) == _lib.ERR_INVALID_ARGUMENT
        a = np.array([4, 5, 6, 10], dtype=np.uint32)
        for wrong in (good.nbytes - 8, good.nbytes + 8, 0):
            assert L.b200_sixdof_trajectory_covariance(ex._h, a.ctypes.data_as(up), 4, good.ctypes.data, wrong) \
                == _lib.ERR_VALUE_SIZE_MISMATCH
        assert ex.state_covariance(list(range(25))).shape == (N, 651)   # the state has every plane
        assert L.b200_sixdof_status(ex._h) == 0
        assert ex.trajectory_covariance((4, 5, 6, 10)).tobytes() == good.tobytes()
        dev = torch.empty(good.shape, dtype=torch.float64, device="cuda")
        ex.trajectory_covariance((4, 5, 6, 10), out_ptr=dev.data_ptr())
        assert dev.cpu().numpy().tobytes() == good.tobytes()
        ex.trajectory_reset()                                           # an empty ring: bytes = 0, no launch
        n0 = ex.timings()["kernel_launches"]
        assert ex.trajectory_covariance((4,)).shape == (0, N, 3)
        assert ex.timings()["kernel_launches"] == n0


@pytest.mark.gpu
def test_two_handles_merged_match_one():
    need_gpu()
    from tests.util import near_world

    M, N = 20_001, 2
    pos, vel, ine, cols, dt = near_world(9, M, N)
    half = M // 3
    part = lambda a, lo, hi: np.ascontiguousarray(a[lo:hi])
    sub = lambda lo, hi: (part(pos, lo, hi), part(vel, lo, hi), part(ine, lo, hi),
                          {k: part(v, lo, hi) for k, v in cols.items()}, dt)
    whole, _ = handle(ROCKET, M, N, "fast", capacity=3, state=(pos, vel, ine, cols, dt))
    a, _ = handle(ROCKET, half, N, "fast", capacity=3, state=sub(0, half))
    b, _ = handle(ROCKET, M - half, N, "fast", capacity=3, state=sub(half, M))
    sel = SELECTIONS[13]
    with whole, a, b:
        for ex in (whole, a, b):
            ex.step(3)
        want = whole.trajectory_covariance(sel)
        traj = np.moveaxis(whole.trajectory(), 1, 0)
        got = el.merge_covariance([a.trajectory_covariance(sel), b.trajectory_covariance(sel)])
    assert np.array_equal(got[..., 0], want[..., 0])
    check_table(got, ref_table(traj, sel), scales(traj, sel), "two handles")
    check_table(want, ref_table(traj, sel), scales(traj, sel), "one handle")


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
def test_exec_covariance_against_the_default_mode(math_mode):
    need_gpu()
    M, ticks = 300, 23
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=24.0, math=math_mode, n_worlds=M, world_params=params)
    ref = w.build(sys_, **kw)
    ref.run(ticks)
    spec = [("world_pos", (4, 5, 6)), ("world_vel", (3, 4, 5)), "force"]
    runs = {}
    for name, ring, host in (("ring1", 1, False), ("ring16", 16, False), ("host", 3, True)):
        s = (sys_ | el.host_system(lambda ctx: None)) if host else sys_
        ex = w.build(s, ensemble=True, ensemble_ring=ring, covariance=spec, **kw)
        ex.run(ticks)
        runs[name] = ex
    labels = ["world_pos[4]", "world_pos[5]", "world_pos[6]", "world_vel[3]", "world_vel[4]", "world_vel[5]"] + \
        [f"force[{i}]" for i in range(6)]
    p = len(labels)
    for ent in ("rocket", "ball"):
        x = np.concatenate([ref.history_worlds(f"{ent}.world_pos")[..., 4:7], ref.history_worlds(f"{ent}.world_vel")[..., 3:6],
                            ref.history_worlds(f"{ent}.force")], -1)       # [rows, M, 12]
        got = runs["ring1"].covariance(ent)
        assert got["planes"] == labels
        assert got["count"].shape == (6,) and got["mean"].shape == (6, p) and got["cov"].shape == (6, p, p)
        want = ref_table(np.moveaxis(x, 1, 0), range(p))
        table = np.concatenate([got["count"][:, None], got["mean"], (got["cov"] * got["count"][:, None, None]).reshape(6, -1)], -1)
        check_table(table, want, scales(np.moveaxis(x, 1, 0), range(p)), ent)
        assert np.array_equal(got["cov"], np.swapaxes(got["cov"], 1, 2))
        for name, ex in runs.items():
            other = ex.covariance(ent)
            for k in ("count", "mean", "cov"):
                assert other[k].tobytes() == got[k].tobytes(), f"{ent} {k}: {name} differs from ring1"
    with pytest.raises(_lib.B200Error, match="covariance="):
        w.build(sys_, ensemble=True, **kw).covariance("rocket")
    with pytest.raises(_lib.B200ValueError):
        runs["ring1"].covariance("nobody")
