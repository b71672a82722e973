"""Ensemble quantiles over the world axis (b200_sixdof_trajectory_quantiles / _state_quantiles, Exec.quantiles) against
a numpy reference of the documented definition.  A quantile is two order statistics and one fixed lerp, so every GPU
comparison is bit for bit, the sign of zero included."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from tests.ensemble_util import SAMPLED, need_gpu, no_device, rocket_world, sampled_state, two_body_world  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = (0.0, 1e-3, 1 / 3, 0.5, 0.9, 0.999, 1.0)
DBL_MAX = np.finfo(np.float64).max


# --------------------------------------------------------------------------- reference


def _keys(x):
    """IEEE totalOrder as int64 (-0 < +0); non-finite values sort after every finite one."""
    b = np.ascontiguousarray(x, dtype=np.float64).view(np.int64)
    k = np.where(b < 0, b ^ np.int64(0x7FFFFFFFFFFFFFFF), b)
    return np.where(np.isfinite(x), k, np.iinfo(np.int64).max)


def ref_quantiles(x, q, shift=0):
    """x [M, ...] -> [..., n_q]: the definition over axis 0, with rank i replaced by i + shift (the sensitivity probe)."""
    x = np.asarray(x, dtype=np.float64)
    if x.shape[0] == 0:
        return np.full(x.shape[1:] + (len(q),), np.nan)
    s = np.take_along_axis(x, np.argsort(_keys(x), axis=0, kind="stable"), 0)
    n = np.isfinite(x).sum(0)
    out = np.empty(x.shape[1:] + (len(q),))
    last = np.maximum(n - 1, 0)
    pick = lambda r: np.take_along_axis(s, np.clip(r, 0, max(x.shape[0] - 1, 0))[None], 0)[0]
    with np.errstate(invalid="ignore", over="ignore"):
        for l, lv in enumerate(q):
            h = (n.astype(np.float64) - 1.0) * np.float64(lv)
            top = h >= n - 1
            i = np.floor(np.where(top, 0, h)).astype(np.int64)
            t = h - i
            a, b = pick(np.clip(i + shift, 0, last)), pick(np.clip(i + 1 + shift, 0, last))
            d = b - a
            v = np.where(t >= 0.5, b - d * (1.0 - t), a + d * t)
            v = np.where(top, pick(np.clip(last + shift, 0, last)), v)
            out[..., l] = np.where(n == 0, np.nan, v)
    return out


def same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def sensitive(x, q, frac=0.6):
    """An off-by-one rank changes the result of most groups of x (so a bit-exact pass pins the rank)."""
    want = ref_quantiles(x, q)
    moved = [~np.equal(ref_quantiles(x, q, s), want) & ~np.isnan(want) for s in (-1, 1)]
    groups = (moved[0] | moved[1]).any(-1)
    return groups.mean() >= frac


# --------------------------------------------------------------------------- CPU


def _cpu_groups(rng):
    gs = []
    for k in range(400):
        n = int(rng.integers(0, 300))
        kind = k % 6
        x = rng.normal(0.0, 1.0, n)
        if kind == 1:
            x = rng.normal(7e6, 7.0, n)                                  # |mean| / std = 1e6
        elif kind == 2:
            x = np.round(x * 2) / 2                                      # ties
        elif kind == 3:
            x[rng.random(n) < 0.2] = np.nan
            x[rng.random(n) < 0.05] = np.inf
            x[rng.random(n) < 0.05] = -np.inf
        elif kind == 4:
            x = rng.choice([DBL_MAX, -DBL_MAX, 0.0, -0.0, 5e-324], n)
        gs.append(x)
    gs += [np.array([]), np.array([np.nan, np.inf]), np.array([2.5]), np.array([-1.0, 3.0]), np.array([-DBL_MAX, DBL_MAX])]
    return gs


def test_reference_equals_numpy():
    rng = np.random.default_rng(0)
    for x in _cpu_groups(rng):
        got = ref_quantiles(x[:, None], LEVELS)[0]
        f = x[np.isfinite(x)]
        with np.errstate(invalid="ignore", over="ignore"):
            want = np.quantile(f, LEVELS) if f.size else np.full(len(LEVELS), np.nan)
        ok = (got == want) | (np.isnan(got) & np.isnan(want))
        assert ok.all(), (x, got, want)


def test_reference_is_rank_sensitive_on_the_test_data():
    rng = np.random.default_rng(1)
    assert sensitive(rng.normal(size=(1000, 50)), LEVELS)
    assert sensitive(rng.normal(7e6, 7.0, size=(5000, 5)), LEVELS)
    assert sensitive(_degenerate(20000), LEVELS, frac=0.3)


def test_build_validates_quantiles_before_the_device(no_device):
    w, sys_ = two_body_world(), el.six_dof()
    for bad in ((0.5,), [float("nan")], []):                             # the mode is checked before the levels
        with pytest.raises(_lib.B200Error, match="ensemble=True") as e:
            w.build(sys_, quantiles=bad)
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    for bad in ([float("nan")], [1.5], [-0.1], [0.5, 1.0 + 1e-16 * 3]):
        with pytest.raises(ValueError, match="not in"):
            w.build(sys_, ensemble=True, quantiles=bad)
    for bad in ([True], [0.5, "0.9"], "0.5", 0.5):
        with pytest.raises(TypeError):
            w.build(sys_, ensemble=True, quantiles=bad)
    for bad in ([], [0.5] * 17):
        with pytest.raises(ValueError, match="1 to 16"):
            w.build(sys_, ensemble=True, quantiles=bad)
    with pytest.raises(AssertionError, match="handle is created"):
        w.build(sys_, ensemble=True, quantiles=list(np.linspace(0, 1, 16)))
    with pytest.raises(AssertionError, match="handle is created"):
        w.build(sys_, ensemble=True, quantiles=(0.9, 0.1, 0.9, np.float32(0.5), 1))


def test_quantile_symbols_and_constant_match_the_header(tmp_path):
    L = _lib.lib()
    for name in ("b200_sixdof_trajectory_quantiles", "b200_sixdof_state_quantiles", "b200_sixdof_quantile_reads"):
        assert name in _lib.SYMBOLS and hasattr(L, name)
    c = tmp_path / "q.c"
    c.write_text('#include <stdio.h>\n#include "b200_sixdof.h"\nint main(void) { printf("%u\\n", B200_MAX_QUANTILES); '
                 'return 0; }\n')
    exe = tmp_path / "q"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", str(c), "-I", os.path.join(ROOT, "include"), "-o", str(exe)],
                   check=True)
    assert int(subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout) == _lib.MAX_QUANTILES


# --------------------------------------------------------------------------- GPU


def _handle(M, N, math_mode, capacity, rocket, full, seed=0):
    from tests.util import near_world

    pos, vel, ine, cols, dt = near_world(seed, M, N)
    effs = [el.GravityConst((0.0, 0.0, -9.81)), el.ThrustBody((-1.0, 0.0, 0.0), "thrust"),
            el.DragQuadratic(0.6125, 0.0025, "wind")] if rocket else []
    ex = el.B200Exec(N, M, dt, None, effs, "rk4", math_mode, trajectory_every=1, trajectory_capacity=capacity,
                     trajectory_full=full)
    ex.set_state(pos, vel, ine, **({"thrust": cols["thrust"], "wind": cols["wind"]} if rocket else {}))
    return ex


SHAPES = [(1, 1), (7, 3), ((1 << 16) + 3, 1), (5, 1024), (100, 300), ((1 << 20) + 5, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_ring_and_state_quantiles_equal_the_reference(shape, math_mode):
    need_gpu()
    M, N = shape
    q = LEVELS
    huge = M > 1 << 20                                                  # one sample of one set: the reference sorts
    for rocket, full in ((True, True),) if huge else ((True, True), (False, False)):
        S = 1 if huge else 2
        with _handle(M, N, math_mode, S, rocket, full) as ex:
            ex.step(S)
            traj = ex.trajectory()                                      # [S, M, N, W]
            got = ex.trajectory_quantiles(q)
            assert got.shape == (S, N, 25 if full else 13, len(q))
            assert ex.trajectory_quantiles(q).tobytes() == got.tobytes()
            assert same_bits(got, ref_quantiles(np.moveaxis(traj, 1, 0), q)), (rocket, full)
            st = ex.state_quantiles(q)
            assert same_bits(st, ref_quantiles(sampled_state(ex), q)), (rocket, full)
            if M >= 100:
                assert sensitive(np.moveaxis(traj, 1, 0)[:, 0, :, :7], q, frac=0.5)


def _degenerate(M, seed=3):
    """[M, 25] planes of degenerate data (see test_degenerate_data_equals_the_reference)."""
    rng = np.random.default_rng(seed)
    x = np.empty((M, 25))
    x[:, 0] = 1.25                                                      # all worlds equal
    x[:, 1] = np.where(rng.random(M) < 1e-5, -3.0, 2.0)                 # two values, 1:1e5
    x[: 2, 1] = -3.0
    x[:, 2] = rng.choice([0.0, -0.0, 5e-324, -5e-324, 2.2e-308], M)      # signed zeros and subnormals
    x[:, 3] = rng.normal(0.0, 1.0, M)                                   # straddles zero
    x[:, 4] = 6.9e6 + rng.normal(0.0, 1.0, M)                           # orbital offset, metre spread
    x[:, 5] = rng.choice([DBL_MAX, -DBL_MAX], M)
    x[:, 6] = rng.normal(0.0, 1.0, M)
    x[rng.random(M) < 0.1, 6] = np.nan                                  # non-finite worlds drop out
    x[rng.random(M) < 0.05, 6] = np.inf
    x[rng.random(M) < 0.05, 6] = -np.inf
    x[:, 7] = np.nan                                                    # no finite world
    x[:, 8] = rng.choice([1.0, 2.0, 3.0], M)                            # heavy ties, three values
    x[:, 9] = rng.choice([0.0, -0.0], M)
    x[:, 10] = np.ldexp(rng.random(M), rng.integers(-1074, 1023, M)) * rng.choice([-1, 1], M)  # every binade
    x[:, 11:] = rng.normal(0.0, 1.0, (M, 14)) * np.logspace(-300, 300, 14)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("M", [1000, 20000, (1 << 18) + 1])
def test_degenerate_data_equals_the_reference(M, math_mode):
    need_gpu()
    x = _degenerate(M)[:, None, :]                                       # [M, 1, 25]
    ine = np.tile(np.array([1.0, 1.0, 1.0, 0, 0, 0, 1.0]), (M, 1, 1))
    with el.B200Exec(1, M, 0.01, None, [], "rk4", math_mode) as ex:
        ex.set_state(x[..., :7], x[..., 7:13], ine, accel=x[..., 13:19], force=x[..., 19:25])
        st = sampled_state(ex)
        assert same_bits(st, x)
        got = ex.state_quantiles(LEVELS)
        assert ex.quantile_reads() <= 8
    want = ref_quantiles(x, LEVELS)
    assert same_bits(got, want)
    assert np.all(np.isnan(got[0, 7])) and np.all(got[0, 0] == 1.25)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(100, 3), (10000, 1)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_ring_size_changes_neither_bytes_nor_launch_count(shape):
    need_gpu()
    M, N = shape
    q = (0.01, 0.5, 0.99)
    big = _handle(M, N, "fast", 64, True, False)
    one = _handle(M, N, "fast", 1, True, False)
    with big, one:
        big.step(64)
        n0 = big.timings()["kernel_launches"]
        table = big.trajectory_quantiles(q)
        n64 = big.timings()["kernel_launches"] - n0
        for s in range(64):
            one.trajectory_reset()
            one.step(1)
            n0 = one.timings()["kernel_launches"]
            row = one.trajectory_quantiles(q)
            assert one.timings()["kernel_launches"] - n0 == n64
            assert row.tobytes() == table[s:s + 1].tobytes(), s


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
def test_groups_beyond_one_scratch_slice(math_mode):
    """More groups than one slice of scratch holds: 9000 worlds x 64 samples x 25 planes = 1600 groups (a slice holds
    about 1350), and 9000 worlds x 60 entities x 25 planes in the state.  The slices run the same launch sequence each
    and give the same bytes as the reference."""
    need_gpu()
    M, S = 9000, 64
    q = (0.01, 0.5, 0.99)
    with _handle(M, 1, math_mode, S, True, True) as ex:
        ex.step(1)
        n0 = ex.timings()["kernel_launches"]
        one = ex.trajectory_quantiles(q)                                 # 25 groups: one slice
        per_slice = ex.timings()["kernel_launches"] - n0
        assert per_slice == 18 and same_bits(one, ref_quantiles(np.moveaxis(ex.trajectory(), 1, 0), q))
        ex.trajectory_reset()
        ex.step(S)
        n0 = ex.timings()["kernel_launches"]
        got = ex.trajectory_quantiles(q)
        assert ex.timings()["kernel_launches"] - n0 == 2 * per_slice
        assert same_bits(got, ref_quantiles(np.moveaxis(ex.trajectory(), 1, 0), q))
        assert 1 <= ex.quantile_reads() <= 8
    with _handle(M, 60, math_mode, 1, True, True, seed=5) as ex:
        ex.step(1)
        n0 = ex.timings()["kernel_launches"]
        got = ex.state_quantiles(q)
        assert ex.timings()["kernel_launches"] - n0 == 2 * per_slice
        assert same_bits(got, ref_quantiles(sampled_state(ex), q))


@pytest.mark.gpu
def test_refusals_leave_the_handle_usable_and_device_destinations_match():
    need_gpu()
    import torch

    L = _lib.lib()
    M, N = 20000, 2
    dp = ctypes.POINTER(ctypes.c_double)
    with _handle(M, N, "exact", 2, True, True) as ex:
        ex.step(2)
        good = ex.trajectory_quantiles((0.5, 0.25))
        for lv in ([], [0.5] * 17, [np.nan], [1.5], [-0.1]):
            a = np.array(lv if lv else [0.5])
            with pytest.raises(_lib.B200Error) as e:
                _lib.check(L.b200_sixdof_trajectory_quantiles(ex._h, a.ctypes.data_as(dp), len(lv), good.ctypes.data, 0))
            assert e.value.code == _lib.ERR_INVALID_ARGUMENT, lv
        a = np.array([0.5, 0.25])
        for wrong in (good.nbytes - 8, good.nbytes + 8, 0):
            assert L.b200_sixdof_trajectory_quantiles(ex._h, a.ctypes.data_as(dp), 2, good.ctypes.data, wrong) \
                == _lib.ERR_VALUE_SIZE_MISMATCH
            assert L.b200_sixdof_state_quantiles(ex._h, a.ctypes.data_as(dp), 2, good.ctypes.data, wrong) \
                == _lib.ERR_VALUE_SIZE_MISMATCH
        assert L.b200_sixdof_status(ex._h) == 0
        assert ex.trajectory_quantiles((0.5, 0.25)).tobytes() == good.tobytes()
        dev = torch.empty(good.shape, dtype=torch.float64, device="cuda")
        ex.trajectory_quantiles((0.5, 0.25), out_ptr=dev.data_ptr())
        assert dev.cpu().numpy().tobytes() == good.tobytes()
        ex.trajectory_reset()                                           # an empty ring: bytes = 0, no launch
        n0 = ex.timings()["kernel_launches"]
        assert ex.trajectory_quantiles((0.5,)).shape == (0, N, 25, 1)
        assert ex.timings()["kernel_launches"] == n0


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("M", [300, 9000])
def test_exec_quantiles_against_the_default_mode(M, math_mode):
    need_gpu()
    ticks = 23
    q = (0.01, 0.5, 0.99, 0.5)
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=24.0, math=math_mode, n_worlds=M, world_params=params)
    ref = w.build(sys_, **kw)
    ref.run(ticks)
    plain = w.build(sys_, ensemble=True, extrema=True, **kw)
    plain.run(ticks)
    runs = {}
    for name, ring, host in (("ring1", 1, False), ("ring16", 16, False), ("host", 3, True), ("default_ring", None, False)):
        s = (sys_ | el.host_system(lambda ctx: None)) if host else sys_
        ex = w.build(s, ensemble=True, ensemble_ring=ring, extrema=True, quantiles=q, **kw)
        ex.run(ticks)
        runs[name] = ex
        for ent in ("rocket", "ball"):
            for comp in SAMPLED:
                pair = f"{ent}.{comp}"
                got = ex.quantiles(pair)
                rows = ref.history_worlds(pair)                          # [R, M, width]
                with np.errstate(invalid="ignore", over="ignore"):
                    want = np.stack([np.quantile(r, q, axis=0) for r in rows])  # [R, n_q, width]
                assert got.shape == want.shape and np.all(got == want), f"{name} {pair}"
                assert same_bits(got, np.moveaxis(ref_quantiles(np.moveaxis(rows, 1, 0), q), -1, 1)), f"{name} {pair}"
                a, b = ex.ensemble(pair), plain.ensemble(pair)
                assert all(a[k].tobytes() == b[k].tobytes() for k in a), f"{name}: ensemble {pair} changed"
                a, b = ex.extrema(pair), plain.extrema(pair)
                assert all(a[k].tobytes() == b[k].tobytes() for k in a), f"{name}: extrema {pair} changed"
        for cname in SAMPLED:
            cid = el.component_id(cname)
            assert np.array_equal(ex.world.columns[cid].buffer, plain.world.columns[cid].buffer), f"{name}: final {cname}"
    for name, ex in runs.items():
        for pair in ("rocket.world_pos", "rocket.world_vel", "ball.force"):
            assert ex.quantiles(pair).tobytes() == runs["ring1"].quantiles(pair).tobytes(), name
        ex.backend.close()
    with pytest.raises(_lib.B200Error, match="quantiles=") as e:
        plain.quantiles("rocket.world_pos")
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    for pair in ("rocket.inertia", "rocket.thrust"):
        with pytest.raises(_lib.B200ValueError) as e:
            runs["ring1"].quantiles(pair)
        assert e.value.code == _lib.ERR_COMPONENT_NOT_FOUND
