"""Run summaries over the time axis (b200_sixdof_summary_* / Exec's extrema and thresholds in ensemble mode) against
plain numpy on the same rows.  Nothing here involves arithmetic, so every comparison is exact: values with
np.array_equal (NaN equal to NaN), ticks with ==."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from tests.ensemble_util import SAMPLED, need_gpu, no_device, rocket_world, sampled_state, two_body_world  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# --------------------------------------------------------------------------- numpy references


def ref_extrema(rows, ticks):
    """rows [R, ...] in tick order, ticks [R] -> (min, max, min_tick, max_tick, first_nonfinite_tick), each [...]."""
    rows = np.asarray(rows, dtype=np.float64)
    ticks = np.asarray(ticks, dtype=np.int64)
    fin = np.isfinite(rows)
    anyf = fin.any(0)
    kmin = np.argmin(np.where(fin, rows, np.inf), 0)  # the first of equal values: the earliest tick
    kmax = np.argmax(np.where(fin, rows, -np.inf), 0)
    pick = lambda k: np.take_along_axis(rows, k[None], 0)[0]
    mn = np.where(anyf, pick(kmin), np.nan)
    mx = np.where(anyf, pick(kmax), np.nan)
    bad = ~fin
    return (mn, mx, np.where(anyf, ticks[kmin], -1), np.where(anyf, ticks[kmax], -1),
            np.where(bad.any(0), ticks[np.argmax(bad, 0)], -1))


def ref_threshold(state, ticks, plane, above, value):
    """state [R, M, 25] of the threshold's entity -> (tick [M], planes [M, 25])."""
    x = state[:, :, plane]
    fire = x > value if above else x < value  # NaN never fires
    hit = fire.any(0)
    k = np.argmax(fire, 0)
    planes = state[k, np.arange(state.shape[1])]
    planes[~hit] = np.nan
    return np.where(hit, np.asarray(ticks, dtype=np.int64)[k], -1), planes


def ref_tables(rows, ticks, thresholds):
    """rows [R, M, N, 25] -> the two public tables: [M, N, 25, 5] and [M, T, 26]."""
    ext = np.stack([f.astype(np.float64) for f in ref_extrema(rows, ticks)], -1)
    thr = np.empty((rows.shape[1], len(thresholds), 26))
    for i, (ent, plane, above, value) in enumerate(thresholds):
        tick, planes = ref_threshold(rows[:, :, ent, :], ticks, plane, above, value)
        thr[:, i, 0] = tick
        thr[:, i, 1:] = planes
    return ext, thr


def same(a, b):
    return np.array_equal(a, b, equal_nan=True)


# --------------------------------------------------------------------------- CPU: validation before any device call


def test_threshold_validates_its_arguments():
    t = el.Threshold("ball.world_pos", 6, below=0.0)
    assert (t.plane, t.above, t.value) == (6, False, 0.0)
    assert el.Threshold("rocket.force", 5, above=1).plane == 24
    assert el.Threshold("rocket.world_vel", 0, above=-3.5).plane == 7
    with pytest.raises(ValueError, match="exactly one"):
        el.Threshold("ball.world_pos", 6)
    with pytest.raises(ValueError, match="exactly one"):
        el.Threshold("ball.world_pos", 6, below=0.0, above=1.0)
    with pytest.raises(ValueError, match="NaN"):
        el.Threshold("ball.world_pos", 6, below=float("nan"))
    for bad in (7, -1, 2.0, True):
        with pytest.raises(ValueError, match="index"):
            el.Threshold("ball.world_pos", bad, below=0.0)
    with pytest.raises(ValueError, match="index"):
        el.Threshold("ball.force", 6, above=0.0)
    for pair in ("ball.inertia", "ball.thrust", "world_pos"):
        with pytest.raises(_lib.B200ValueError, match=pair) as e:
            el.Threshold(pair, 0, below=0.0)
        assert e.value.code == _lib.ERR_COMPONENT_NOT_FOUND


def test_build_validates_summaries_before_the_device(no_device):
    w = two_body_world()
    sys_ = el.six_dof()
    with pytest.raises(_lib.B200ValueError, match="nosuch.world_pos") as e:
        w.build(sys_, ensemble=True, thresholds=[el.Threshold("nosuch.world_pos", 6, below=0.0)])
    assert e.value.code == _lib.ERR_COMPONENT_NOT_FOUND
    for kw in (dict(extrema=True), dict(thresholds=[el.Threshold("ball.world_pos", 6, below=0.0)])):
        with pytest.raises(_lib.B200Error, match="ensemble=True") as e:
            w.build(sys_, **kw)
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    with pytest.raises(ValueError, match="at most 8"):
        w.build(sys_, ensemble=True, thresholds=[el.Threshold("ball.world_pos", 6, below=0.0)] * 9)
    with pytest.raises(TypeError):
        w.build(sys_, ensemble=True, thresholds=[("ball.world_pos", 6, 0.0)])
    # a valid request gets as far as the handle
    with pytest.raises(AssertionError, match="handle is created"):
        w.build(sys_, ensemble=True, extrema=True, thresholds=[el.Threshold("ball.world_pos", 6, below=0.0)] * 8)


def test_threshold_struct_matches_header(tmp_path):
    st = _lib.Threshold
    assert ctypes.sizeof(st) == 24
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200_sixdof.h"', 'int main(void) {',
           'printf("size %zu\\n", sizeof(b200_threshold));',
           'printf("fields %u\\n", B200_EXTREMA_FIELDS);', 'printf("max %u\\n", B200_MAX_THRESHOLDS);']
    src += [f'printf("{f} %zu\\n", offsetof(b200_threshold, {f}));' for f, _ in st._fields_]
    src += ["return 0; }"]
    c = tmp_path / "thr.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "thr"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", str(c), "-I", os.path.join(ROOT, "include"), "-o", str(exe)],
                   check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(st)
    assert int(got["fields"]) == _lib.EXTREMA_FIELDS and int(got["max"]) == _lib.MAX_THRESHOLDS
    for f, _ in st._fields_:
        assert int(got[f]) == getattr(st, f).offset, f


def test_references_pick_the_earliest_tick_and_skip_non_finite_rows():
    """The numpy references themselves, on rows with ties, signed zeros and non-finite values."""
    nan, inf = np.nan, np.inf
    rows = np.array([[0.0, nan, 5.0], [-0.0, 1.0, inf], [-2.0, nan, 5.0], [-2.0, 1.0, -inf]])  # [R=4, 3]
    mn, mx, mn_t, mx_t, nf_t = ref_extrema(rows, [0, 5, 10, 15])
    assert same(mn, [-2.0, 1.0, 5.0]) and same(mx, [0.0, 1.0, 5.0])
    assert list(mn_t) == [10, 5, 0] and list(mx_t) == [0, 5, 0] and list(nf_t) == [-1, 0, 5]
    assert not np.signbit(mx[0])  # +0 at tick 0 came first
    state = rows[:, :, None].repeat(25, -1)
    tick, planes = ref_threshold(state, [0, 5, 10, 15], 0, False, -1.0)
    assert list(tick) == [10, -1, 15]
    assert same(planes[0], np.full(25, -2.0)) and np.all(np.isnan(planes[1])) and same(planes[2], np.full(25, -inf))
    tick, _ = ref_threshold(state, [0, 5, 10, 15], 0, True, 4.0)
    assert list(tick) == [-1, -1, 0]


# --------------------------------------------------------------------------- GPU


def _rows(ref, entities):
    """[R, M, N, 25] from a default-mode run's history."""
    return np.stack([np.concatenate([ref.history_worlds(f"{e}.{c}") for c in SAMPLED], -1) for e in entities], 2)


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
def test_exec_summaries_against_the_default_mode(math_mode):
    """Extrema and threshold events of every ensemble route equal numpy on the default mode's history_worlds rows,
    bit for bit, and switching them on changes no ensemble row and no final state."""
    need_gpu()
    M, ticks = 300, 23
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=24.0, math=math_mode, n_worlds=M, world_params=params)
    ref = w.build(sys_, **kw)
    ref.run(ticks)
    entities = ("rocket", "ball")
    rows = _rows(ref, entities)                                           # [6, M, 2, 25]
    row_ticks = np.asarray(ref.history("globals.tick")["globals.tick"], dtype=np.int64)
    assert list(row_ticks) == [0, 5, 10, 15, 20, 23]
    mid = float(np.median(rows[4, :, 0, 4]))                              # rocket x: fires at world-dependent rows
    thresholds = [el.Threshold("ball.world_pos", 6, below=0.0),           # the ball falls: fires at row 1, not row 0
                  el.Threshold("rocket.world_pos", 6, below=2.0),         # the rocket starts at z = 1: row 0
                  el.Threshold("rocket.world_pos", 6, above=1e9),         # never
                  el.Threshold("rocket.world_pos", 4, above=mid) if rows[4, 0, 0, 4] > rows[0, 0, 0, 4]
                  else el.Threshold("rocket.world_pos", 4, below=mid),
                  el.Threshold("ball.force", 5, below=0.0)]               # row 0 holds the spawned zero force: row 1
    spec = [(entities.index(t.pair.split(".")[0]), t.plane, t.above, t.value) for t in thresholds]
    want_ext, want_thr = ref_tables(rows, row_ticks, spec)
    assert list(want_thr[0, :3, 0]) == [5, 0, -1] and np.all(want_thr[:, 4, 0] == 5)
    assert len(set(want_thr[:, 3, 0])) >= 2

    plain = w.build(sys_, ensemble=True, **kw)
    plain.run(ticks)
    for name, ring, host in (("ring1", 1, False), ("ring16", 16, False), ("host", 3, True), ("default_ring", None, False)):
        s = (sys_ | el.host_system(lambda ctx: None)) if host else sys_
        ex = w.build(s, ensemble=True, ensemble_ring=ring, extrema=True, thresholds=thresholds, **kw)
        launches = ex.backend.timings()["kernel_launches"]
        ex.run(ticks)
        assert ex.backend.timings()["kernel_launches"] > launches
        for e, ent in enumerate(entities):
            for comp, (lo, hi) in SAMPLED.items():
                got = ex.extrema(f"{ent}.{comp}")
                for f, key in enumerate(("min", "max", "min_tick", "max_tick", "first_nonfinite_tick")):
                    want = want_ext[:, e, lo:hi, f]
                    if f < 2:
                        assert got[key].shape == (M, hi - lo) and same(got[key], want), f"{name} {ent}.{comp} {key}"
                    else:
                        assert got[key].dtype == np.int64 and np.all(got[key] == want), f"{name} {ent}.{comp} {key}"
        for i in range(len(thresholds)):
            got = ex.threshold(i)
            assert got["tick"].dtype == np.int64 and np.all(got["tick"] == want_thr[:, i, 0]), f"{name} threshold {i}"
            for comp, (lo, hi) in SAMPLED.items():
                assert got[comp].shape == (M, hi - lo) and same(got[comp], want_thr[:, i, 1 + lo:1 + hi]), f"{name} {i} {comp}"
        for pair in ("rocket.world_pos", "rocket.force", "ball.world_vel", "ball.world_accel"):
            a, b = ex.ensemble(pair), plain.ensemble(pair)
            for k in a:
                assert a[k].tobytes() == b[k].tobytes(), f"{name}: ensemble {pair} {k} changed"
        for cname in SAMPLED:
            cid = el.component_id(cname)
            assert np.array_equal(ex.world.columns[cid].buffer, plain.world.columns[cid].buffer), f"{name}: final {cname}"
        assert ex.tick == ticks
        ex.backend.close()
    with pytest.raises(_lib.B200Error, match="extrema=True") as e:
        plain.extrema("rocket.world_pos")
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    with pytest.raises(_lib.B200Error, match="thresholds=") as e:
        plain.threshold(0)
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT


def _handle(M, N, math_mode, capacity, full=True, seed=0, state=None):
    """A rocket-set handle with a trajectory ring sampled every tick and a random initial state."""
    from tests.util import near_world

    pos, vel, ine, cols, dt = near_world(seed, M, N) if state is None else state
    effs = [el.GravityConst((0.0, 0.0, -9.81)), el.ThrustBody((-1.0, 0.0, 0.0), "thrust"),
            el.DragQuadratic(0.6125, 0.0025, "wind")]
    ex = el.B200Exec(N, M, dt, None, effs, "rk4", math_mode, trajectory_every=1, trajectory_capacity=capacity,
                     trajectory_full=full)
    ex.set_state(pos, vel, ine, thrust=cols["thrust"], wind=cols["wind"])
    return ex, (pos, vel, ine, cols, dt)


def _spec(N, rows):
    """Thresholds: two whose bound lies between rows 3 and 4 of one world (so that world fires mid-run), one at the
    median of row 0 (half the worlds fire at row 0), one that never fires and one that fires at row 0 everywhere."""
    def crossing(w, e, p):
        x = rows[:, w, e, p]
        return (e, p, bool(x[4] > x[3]), float(0.5 * (x[3] + x[4])))
    last = N - 1
    return [crossing(0, 0, 6), crossing(-1, last, 10), (last, 4, False, float(np.median(rows[0, :, last, 4]))),
            (0, 24, True, 1e300), (0, 19, True, -1e300)]


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("shape", [(7, 3), ((1 << 16) + 3, 1), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_one_fold_equals_single_sample_folds_and_refolding_changes_nothing(shape, math_mode):
    need_gpu()
    M, N = shape
    S = 7
    probe, state = _handle(M, N, math_mode, capacity=S)                 # the rows, for the bounds and the reference
    with probe:
        row0 = sampled_state(probe)
        probe.step(S)
        rows = np.concatenate([row0[None], probe.trajectory()])          # [S + 1, M, N, 25]
    spec = _spec(N, rows)
    big, _ = _handle(M, N, math_mode, capacity=S, state=state)
    one, _ = _handle(M, N, math_mode, capacity=1, state=state)
    with big, one:
        for ex in (big, one):
            ex.summary_begin(True, spec)
            ex.summary_add_state()                                        # row 0 at tick 0
        big.step(S)
        launches = big.timings()["kernel_launches"]
        big.summary_add_trajectory()                                      # rows 1..S in one fold
        assert big.timings()["kernel_launches"] == launches + 1
        ext, thr = big.extrema(), big.thresholds()
        for s in range(S):
            one.trajectory_reset()
            one.step(1)
            one.summary_add_trajectory()
        assert one.tick == big.tick == S
        assert ext.tobytes() == one.extrema().tobytes()
        assert thr.tobytes() == one.thresholds().tobytes()
        big.summary_add_trajectory()                                      # the same S rows again
        big.summary_add_state()                                           # and the last one a third time
        assert big.extrema().tobytes() == ext.tobytes() and big.thresholds().tobytes() == thr.tobytes()
        assert big.timings()["kernel_launches"] > launches + 1
        assert _lib.lib().b200_sixdof_status(big._h) == 0
    want_ext, want_thr = ref_tables(rows, np.arange(S + 1), spec)
    assert ext.shape == (M, N, 25, 5) and thr.shape == (M, len(spec), 26)
    assert same(ext, want_ext) and same(thr, want_thr)
    assert np.all(thr[:, 3, 0] == -1) and np.all(thr[:, 4, 0] == 0)
    assert 0 < thr[0, 0, 0] <= 4 and 0 < thr[-1, 1, 0] <= 4  # mid-run events, caught in the S-row fold
    assert np.any(thr[:, 2, 0] == 0) and np.any(thr[:, 2, 0] != 0)


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
@pytest.mark.parametrize("shape", [(7, 3), ((1 << 16) + 3, 1), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_non_finite_rows_are_reported_and_skipped(shape, math_mode):
    """Free bodies: a NaN / inf put into a world's position stays in its plane, so first_nonfinite_tick is 0 exactly
    there and -1 everywhere else, and min / max come from the finite rows alone."""
    need_gpu()
    from tests.util import near_world

    M, N = shape
    pos, vel, ine, _, dt = near_world(2, M, N)
    bad = [(1, 0, 4, np.nan), (M // 2, N - 1, 6, -np.inf), (M - 2, 0, 5, np.inf)]
    for w, e, p, v in bad:
        pos[w, e, p] = v
    S = 5
    with el.B200Exec(N, M, dt, None, [], "rk4", math_mode, trajectory_every=1, trajectory_capacity=S,
                     trajectory_full=True) as ex:
        ex.set_state(pos, vel, ine)
        ex.summary_begin(True, [(0, 4, True, -1e300)])                   # every finite x fires at row 0
        row0 = sampled_state(ex)
        ex.summary_add_state()
        ex.step(S)
        traj = ex.trajectory()
        ex.summary_add_trajectory()
        ext, thr = ex.extrema(), ex.thresholds()
    rows = np.concatenate([row0[None], traj])
    want_ext, want_thr = ref_tables(rows, np.arange(S + 1), [(0, 4, True, -1e300)])
    assert same(ext, want_ext) and same(thr, want_thr)
    nf = np.full((M, N, 25), -1.0)
    for w, e, p, _ in bad:
        nf[w, e, p] = 0.0
    assert np.array_equal(ext[..., 4], nf)
    w, e, p, _ = bad[0]
    assert np.all(np.isnan(ext[w, e, p, :2])) and list(ext[w, e, p, 2:4]) == [-1.0, -1.0]  # x never finite
    assert thr[w, 0, 0] == -1 and np.all(np.isnan(thr[w, 0, 1:]))     # NaN never fires
    assert np.all(np.delete(thr[:, 0, 0], w) == 0)


@pytest.mark.gpu
def test_refusals_leave_the_handle_usable():
    need_gpu()
    L = _lib.lib()
    M, N = 9, 2
    thin, _ = _handle(M, N, "fast", capacity=2, full=False)
    ex, _ = _handle(M, N, "fast", capacity=2)
    with thin, ex:
        for call in (ex.summary_add_state, ex.summary_add_trajectory, ex.extrema, ex.thresholds):
            with pytest.raises(_lib.B200Error, match="summary_begin") as e:
                call()
            assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        for extrema, spec in ((True, [(N, 0, False, 0.0)]), (True, [(0, 25, False, 0.0)]),
                              (True, [(0, 6, True, float("nan"))]), (True, [(0, 6, False, 0.0)] * 9), (False, [])):
            with pytest.raises(_lib.B200Error) as e:
                ex.summary_begin(extrema, spec)
            assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        thin.summary_begin(True)
        thin.step(2)
        with pytest.raises(_lib.B200Error, match="B200_TRAJ_FULL") as e:
            thin.summary_add_trajectory()
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        with pytest.raises(_lib.B200Error, match="no thresholds") as e:
            thin.thresholds()
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT

        ex.summary_begin(False, [(1, 6, False, 0.0)])
        with pytest.raises(_lib.B200Error, match="no extrema") as e:
            ex.extrema()
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        ex.summary_begin(True, [(1, 6, False, 0.0), (0, 0, True, -1e300)])
        n_ext, n_thr = M * N * 25 * 5 * 8, M * 2 * 26 * 8
        buf = np.empty(n_ext // 8 + 1)
        for fn, n in ((L.b200_sixdof_extrema_download, n_ext), (L.b200_sixdof_thresholds_download, n_thr)):
            for wrong in (n - 8, n + 8, 0):
                assert fn(ex._h, buf.ctypes.data, wrong) == _lib.ERR_VALUE_SIZE_MISMATCH
        for h in (ex._h, thin._h):
            assert L.b200_sixdof_status(h) == 0
        # begin starts over: nothing folded yet reads as "never"
        ex.summary_add_state()
        ex.step(2)
        ex.summary_add_trajectory()
        assert np.all(ex.thresholds()[:, 1, 0] == 0)
        ex.summary_begin(True, [(1, 6, False, 0.0)])
        ext, thr = ex.extrema(), ex.thresholds()
        assert np.all(np.isnan(ext[..., :2])) and np.all(ext[..., 2:] == -1.0)
        assert thr.shape == (M, 1, 26) and np.all(thr[..., 0] == -1.0) and np.all(np.isnan(thr[..., 1:]))
        # device destinations take the same tables
        import torch

        ex.summary_add_state()
        host = ex.extrema()
        dev = torch.empty(host.shape, dtype=torch.float64, device="cuda")
        _lib.check(L.b200_sixdof_extrema_download(ex._h, dev.data_ptr(), host.nbytes))
        assert same(dev.cpu().numpy(), host)
        t_host = ex.thresholds()
        t_dev = torch.empty(t_host.shape, dtype=torch.float64, device="cuda")
        _lib.check(L.b200_sixdof_thresholds_download(ex._h, t_dev.data_ptr(), t_host.nbytes))
        assert same(t_dev.cpu().numpy(), t_host)
