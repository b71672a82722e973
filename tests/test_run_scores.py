"""Run scores over the time axis: per-world run moments (count, mean, m2 of chosen planes) and dwells (rows beyond a
bound, first and last tick), folded with the extrema by b200_sixdof_summary_start and read by Exec.moments / Exec.dwell.

The CPU tests check the validation before any device call, the spec struct against the header, and the numpy
references themselves (the sequential shifted sums against exact rationals).  The GPU tests, in both math modes, hold
every Exec route to the sequential numpy fold of a default-mode Exec's rows bit for bit, one fold to many single-row
folds at the handle level, the old entry to its old bytes and launches, and the refusals to the previous spec."""

import ctypes
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200.executor import WORLD_POS
from tests.ensemble_util import ROCKET, SAMPLED, handle, need_gpu, no_device, rocket_world, sampled_state, two_body_world  # noqa: F401
from tests.test_ensemble_histograms import state_handle
from tests.test_run_summary import ref_tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("exact", "fast")


# --------------------------------------------------------------------------- numpy references


@np.errstate(over="ignore", invalid="ignore", divide="ignore")
def ref_moments(rows):
    """rows [R, ...] in fold order -> (n, mean, m2), each [...]: the header's four operations over the finite rows,
    one correctly rounded numpy operation each, then the table's (mean, m2)."""
    rows = np.asarray(rows, dtype=np.float64)
    n, K, S1, S2 = (np.zeros(rows.shape[1:]) for _ in range(4))
    for x in rows:
        fin = np.isfinite(x)
        K = np.where(fin & (n == 0.0), x, K)
        y = x - K
        S1 = np.where(fin, S1 + y, S1)
        S2 = np.where(fin, S2 + y * y, S2)
        n = np.where(fin, n + 1.0, n)
    mean = K + S1 / n
    d = S2 - S1 * (S1 / n)
    m2 = np.where(S2 > np.finfo(np.float64).max, np.inf, np.where(d < 0.0, 0.0, d))
    none = n == 0.0
    return n, np.where(none, np.nan, mean), np.where(none, np.nan, m2)


def ref_dwell(x, ticks, above, value):
    """x [R, ...] of the dwell's (entity, plane) -> (rows, first_tick, last_tick), each int64 [...]."""
    ticks = np.asarray(ticks, dtype=np.int64)
    hit = x > value if above else x < value  # NaN never counts
    anyh = hit.any(0)
    last = hit.shape[0] - 1 - np.argmax(hit[::-1], 0)
    return (hit.sum(0).astype(np.int64), np.where(anyh, ticks[np.argmax(hit, 0)], -1),
            np.where(anyh, ticks[last], -1))


def same(a, b):
    return np.array_equal(a, b, equal_nan=True)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


# --------------------------------------------------------------------------- CPU: validation before any device call


THR = el.Threshold("ball.world_pos", 6, below=0.0)


@pytest.mark.parametrize("kw, exc, match", [
    (dict(moments=["world_pos"]), _lib.B200Error, "moments: need World.build"),
    (dict(dwells=[THR]), _lib.B200Error, "dwells: need World.build"),
    (dict(ensemble=True, dwells=[THR] * 9), ValueError, "9 dwells: at most 8"),
    (dict(ensemble=True, dwells=[("ball.world_pos", 6, 0.0)]), TypeError, "dwells take el.Threshold"),
    (dict(ensemble=True, dwells=THR), TypeError, "dwells take a sequence"),
    (dict(ensemble=True, dwells=[el.Threshold("nosuch.world_pos", 6, below=0.0)]), _lib.B200ValueError, "nosuch"),
    (dict(ensemble=True, moments=["inertia"]), _lib.B200ValueError, "component not found: inertia"),
    (dict(ensemble=True, moments=[("world_pos", (7,))]), ValueError, r"moments item .*\[0, 7\)"),
    (dict(ensemble=True, moments=[("world_vel", (1, 1))]), ValueError, r"moments selects world_vel\[1\] twice"),
    (dict(ensemble=True, moments=["world_pos", ("world_pos", (6,))]), ValueError, "twice"),
    (dict(ensemble=True, moments=[]), ValueError, "moments selects 0 planes"),
    (dict(ensemble=True, moments="world_pos"), TypeError, "moments takes a sequence"),
    (dict(ensemble=True, moments=[("channels", (0,))]), ValueError, "channel 0, this Exec has 0"),
    (dict(ensemble=True, channels=[el.Norm("speed", "world_vel", (3, 4, 5))], moments=[("channels", (1,))]),
     ValueError, "channel 1, this Exec has 1"),
    (dict(ensemble=True, channels=[el.Norm("speed", "world_vel", (3, 4, 5))],
          dwells=[el.Threshold("ball.channels", 2, above=1.0)]), ValueError, "channel 2, this Exec has 1"),
])
def test_build_validates_scores_before_the_device(no_device, kw, exc, match):  # noqa: F811
    with pytest.raises(exc, match=match):
        two_body_world().build(el.six_dof(), **kw)


def test_dwell_on_a_non_body_entity_is_refused(no_device):  # noqa: F811
    Thrust = el.Annotated[np.ndarray, el.Component("thrust", el.ComponentType.F64)]

    @el.dataclass
    class Motor(el.Archetype):
        thrust: Thrust

    w = two_body_world()
    w.spawn(Motor(np.array([1.0])), name="motor")
    with pytest.raises(_lib.B200ValueError, match="component not found: motor.world_pos") as e:
        w.build(el.six_dof(), ensemble=True, dwells=[el.Threshold("motor.world_pos", 6, below=0.0)])
    assert e.value.code == _lib.ERR_COMPONENT_NOT_FOUND


def test_valid_scores_reach_the_handle(no_device):  # noqa: F811
    chans = [el.Norm("speed", "world_vel", (3, 4, 5))] * 1
    with pytest.raises(AssertionError, match="handle is created"):
        two_body_world().build(el.six_dof(), ensemble=True, channels=chans,
                               moments=[("world_pos", (6,)), "world_vel", "world_accel", "force", ("channels", (0,))],
                               dwells=[THR] * 8)


def test_existing_refusal_messages_are_unchanged(no_device):  # noqa: F811
    w = two_body_world()
    with pytest.raises(ValueError, match=r"covariance selects world_vel\[1\] twice"):
        w.build(el.six_dof(), ensemble=True, covariance=[("world_vel", (1, 1))])
    with pytest.raises(ValueError, match="covariance selects 26 planes: 1 to 25"):
        w.build(el.six_dof(), ensemble=True, channels=[el.Norm("speed", "world_vel", (3, 4, 5))],
                covariance=list(SAMPLED) + ["channels"])
    with pytest.raises(TypeError, match="thresholds take el.Threshold objects"):
        w.build(el.six_dof(), ensemble=True, thresholds=[("ball.world_pos", 6, 0.0)])


def test_spec_struct_matches_header(tmp_path):
    st = _lib.SummarySpec
    assert ctypes.sizeof(st) == 40
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200_sixdof.h"', 'int main(void) {',
           'printf("size %zu\\n", sizeof(b200_summary_spec));', 'printf("max %u\\n", B200_MAX_DWELLS);',
           'printf("mfields %u\\n", B200_MOMENT_FIELDS);', 'printf("dfields %u\\n", B200_DWELL_FIELDS);']
    src += [f'printf("{f} %zu\\n", offsetof(b200_summary_spec, {f}));' for f, _ in st._fields_]
    src += ["return 0; }"]
    c = tmp_path / "spec.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "spec"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", str(c), "-I", os.path.join(ROOT, "include"), "-o", str(exe)],
                   check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(st)
    assert int(got["max"]) == _lib.MAX_DWELLS == 8
    assert int(got["mfields"]) == _lib.MOMENT_FIELDS and int(got["dfields"]) == _lib.DWELL_FIELDS
    for f, _ in st._fields_:
        assert int(got[f]) == getattr(st, f).offset, f


def test_score_symbols_are_exported():
    L = _lib.lib()
    for name in ("b200_sixdof_summary_start", "b200_sixdof_moments_download", "b200_sixdof_dwells_download"):
        assert name in _lib.SYMBOLS and hasattr(L, name)


def test_references_on_hand_rows():
    """Ties, signed zeros and non-finite rows: NaN / +-inf rows are skipped by the moments and never count for a dwell
    unless they are beyond its bound (+inf is above any finite bound, NaN never is)."""
    nan, inf = np.nan, np.inf
    rows = np.array([[nan, 0.0, 5.0, -0.0], [2.0, -0.0, inf, -0.0], [nan, 1.0, 5.0, -0.0], [4.0, 1.0, -inf, -0.0]])
    n, mean, m2 = ref_moments(rows)
    assert list(n) == [2, 4, 2, 4]
    assert same(mean, [3.0, 0.5, 5.0, 0.0]) and same(m2, [2.0, 1.0, 0.0, 0.0])
    assert not np.signbit(mean[3])  # K = -0.0, y = -0.0 - K = +0.0, mean = -0.0 + 0.0 / 4 = +0.0
    r, f, l = ref_dwell(rows, [0, 5, 10, 15], True, 0.5)
    assert list(r) == [2, 2, 3, 0] and list(f) == [5, 10, 0, -1] and list(l) == [15, 15, 10, -1]
    r, f, l = ref_dwell(rows, [0, 5, 10, 15], False, 0.0)
    assert list(r) == [0, 0, 1, 0] and list(f) == [-1, -1, 15, -1] and list(l) == [-1, -1, 15, -1]
    # the first finite value sets K, after leading NaN rows: with K = 1e16 the rounding of y = x - K is exact
    x = np.array([nan, nan, 1e16, 1e16 + 2.0, 1e16 + 4.0])
    n, mean, m2 = ref_moments(x[:, None])
    assert n[0] == 3 and mean[0] == 1e16 + 2.0 and m2[0] == 8.0
    n, mean, m2 = ref_moments(np.full((3, 2), nan))
    assert list(n) == [0, 0] and np.all(np.isnan(mean)) and np.all(np.isnan(m2))


def test_reference_against_exact_rationals():
    """mean and m2 of the shifted sums within a few ulp of the exact values on spread data, and m2 = +inf at
    +-2^1000, where the exact m2 is beyond the f64 range (the statistics' rule: a diverging plane reads as an infinite
    spread, never 0)."""
    rng = np.random.default_rng(3)
    for scale, shift in ((1.0, 0.0), (1e-3, 1e6), (50.0, -3.0)):
        x = rng.normal(shift, scale, (40, 1))
        n, mean, m2 = ref_moments(x)
        fx = [Fraction(v) for v in x[:, 0]]
        mu = sum(fx) / len(fx)
        m2_exact = sum((v - mu) ** 2 for v in fx)
        assert abs(Fraction(mean[0]) - mu) <= 4 * Fraction(np.spacing(np.abs(x).max()))  # K + S1 / n: the shift's ulp
        assert abs(Fraction(m2[0]) - m2_exact) <= Fraction(1, 10 ** 6) * m2_exact
    big = 2.0 ** 1000
    x = np.array([big, -big, big, -big, big])[:, None]
    n, mean, m2 = ref_moments(x)
    fx = [Fraction(v) for v in x[:, 0]]
    mu = sum(fx) / len(fx)
    assert sum((v - mu) ** 2 for v in fx) > Fraction(np.finfo(np.float64).max)
    assert m2[0] == np.inf and n[0] == 5
    assert abs(Fraction(mean[0]) - mu) <= 2 * Fraction(np.spacing(float(mu)))  # K + S1 / n, two roundings


# --------------------------------------------------------------------------- GPU: Exec against the default mode


CHANS = [el.Norm("speed", "world_vel", (3, 4, 5)), el.AxisAngle("pitch", (-1.0, 0.0, 0.0), (0.0, 0.0, 1.0))]
ENTITIES = ("rocket", "ball")


def _rows(ref):
    """[R, M, N, 25] from a default-mode run's history."""
    return np.stack([np.concatenate([ref.history_worlds(f"{e}.{c}") for c in SAMPLED], -1) for e in ENTITIES], 2)


def _with_channels(rows, mode):
    """rows [R, M, N, 25] widened by CHANS, computed on the device by the channel pass of a handle holding each row."""
    recs = [c._record() for c in CHANS]
    with state_handle(rows[0], mode) as h:
        h.set_channels(recs)
        ch = []
        for x in rows:
            h.set_state(x[..., :7], x[..., 7:13], None, accel=x[..., 13:19], force=x[..., 19:25])
            ch.append(h.state_channels())
    return np.concatenate([rows, np.stack(ch)], -1)


def _check_moments(got, rows, planes):
    """got [M, N, k, 3] (B200Exec.moments) against ref_moments of rows [R, M, N, R'] at `planes`, bit for bit."""
    n, mean, m2 = ref_moments(rows[..., planes])
    want = np.stack([n, mean, m2], -1)
    assert got.shape == want.shape
    assert np.array_equal(bits(got), bits(want)), np.argwhere(bits(got) != bits(want))[:5]


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", MODES)
def test_exec_scores_against_the_default_mode(math_mode):
    """Moments and dwells of every ensemble route equal the sequential numpy fold of the default mode's rows bit for bit
    (a partial last cycle included), and switching them on changes no ensemble table, extrema, threshold or final
    state."""
    need_gpu()
    M, ticks = 300, 23
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=24.0, math=math_mode, n_worlds=M, world_params=params)
    ref = w.build(sys_, **kw)
    ref.run(ticks)
    rows = _with_channels(_rows(ref), math_mode)                           # [6, M, 2, 27]
    row_ticks = np.asarray(ref.history("globals.tick")["globals.tick"], dtype=np.int64)
    assert list(row_ticks) == [0, 5, 10, 15, 20, 23]
    up = rows[4, 0, 0, 4] > rows[0, 0, 0, 4]
    mid = float(np.median(rows[3, :, 0, 4]))                              # rocket x: world-dependent counts
    conds = [el.Threshold("rocket.world_pos", 6, below=2.0),              # the rocket starts at z = 1: counts at row 0
             el.Threshold("rocket.world_pos", 6, above=1e9),              # never
             el.Threshold("rocket.channels", 0, above=5.0),               # speed, a channel plane
             el.Threshold("rocket.world_pos", 4, above=mid) if up else el.Threshold("rocket.world_pos", 4, below=mid),
             el.Threshold("ball.world_pos", 6, below=0.0)]
    moments = [("world_pos", (6,)), "world_vel", ("channels", (0, 1))]
    planes = [6] + list(range(7, 13)) + [25, 26]
    spec = [(ENTITIES.index(t.pair.split(".")[0]), t.plane, t.above, t.value) for t in conds]
    want_dw = [ref_dwell(rows[:, :, e, p], row_ticks, a, v) for e, p, a, v in spec]
    assert np.all(want_dw[0][1] == 0) and np.all(want_dw[1][0] == 0) and np.all(want_dw[1][1] == -1)
    assert len(set(want_dw[3][0])) >= 2 and np.any(want_dw[2][0] > 0)

    opts = dict(ensemble=True, channels=CHANS, extrema=True, thresholds=conds, covariance=[("channels", (0, 1))],
                quantiles=[0.1, 0.9])
    plain = w.build(sys_, **opts, **kw)
    plain.run(ticks)
    for name, ring, host in (("ring1", 1, False), ("ring16", 16, False), ("host", 3, True), ("default_ring", None, False)):
        s = (sys_ | el.host_system(lambda ctx: None)) if host else sys_
        ex = w.build(s, ensemble_ring=ring, moments=moments, dwells=conds, **opts, **kw)
        ex.run(ticks)
        _check_moments(ex.backend.moments(), rows, planes)
        n, mean, m2 = ref_moments(rows[..., planes])
        for pair, cols, idx in (("rocket.world_pos", [0], [6]), ("ball.world_vel", list(range(1, 7)), list(range(6))),
                                ("rocket.channels", [7, 8], [0, 1])):
            got = ex.moments(pair)
            e = ENTITIES.index(pair.split(".")[0])
            assert list(got["index"]) == idx
            assert got["count"].dtype == np.int64 and np.all(got["count"] == n[:, e, cols])
            assert np.array_equal(bits(got["mean"]), bits(mean[:, e, cols])), f"{name} {pair} mean"
            with np.errstate(invalid="ignore", divide="ignore"):
                var = m2[:, e, cols] / n[:, e, cols]
                assert np.array_equal(bits(got["std"]), bits(np.sqrt(var))), f"{name} {pair} std"
                assert np.array_equal(bits(got["rms"]), bits(np.sqrt(mean[:, e, cols] ** 2 + var))), f"{name} {pair} rms"
            x = rows[:, :, e][..., [planes[c] for c in cols]]
            rms = np.sqrt(np.mean(x * x, 0))
            assert np.all(np.abs(got["rms"] - rms) <= 8 * np.spacing(rms)), f"{name} {pair} rms vs numpy"
        for i in range(len(conds)):
            got = ex.dwell(i)
            for k, wnt in zip(("rows", "first_tick", "last_tick"), want_dw[i]):
                assert got[k].dtype == np.int64 and np.array_equal(got[k], wnt), f"{name} dwell {i} {k}"
            assert np.array_equal(got["first_tick"], ex.threshold(i)["tick"]), f"{name} dwell {i} vs threshold"
        assert ex.backend.extrema().tobytes() == plain.backend.extrema().tobytes(), name
        assert ex.backend.thresholds().tobytes() == plain.backend.thresholds().tobytes(), name
        for kind in plain._ens_rows:
            assert np.concatenate(ex._ens_rows[kind]).tobytes() == np.concatenate(plain._ens_rows[kind]).tobytes(), kind
        for cname in SAMPLED:
            cid = el.component_id(cname)
            assert ex.world.columns[cid].buffer.tobytes() == plain.world.columns[cid].buffer.tobytes(), f"{name}: final {cname}"
        assert ex.tick == ticks
        with pytest.raises(_lib.B200Error, match="no index of it is selected"):
            ex.moments("rocket.world_accel")
        with pytest.raises(IndexError):
            ex.dwell(len(conds))
        ex.backend.close()
    with pytest.raises(_lib.B200Error, match=r"moments=\[") as e:
        plain.moments("rocket.world_pos")
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT
    with pytest.raises(_lib.B200Error, match=r"dwells=\[") as e:
        plain.dwell(0)
    assert e.value.code == _lib.ERR_INVALID_ARGUMENT


# --------------------------------------------------------------------------- GPU: the handle


MOMENT_PLANES = [6, 10, 4, 24, 0, 13]


def _dwell_spec(N, rows):
    """Dwells: two whose bound lies between rows 3 and 4 of one world, one at the median of row 0, one that never
    counts and one that counts on every finite row."""
    def crossing(w, e, p):
        x = rows[:, w, e, p]
        return (e, p, bool(x[4] > x[3]), float(0.5 * (x[3] + x[4])))
    last = N - 1
    return [crossing(0, 0, 6), crossing(-1, last, 10), (last, 4, False, float(np.median(rows[0, :, last, 4]))),
            (0, 24, True, 1e300), (0, 19, True, -1e300)]


def _plane_view(ex, cid, k):
    """Plane k of column cid, the whole stride (padding included), as a torch tensor on the device."""
    import torch

    ptr = ex.device_plane(cid, k)
    assert ptr

    class Plane:
        __cuda_array_interface__ = {"shape": (ex.plane_stride,), "typestr": "<f8", "data": (ptr, False), "version": 3}

    return torch.as_tensor(Plane(), device="cuda")


def _poison(ex, M, N):
    """Non-finite values written through device_plane before row 0 (world_accel and force are recomputed by the next
    tick, world_pos is not)."""
    import torch

    from elodin_b200.executor import FORCE, WORLD_ACCEL

    for cid, k, b, v in ((WORLD_ACCEL, 0, 1, np.nan), (FORCE, 4, M * N // 2, np.inf), (WORLD_POS, 4, M * N - 1, -np.inf),
                         (WORLD_ACCEL, 0, M * N - 2, -np.inf)):
        _plane_view(ex, cid, k)[b] = v
    torch.cuda.synchronize()


CANARY = 1.25e300


def _canaries(ex, M, N):
    """A canary in the ld padding of every state plane a fold of MOMENT_PLANES and _dwell_spec reads."""
    import torch

    from elodin_b200.executor import FORCE, WORLD_ACCEL, WORLD_VEL

    views = []
    for p in sorted(set(MOMENT_PLANES) | {6, 10, 4, 24, 19}):
        cid, k = next((c, p - lo) for c, (lo, hi) in zip((WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE), SAMPLED.values())
                      if lo <= p < hi)
        v = _plane_view(ex, cid, k)
        v[M * N:] = CANARY
        views.append(v)
    torch.cuda.synchronize()
    return views


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", MODES)
@pytest.mark.parametrize("shape", [(7, 3), ((1 << 16) + 3, 1), (100, 300)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_one_fold_equals_single_sample_folds(shape, math_mode):
    """S rows folded at once give the bits of S one-row folds and of the numpy fold; non-finite rows are skipped; the
    ld padding is left alone; and the extrema and thresholds keep the bits of the same summary without scores."""
    need_gpu()
    M, N = shape
    S = 7
    probe, state = handle(ROCKET, M, N, math_mode, capacity=S)            # the rows, for the bounds and the reference
    with probe:
        _poison(probe, M, N)
        row0 = sampled_state(probe)
        probe.step(S)
        rows = np.concatenate([row0[None], probe.trajectory()])          # [S + 1, M, N, 25]
    assert not np.all(np.isfinite(rows))
    dw = _dwell_spec(N, rows)
    thr = dw[:3]
    big, _ = handle(ROCKET, M, N, math_mode, capacity=S, state=state)
    one, _ = handle(ROCKET, M, N, math_mode, capacity=1, state=state)
    old, _ = handle(ROCKET, M, N, math_mode, capacity=S, state=state)
    with big, one, old:
        for ex in (big, one, old):
            _poison(ex, M, N)
            if ex is old:
                ex.summary_begin(True, thr)
            else:
                ex.summary_begin(True, thr, MOMENT_PLANES, dw)
            views = _canaries(ex, M, N)
            ex.summary_add_state()                                        # row 0 at tick 0, from the state planes
            ex.sync()
            assert all(bool((v[M * N:] == CANARY).all()) for v in views)  # the padding is never written
        for ex in (big, old):
            ex.step(S)
            n0 = ex.timings()["kernel_launches"]
            ex.summary_add_trajectory()                                   # rows 1..S in one fold
            assert ex.timings()["kernel_launches"] == n0 + 1
        for s in range(S):
            one.trajectory_reset()
            one.step(1)
            one.summary_add_trajectory()
        assert one.tick == big.tick == S
        mom, dwl = big.moments(), big.dwells()
        assert mom.tobytes() == one.moments().tobytes() and dwl.tobytes() == one.dwells().tobytes()
        assert big.extrema().tobytes() == old.extrema().tobytes() == one.extrema().tobytes()
        assert big.thresholds().tobytes() == old.thresholds().tobytes() == one.thresholds().tobytes()
        ext_old, thr_old = old.extrema(), old.thresholds()
        for ex in (big, one, old):
            assert _lib.lib().b200_sixdof_status(ex._h) == 0
    _check_moments(mom, rows, MOMENT_PLANES)
    assert mom.shape == (M, N, len(MOMENT_PLANES), 3) and dwl.shape == (M, len(dw), 3)
    assert np.any(mom[..., 0] < S + 1) and np.any(mom[..., 0] == S + 1)
    for i, (e, p, a, v) in enumerate(dw):
        want = np.stack(ref_dwell(rows[:, :, e, p], np.arange(S + 1), a, v), -1).astype(np.float64)
        assert np.array_equal(dwl[:, i], want), i
    ext, th = ref_tables(rows, np.arange(S + 1), thr)
    assert same(ext_old, ext) and same(thr_old, th)
    assert np.all(dwl[:, 3, 0] == 0) and np.all(dwl[:, 3, 1] == -1)
    assert dwl[0, 0, 0] >= 1 and dwl[0, 0, 2] >= 4                       # counts inside the S-row fold


@pytest.mark.gpu
def test_old_entry_keeps_its_launches_and_bytes():
    """b200_sixdof_summary_begin is summary_start without scores: same launches per call, same tables."""
    need_gpu()
    M, N, S = 500, 2, 4
    a, state = handle(ROCKET, M, N, "exact", capacity=S)
    b, _ = handle(ROCKET, M, N, "exact", capacity=S, state=state)
    L = _lib.lib()
    thr = [(1, 6, False, 0.0), (0, 24, True, 1.0)]
    with a, b:
        counts = {}
        for ex in (a, b):
            n0 = ex.timings()["kernel_launches"]
            if ex is a:
                ex.summary_begin(True, thr)
            else:
                arr, n = ex._conditions(thr)
                spec = _lib.SummarySpec(1, n, arr, 0, 0, None, None)
                _lib.check(L.b200_sixdof_summary_start(ex._h, ctypes.byref(spec)))
                ex._n_thresholds = n
            n1 = ex.timings()["kernel_launches"]
            ex.summary_add_state()
            ex.step(S)
            n2 = ex.timings()["kernel_launches"]
            ex.summary_add_trajectory()
            n3 = ex.timings()["kernel_launches"]
            tables = (ex.extrema(), ex.thresholds())
            n4 = ex.timings()["kernel_launches"]
            counts[ex is a] = (n1 - n0, n3 - n2, n4 - n3)
            counts[(ex is a, "t")] = tables
        assert counts[True] == counts[False] == (1, 1, 1)
        for x, y in zip(counts[(True, "t")], counts[(False, "t")]):
            assert x.tobytes() == y.tobytes()
        # with scores: one more clear launch, still one fold launch, and the moment table one launch per chunk
        n0 = a.timings()["kernel_launches"]
        a.summary_begin(True, thr, [6], [(0, 6, True, 0.0)])
        assert a.timings()["kernel_launches"] - n0 == 2
        n0 = a.timings()["kernel_launches"]
        a.summary_add_state()
        a.moments()
        a.dwells()
        assert a.timings()["kernel_launches"] - n0 == 2


@pytest.mark.gpu
def test_refusals_leave_the_previous_spec_in_force():
    need_gpu()
    L = _lib.lib()
    M, N = 9, 2
    ex, _ = handle(ROCKET, M, N, "fast", capacity=2)
    with ex:
        for call in (ex.moments, ex.dwells):
            with pytest.raises(_lib.B200Error, match="summary_begin") as e:
                call()
            assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        ex.summary_begin(False, [], [6, 24], [(1, 6, False, 0.0)])
        ex.summary_add_state()
        mom, dwl = ex.moments(), ex.dwells()
        cases = [((False, [], [], []), "no extrema, thresholds, moments or dwells"),
                 ((False, [], [25]), "moment 0: plane 25, a row has 25"),
                 ((False, [], [4, 6, 4]), "moments: plane 4 twice"),
                 ((False, [], [], [(0, 6, True, float("nan"))]), "dwell 0: the bound is NaN"),
                 ((False, [], [], [(0, 6, True, 0.0)] * 9), "9 dwells: at most 8"),
                 ((False, [], [], [(N, 6, True, 0.0)]), "dwell 0: entity row 2, the world has 2"),
                 ((False, [], [], [(0, 25, True, 0.0)]), "dwell 0: plane 25, a row has 25"),
                 ((True, [(0, 6, True, 0.0)] * 9, [6]), "9 thresholds: at most 8")]
        for args, msg in cases:
            with pytest.raises(_lib.B200Error, match=msg) as e:
                if len(args) == 3:
                    args = args + ([],)
                extrema, thr, mo, dw = args
                if not mo and not dw:   # the old entry cannot carry scores: go through summary_start itself
                    spec = _lib.SummarySpec(0, 0, None, 0, 0, None, None)
                    _lib.check(L.b200_sixdof_summary_start(ex._h, ctypes.byref(spec)))
                else:
                    ex.summary_begin(extrema, thr, mo, dw)
            assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        assert L.b200_sixdof_summary_start(ex._h, None) == _lib.ERR_INVALID_ARGUMENT
        assert L.b200_sixdof_summary_start(None, None) == _lib.ERR_INVALID_ARGUMENT
        assert ex.moments().tobytes() == mom.tobytes() and ex.dwells().tobytes() == dwl.tobytes()
        ex.summary_add_state()                                            # the state again: counted twice
        m2, d2 = ex.moments(), ex.dwells()
        assert np.array_equal(m2[..., 0], 2 * mom[..., 0]) and np.array_equal(d2[:, :, 0], 2 * dwl[:, :, 0])
        assert np.array_equal(m2[..., 1], mom[..., 1])                   # the same value twice: the same mean
        n_mom, n_dwl = M * N * 2 * 3 * 8, M * 1 * 3 * 8
        buf = np.empty(n_mom // 8 + 1)
        for fn, n in ((L.b200_sixdof_moments_download, n_mom), (L.b200_sixdof_dwells_download, n_dwl)):
            for wrong in (n - 8, n + 8, 0):
                assert fn(ex._h, buf.ctypes.data, wrong) == _lib.ERR_VALUE_SIZE_MISMATCH
        assert L.b200_sixdof_status(ex._h) == 0
        ex.summary_begin(True)                                            # no scores: both downloads refuse
        with pytest.raises(_lib.B200Error, match="no moments"):
            _lib.check(L.b200_sixdof_moments_download(ex._h, buf.ctypes.data, 0))
        with pytest.raises(_lib.B200Error, match="no dwells"):
            _lib.check(L.b200_sixdof_dwells_download(ex._h, buf.ctypes.data, 0))
        # a new start clears: nothing folded reads as n = 0, NaN, and rows = 0, ticks -1
        ex.summary_begin(False, [], [6], [(0, 6, True, -1e300)])
        m0, d0 = ex.moments(), ex.dwells()
        assert np.all(m0[..., 0] == 0) and np.all(np.isnan(m0[..., 1:]))
        assert np.all(d0[..., 0] == 0) and np.all(d0[..., 1:] == -1)
        # device destinations take the same tables
        import torch

        ex.summary_add_state()
        for fn, host in ((L.b200_sixdof_moments_download, ex.moments()), (L.b200_sixdof_dwells_download, ex.dwells())):
            dev = torch.empty(host.shape, dtype=torch.float64, device="cuda")
            _lib.check(fn(ex._h, dev.data_ptr(), host.nbytes))
            assert same(dev.cpu().numpy(), host)
