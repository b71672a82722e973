"""Derived channels in ensemble mode: per-body speeds, distances, altitudes and pointing angles computed on the device
(b200_sixdof_set_channels, channel_kernels.cu) and reduced as planes 25 + k of every ensemble table.

The CPU tests check the numpy restatement of both channel kinds against exact arithmetic and the oracle's rotation,
the validation of el.Norm / el.AxisAngle / World.build(..., channels=...) before any device call, and the addressing
of "<entity>.channels" through a fake backend.  The GPU tests, in both math modes, hold the channel values to the
restatement (NORM bit for bit, AXIS_ANGLE within CUDA's documented 2 ulp for double atan2), every reduction of a
channel plane to its exact reference, planes 0-24 of every table to the same handle without channels, the run
summaries to a numpy fold, an Exec to a default-mode Exec over the same worlds, the refusals of the C ABI, and two
gloo ranks to one."""

from fractions import Fraction

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from oracle import oracle as O
from tests.ensemble_util import (ROCKET, handle, need_gpu, no_device, rocket_world, run_gloo,  # noqa: F401
                                 sampled_state, two_body_world)
from tests.test_ensemble_histograms import state_handle
from tests.test_ensemble_retained import _EnsembleFake
from tests.test_host_logic import _FakeBackend

MODES = ("exact", "fast")
ATAN2_ULP = 2  # CUDA Math API: maximum ulp error of double atan2(y, x)
LEVELS = (0.0, 0.1, 0.5, 0.9, 1.0)


# --------------------------------------------------------------------------- the numpy restatement


def qrot(q, v):
    """sixdof_device.cuh ex::qrot, vectorised: q * [v, 0] * q.inverse() in correctly rounded f64 operations, in the
    device's order (numpy neither contracts nor reorders elementwise operations)."""
    i, j, k, w = (q[..., n] for n in range(4))
    vx, vy, vz = (np.broadcast_to(v[..., n], i.shape) for n in range(3))
    n2 = ((i * i + j * j) + k * k) + w * w
    ii, ij, ik, iw = -i / n2, -j / n2, -k / n2, w / n2
    z = np.zeros_like(i)

    def mul(l, r):
        li, lj, lk, lw = l
        ri, rj, rk, rw = r
        return (((lw * ri + li * rw) + lj * rk) - lk * rj,
                ((lw * rj - li * rk) + lj * rw) + lk * ri,
                ((lw * rk + li * rj) - lj * ri) + lk * rw,
                ((lw * rw - li * ri) - lj * rj) - lk * rk)

    r = mul(mul((i, j, k, w), (vx, vy, vz, z)), (ii, ij, ik, iw))
    return np.stack(r[:3], -1)


def norm_channel(rows, planes, c=(0.0, 0.0, 0.0), r0=0.0):
    s = None
    for n, p in enumerate(planes):
        d = rows[..., p] - c[n]
        s = d * d if s is None else s + d * d
    return np.sqrt(s) - r0


def angle_parts(rows, axis, d=None, plane=None):
    """(s, t) of an AXIS_ANGLE channel: |u x v| and u . v in the header's order."""
    u = qrot(rows[..., :4], np.asarray(axis, dtype=np.float64))
    v = np.broadcast_to(np.asarray(d, dtype=np.float64), u.shape) if plane is None else rows[..., plane:plane + 3]
    cx = u[..., 1] * v[..., 2] - u[..., 2] * v[..., 1]
    cy = u[..., 2] * v[..., 0] - u[..., 0] * v[..., 2]
    cz = u[..., 0] * v[..., 1] - u[..., 1] * v[..., 0]
    s = np.sqrt((cx * cx + cy * cy) + cz * cz)
    t = (u[..., 0] * v[..., 0] + u[..., 1] * v[..., 1]) + u[..., 2] * v[..., 2]
    return s, t


# (kind, C record fields, restatement)
CHANNELS = [
    ("speed", (_lib.CHANNEL_NORM, 3, (10, 11, 12), (), (), 0.0), lambda r: norm_channel(r, (10, 11, 12))),
    ("range", (_lib.CHANNEL_NORM, 2, (4, 5), (1.5, -2.0), (), 0.0), lambda r: norm_channel(r, (4, 5), (1.5, -2.0))),
    ("alt", (_lib.CHANNEL_NORM, 3, (4, 5, 6), (0.0, 0.0, 0.0), (), 0.75), lambda r: norm_channel(r, (4, 5, 6), r0=0.75)),
    ("accel", (_lib.CHANNEL_NORM, 3, (18, 16, 17), (), (), 0.0), lambda r: norm_channel(r, (18, 16, 17))),
    ("dz", (_lib.CHANNEL_NORM, 1, (6,), (-3.0,), (), 0.0), lambda r: norm_channel(r, (6,), (-3.0,))),
    ("pitch", (_lib.CHANNEL_AXIS_ANGLE, 0, (), (-1.0, 0.0, 0.0), (0.0, 0.0, 1.0), 0.0), None),
    ("aoa", (_lib.CHANNEL_AXIS_ANGLE, 3, (10,), (0.3, -2.0, 0.5), (), 0.0), None),
    ("omega_dir", (_lib.CHANNEL_AXIS_ANGLE, 3, (7,), (0.0, 0.0, 2.0), (), 0.0), None),
]


@np.errstate(over="ignore", invalid="ignore")
def ref_channels(rows, chans=CHANNELS):
    """[..., n_c] restated values, and a mask of the AXIS_ANGLE columns"""
    out, angle = [], []
    for _, (kind, n, planes, c, d, r0), f in chans:
        if kind == _lib.CHANNEL_NORM:
            out.append(f(rows))
            angle.append(False)
        else:
            s, t = angle_parts(rows, c, d=d if n == 0 else None, plane=planes[0] if n == 3 else None)
            out.append(np.arctan2(s, t))
            angle.append(True)
    return np.stack(out, -1), np.array(angle)


def check_values(got, want, angle):
    """NORM columns bit for bit; AXIS_ANGLE columns within ATAN2_ULP of np.arctan2, NaN where it is NaN"""
    assert got.shape == want.shape
    gn, wn = got[..., ~angle], want[..., ~angle]
    assert np.array_equal(gn.view(np.uint64), wn.view(np.uint64)), np.argwhere(gn.view(np.uint64) != wn.view(np.uint64))[:5]
    ga, wa = got[..., angle], want[..., angle]
    assert np.array_equal(np.isnan(ga), np.isnan(wa))
    fin = ~np.isnan(wa)
    err = np.abs(ga[fin] - wa[fin])
    assert np.all(err <= ATAN2_ULP * np.spacing(np.abs(wa[fin]))), err.max()
    assert np.all((ga[fin] >= 0.0) & (ga[fin] <= np.pi))


def records(chans=CHANNELS):
    return [_lib.channel(*rec) for _, rec, _ in chans]


# --------------------------------------------------------------------------- CPU: the restatement


def test_norm_restatement_is_the_correctly_rounded_sum_of_squares_in_order():
    """s = d0*d0; s = s + d1*d1; s = s + d2*d2, each step one correct rounding: Fraction arithmetic, rounded once per
    operation, gives numpy's bits; a square that overflows is +inf."""
    rng = np.random.default_rng(3)
    rows = rng.normal(0.0, 1.0, (400, 25)) * 10.0 ** rng.integers(-150, 150, (400, 25))
    rows[0, 10:13] = (1e200, 1.0, 0.0)
    rows[1, 10:13] = (-0.0, 0.0, -0.0)
    with np.errstate(over="ignore"):
        got = norm_channel(rows, (10, 11, 12), (0.0, 0.5, -0.25), 2.0)

    def rnd(x):  # one correct rounding of an exact value (Fraction -> float divides integers exactly rounded)
        try:
            return float(x)
        except OverflowError:
            return np.inf

    for r in range(rows.shape[0]):
        s = None
        for p, c in zip((10, 11, 12), (0.0, 0.5, -0.25)):
            d = rnd(Fraction(rows[r, p]) - Fraction(c))
            sq = rnd(Fraction(d) * Fraction(d))
            s = sq if s is None else (np.inf if np.isinf(s) or np.isinf(sq) else rnd(Fraction(s) + Fraction(sq)))
        want = np.sqrt(s) - 2.0  # sqrt and one subtraction: correctly rounded in numpy
        assert got[r] == want, r
    assert got[0] == np.inf and got[1] == np.sqrt(0.3125) - 2.0


def test_axis_angle_parts_use_the_oracles_rotation():
    """u of the restatement is the oracle's orc_qrot bit for bit, on non-unit quaternions"""
    rng = np.random.default_rng(5)
    q = rng.normal(0.0, 1.0, (300, 4)) * rng.uniform(0.1, 10.0, (300, 1))
    a = rng.normal(0.0, 1.0, (300, 3))
    got = qrot(q, a)
    want = np.array([O.qrot(q[i], a[i]) for i in range(300)])
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    rows = np.zeros((300, 25))
    rows[:, :4], rows[:, 10:13] = q, rng.normal(0.0, 1.0, (300, 3))
    s, t = angle_parts(rows, (1.0, 0.0, 0.0), plane=10)
    u = np.array([O.qrot(q[i], np.array([1.0, 0.0, 0.0])) for i in range(300)])
    v = rows[:, 10:13]
    c = np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1], u[:, 2] * v[:, 0] - u[:, 0] * v[:, 2],
                  u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], -1)
    assert np.array_equal(s, np.sqrt((c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2]))
    assert np.array_equal(t, (u[:, 0] * v[:, 0] + u[:, 1] * v[:, 1]) + u[:, 2] * v[:, 2])
    assert np.arctan2(0.0, 0.0) == 0.0  # a body at rest


# --------------------------------------------------------------------------- CPU: validation before the device


@pytest.mark.parametrize("make, exc, match", [
    (lambda: el.Norm("", "world_vel", (3, 4, 5)), ValueError, "name"),
    (lambda: el.Norm("a", "inertia", (0,)), el.B200ValueError, "component not found: inertia"),
    (lambda: el.Norm("a", "world_vel", ()), ValueError, "1 to 3"),
    (lambda: el.Norm("a", "world_vel", (0, 1, 2, 3)), ValueError, "1 to 3"),
    (lambda: el.Norm("a", "world_vel", (3, 3)), ValueError, "twice"),
    (lambda: el.Norm("a", "world_vel", (6,)), ValueError, r"\[0, 6\)"),
    (lambda: el.Norm("a", "world_pos", (4, 5), center=(1.0,)), ValueError, "center"),
    (lambda: el.Norm("a", "world_pos", (4,), center=(np.nan,)), ValueError, "center"),
    (lambda: el.Norm("a", "world_pos", (4,), minus=np.inf), ValueError, "minus"),
    (lambda: el.AxisAngle("a", (0, 0, 0), (0, 0, 1)), ValueError, "zero"),
    (lambda: el.AxisAngle("a", (1, 0), (0, 0, 1)), ValueError, "3-vector"),
    (lambda: el.AxisAngle("a", (1, 0, 0), (0, np.inf, 1)), ValueError, "finite"),
    (lambda: el.AxisAngle("a", (1, 0, 0), (0, 0, 0)), ValueError, "zero"),
    (lambda: el.AxisAngle("a", (1, 0, 0), ("world_vel", (3, 5, 4))), ValueError, "consecutive"),
    (lambda: el.AxisAngle("a", (1, 0, 0), ("world_vel", (4, 5, 6))), ValueError, r"\[0, 6\)"),
    (lambda: el.AxisAngle("a", (1, 0, 0), ("mass", (0, 1, 2))), el.B200ValueError, "component not found"),
    (lambda: el.Threshold("rocket.channels", 8, below=0.0), ValueError, r"\[0, 8\)"),
    (lambda: el.Histogram("rocket.channels", -1, range=(0, 1)), ValueError, r"\[0, 8\)"),
])
def test_channel_objects_are_validated(make, exc, match):
    with pytest.raises(exc, match=match):
        make()


def test_channel_records():
    n = el.Norm("range", "world_pos", (4, 5), center=(1.0, 2.0), minus=0.5)._record()
    assert (n.kind, n.n, tuple(n.plane), tuple(n.c), n.r0) == (_lib.CHANNEL_NORM, 2, (4, 5, 0), (1.0, 2.0, 0.0), 0.5)
    a = el.AxisAngle("aoa", (1, 0, 0), ("world_vel", (3, 4, 5)))._record()
    assert (a.kind, a.n, a.plane[0], tuple(a.c)) == (_lib.CHANNEL_AXIS_ANGLE, 3, 10, (1.0, 0.0, 0.0))
    f = el.AxisAngle("pitch", (-1, 0, 0), (0, 0, 2))._record()
    assert (f.n, tuple(f.c), tuple(f.d)) == (0, (-1.0, 0.0, 0.0), (0.0, 0.0, 2.0))
    assert _lib.ROW_PLANES == 25 and _lib.MAX_CHANNELS == 8


SPEED = el.Norm("speed", "world_vel", (3, 4, 5))


@pytest.mark.parametrize("kw, exc, match", [
    (dict(channels=[SPEED]), el.B200Error, r"channels: need World.build\(..., ensemble=True\)"),
    (dict(ensemble=True, channels=SPEED), TypeError, "sequence"),
    (dict(ensemble=True, channels=[SPEED, "x"]), TypeError, "el.Norm"),
    (dict(ensemble=True, channels=[]), ValueError, "1 to 8"),
    (dict(ensemble=True, channels=[el.Norm(f"c{i}", "world_vel", (3,)) for i in range(9)]), ValueError, "1 to 8"),
    (dict(ensemble=True, channels=[SPEED, el.Norm("speed", "world_vel", (3,))]), ValueError, "'speed' is used twice"),
    (dict(ensemble=True, channels=[SPEED], thresholds=[el.Threshold("rocket.channels", 1, below=0.0)]), ValueError,
     "this Exec has 1"),
    (dict(ensemble=True, channels=[SPEED], histograms=[el.Histogram("rocket.channels", (0, 1), range=((0, 1), (0, 1)))]),
     ValueError, "this Exec has 1"),
    (dict(ensemble=True, thresholds=[el.Threshold("rocket.channels", 0, below=0.0)]), ValueError, "this Exec has 0"),
    (dict(ensemble=True, channels=[SPEED], covariance=[("channels", (0, 1))]), ValueError, "this Exec has 1"),
    (dict(ensemble=True, covariance=[("channels", (0,))]), ValueError, "this Exec has 0"),
    (dict(ensemble=True, channels=[SPEED], covariance=[("channels", (8,))]), ValueError, r"\[0, 8\)"),
])
def test_build_refuses_bad_channels_before_the_handle(no_device, kw, exc, match):  # noqa: F811
    w = two_body_world()
    with pytest.raises(exc, match=match):
        w.build(el.six_dof(), n_worlds=2, **kw)


def test_existing_refusal_messages_are_unchanged():
    for make in (lambda: el.Threshold("rocket.inertia", 0, below=0.0), lambda: el.Histogram("rocket.wind", 0, range=(0, 1))):
        with pytest.raises(el.B200ValueError, match=r"cover world_pos, world_vel, world_accel, force\)$"):
            make()
    from elodin_b200.world import _covariance_planes

    with pytest.raises(el.B200ValueError, match=r"covers world_pos, world_vel, world_accel, force\)$"):
        _covariance_planes([("inertia", (0,))])


class _ChannelFake(_EnsembleFake):
    """The ensemble fake with channels: tables R = 25 + n_c wide whose values name their plane."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.channel_records = []

    def set_channels(self, recs):
        assert not hasattr(self, "summary"), "channels must be set before summary_begin"
        self.channel_records = list(recs)

    def _table(self, lead, fields):
        R = 25 + len(self.channel_records)
        return np.broadcast_to(np.arange(R, dtype=np.float64)[:, None], lead + (self.n_entities, R, fields)).copy()

    def state_stats(self):
        return self._table((), 5)

    def trajectory_stats(self):
        return self._table((len(self.samples),), 5)

    def state_quantiles(self, q):
        return self._table((), len(q))

    def trajectory_quantiles(self, q):
        return self._table((len(self.samples),), len(q))

    def state_covariance(self, planes):
        p = len(planes)
        t = np.zeros((self.n_entities, 1 + p + p * p))
        t[:, 1:1 + p] = planes
        return t

    def trajectory_covariance(self, planes):
        return np.stack([self.state_covariance(planes)] * len(self.samples)) if self.samples else \
            np.zeros((0, self.n_entities, 1 + len(planes) + len(planes) ** 2))

    def summary_begin(self, extrema, thresholds):
        self.summary = (extrema, list(thresholds))

    def summary_add_state(self):
        pass

    def summary_add_trajectory(self):
        pass

    def extrema(self):
        return self._table((self.n_worlds,), 5)

    def thresholds(self):
        return np.zeros((self.n_worlds, len(self.summary[1]), 26))


def test_channel_addressing_with_a_fake_backend(monkeypatch):
    from elodin_b200 import world as W

    monkeypatch.setattr(W, "B200Exec", _ChannelFake)
    chans = [SPEED, el.Norm("range", "world_pos", (4, 5)), el.AxisAngle("pitch", (-1, 0, 0), (0, 0, 1))]
    w = two_body_world()
    ex = w.build(el.six_dof(), n_worlds=3, ensemble=True, channels=chans, extrema=True, quantiles=LEVELS,
                 thresholds=[el.Threshold("rocket.channels", 1, below=0.0)],
                 covariance=[("channels", (2, 0)), ("world_pos", (4,))])
    be = ex.backend
    assert ex.channels == ["speed", "range", "pitch"]
    assert [(r.kind, r.n) for r in be.channel_records] == [(1, 3), (1, 2), (2, 0)]
    assert be.summary[1] == [(0, 26, False, 0.0)]
    ex.run(2)
    st = ex.ensemble("rocket.channels")
    assert st["mean"].shape == (3, 3) and np.array_equal(st["mean"][0], [25.0, 26.0, 27.0])
    assert np.array_equal(ex.ensemble("rocket.force")["mean"][0], np.arange(19.0, 25.0))
    q = ex.quantiles("rocket.channels")
    assert q.shape == (3, len(LEVELS), 3) and np.array_equal(q[0, 0], [25.0, 26.0, 27.0])
    cov = ex.covariance("rocket")
    assert cov["planes"] == ["pitch", "speed", "world_pos[4]"] and np.array_equal(cov["mean"][0], [27.0, 25.0, 4.0])
    e = ex.extrema("rocket.channels")
    assert e["min"].shape == (3, 3) and np.array_equal(e["min"][0], [25.0, 26.0, 27.0])


def test_channels_need_channels_to_be_addressed(monkeypatch):
    from elodin_b200 import world as W

    monkeypatch.setattr(W, "B200Exec", _ChannelFake)
    ex = two_body_world().build(el.six_dof(), n_worlds=2, ensemble=True)
    assert ex.channels == []
    with pytest.raises(el.B200Error, match=r"rocket.channels: build the Exec with .*channels=\[...\]"):
        ex.ensemble("rocket.channels")


# every table a fake reduction or run summary returns, and the code its values start with
_CODES = {k: i + 1 for i, k in enumerate(("stats", "quantiles", "covariance", "histograms", "group_stats",
                                          "group_quantiles", "group_covariance", "group_histograms",
                                          "extrema", "thresholds", "moments", "dwells"))}


def _named(kind, rows, tail):
    """[len(rows), *tail]: 1e8 * the kind's code + 1e5 * the row + the flat index of the value within the row."""
    n = int(np.prod(tail))
    t = _CODES[kind] * 1e8 + np.asarray(rows, dtype=np.float64)[:, None] * 1e5 + np.arange(n, dtype=np.float64)
    return t.reshape((len(rows),) + tuple(tail))


class _RecordingFake(_ChannelFake):
    """The channel fake with every ensemble call of an Exec recorded with its arguments, and tables from _named: the
    ensemble tables numbered by telemetry row, per kind; the run summaries as row 0."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.rows_seen, self.n_groups = {}, 0

    @staticmethod
    def _log(*call):
        _FakeBackend.calls.append(call)

    def set_channels(self, recs):
        super().set_channels(recs)
        self._log("set_channels", [(r.kind, r.n) for r in recs])

    def summary_begin(self, extrema, thresholds=(), moments=(), dwells=()):
        self.summary = (extrema, list(thresholds), list(moments), list(dwells))
        self._log("summary_begin", *self.summary)

    def set_world_groups(self, sizes):
        self.n_groups = len(sizes)
        self._log("set_world_groups", list(sizes))

    def summary_add_state(self):
        self._log("summary_add_state")

    def summary_add_trajectory(self):
        self._log("summary_add_trajectory")

    def state_worlds(self, worlds):
        self._log("state_worlds", list(worlds))
        return super().state_worlds(worlds)

    def trajectory_worlds(self, worlds):
        self._log("trajectory_worlds", list(worlds))
        return super().trajectory_worlds(worlds)

    def download(self, cid, out):
        self._log("download", cid)
        super().download(cid, out)

    def _reduce(self, kind, ring, arg):
        self._log(f"{'trajectory' if ring else 'state'}_{kind}", *[list(np.asarray(a).tolist()) if isinstance(a, np.ndarray)
                                                                 else a for a in arg])
        E, R = self.n_entities, 25 + len(self.channel_records)
        base = kind.removeprefix("group_")
        if base == "stats":
            tail = (E, R, 5)
        elif base == "quantiles":
            tail = (E, R, len(arg[0]))
        elif base == "covariance":
            tail = (E, 1 + len(arg[0]) + len(arg[0]) ** 2)
        else:
            tail = (sum((2 if len(planes) == 2 else 3) + int(np.prod(bins)) for _, planes, bins, _, _ in arg[0]),)
        tail = (self.n_groups,) + tail if kind != base else tail
        k = len(self.samples) if ring else 1
        r0 = self.rows_seen.get(kind, 0)
        self.rows_seen[kind] = r0 + k
        t = _named(kind, range(r0, r0 + k), tail)
        return t if ring else t[0]

    def extrema(self):
        return _named("extrema", [0], (self.n_worlds, self.n_entities, 25 + len(self.channel_records), 5))[0]

    def thresholds(self):
        return _named("thresholds", [0], (self.n_worlds, len(self.summary[1]), 26))[0]

    def moments(self):
        return _named("moments", [0], (self.n_worlds, self.n_entities, len(self.summary[2]), 3))[0]

    def dwells(self):
        return _named("dwells", [0], (self.n_worlds, len(self.summary[3]), 3))[0]


def _reduction(kind, ring):
    return lambda self, *arg: self._reduce(kind, ring, arg)


for _kind in _CODES:
    if _kind not in ("extrema", "thresholds", "moments", "dwells"):
        setattr(_RecordingFake, f"state_{_kind}", _reduction(_kind, False))
        setattr(_RecordingFake, f"trajectory_{_kind}", _reduction(_kind, True))


@pytest.mark.parametrize("route", ["resident", "host"])
def test_every_ensemble_option_at_once_with_a_fake_backend(monkeypatch, route):
    """One Exec with every ensemble option, on the resident route (ring-fulls of 2, 2 and 1 cycles, then a partial
    cycle) and on the invoke_batch route of a host system (two whole cycles, then a partial one): the exact sequence
    of backend calls, and every accessor's slice of tables whose values name their position."""
    from elodin_b200 import world as W

    monkeypatch.setattr(W, "B200Exec", _RecordingFake)
    chans = [SPEED, el.Norm("range", "world_pos", (4, 5)), el.AxisAngle("pitch", (-1, 0, 0), (0, 0, 1))]
    levels = [0.1, 0.5, 0.9]
    hists = [el.Histogram("ball.world_vel", 3, (-1.0, 1.0), 4),
             el.Histogram("rocket.channels", (0, 1), ((0.0, 1.0), (0.0, 2.0)), (2, 3))]
    M, E, R, G = 5, 2, 28, 3
    sys_ = el.six_dof() if route == "resident" else el.six_dof() | el.host_system(lambda ctx: None)
    ex = two_body_world().build(
        sys_, simulation_rate=120.0, telemetry_rate=40.0, n_worlds=M, ensemble=True, ensemble_ring=2, channels=chans,
        extrema=True, thresholds=[el.Threshold("rocket.channels", 1, below=0.0), el.Threshold("ball.world_pos", 4, above=1.0)],
        quantiles=levels, covariance=[("channels", (2, 0)), ("world_pos", (4,))], histograms=hists, groups=[2, 0, 3],
        retain=[4, 1], moments=[("world_pos", (6,)), ("channels", (1,))],
        dwells=[el.Threshold("rocket.world_pos", 6, below=2.0)])
    be = ex.backend
    ticks = 16 if route == "resident" else 8
    ex.run(ticks)

    hist_specs = [(1, (10,), (4,), (-1.0,), (1.0,)), (0, (25, 26), (2, 3), (0.0, 0.0), (1.0, 2.0))]
    args = {"stats": (), "quantiles": (levels,), "covariance": ([27, 25, 4],), "histograms": (hist_specs,)}
    order = ("stats", "quantiles", "covariance", "histograms", "group_stats", "group_histograms", "group_quantiles",
             "group_covariance")

    def rows(ring, worlds=True):
        src = "trajectory" if ring else "state"
        calls = [(f"{src}_{k}", *args[k.removeprefix("group_")]) for k in order]
        return calls + [(f"summary_add_{src}",)] + ([(f"{src}_worlds", [4, 1])] if worlds else [])

    uploads = [("upload", cid) for cid in be.input_ids]
    want = [("set_channels", [(1, 3), (1, 2), (2, 0)]),
            ("summary_begin", True, [(0, 26, False, 0.0), (1, 4, True, 1.0)], [6, 26], [(0, 6, False, 2.0)]),
            ("set_world_groups", [2, 0, 3])] + uploads + rows(False)
    if route == "resident":                                  # 5 whole cycles of 3 ticks, then one tick
        want += uploads
        for c in (2, 2, 1):
            want += [("reset",), ("step", 3 * c)] + rows(True)
        want += [("step", 1)] + rows(False)
        want += [("download", el.component_id(n)) for n in ("world_pos", "world_vel", "world_accel", "force")]
        n_rows = 7
    else:
        for n in (3, 3, 2):
            want += [("reset",)] + [("invoke", 1), ("step", 1)] * n + rows(n == 3, worlds=False)
        n_rows = 4
    assert _FakeBackend.calls == want
    assert ex.tick == ticks

    rows_ = np.arange(n_rows)
    for pair, e, lo, hi in (("ball.world_vel", 1, 7, 13), ("rocket.channels", 0, 25, 28), ("rocket.world_pos", 0, 0, 7)):
        t = _named("stats", rows_, (E, R, 5))[:, e, lo:hi]
        g = _named("group_stats", rows_, (G, E, R, 5))[:, :, e, lo:hi]
        for got, tab in ((ex.ensemble(pair), t), (ex.ensemble(pair, groups=True), g)):
            assert np.array_equal(got["count"], tab[..., 0]) and np.array_equal(got["mean"], tab[..., 1])
            assert np.array_equal(got["std"], np.sqrt(tab[..., 2] / tab[..., 0]))
            assert np.array_equal(got["min"], tab[..., 3]) and np.array_equal(got["max"], tab[..., 4])
        q = _named("quantiles", rows_, (E, R, 3))[:, e, lo:hi]
        assert np.array_equal(ex.quantiles(pair), q.transpose(0, 2, 1))
        q = _named("group_quantiles", rows_, (G, E, R, 3))[:, :, e, lo:hi]
        assert np.array_equal(ex.quantiles(pair, groups=True), q.transpose(0, 1, 3, 2))
        x = _named("extrema", [0], (M, E, R, 5))[0][:, e, lo:hi]
        got = ex.extrema(pair)
        assert np.array_equal(got["min"], x[..., 0]) and np.array_equal(got["max"], x[..., 1])
        for f, k in enumerate(("min_tick", "max_tick", "first_nonfinite_tick"), start=2):
            assert got[k].dtype == np.int64 and np.array_equal(got[k], x[..., f].astype(np.int64))
    for entity, e in (("rocket", 0), ("ball", 1)):
        for got, t in ((ex.covariance(entity), _named("covariance", rows_, (E, 13))[:, e]),
                       (ex.covariance(entity, groups=True), _named("group_covariance", rows_, (G, E, 13))[:, :, e])):
            assert got["planes"] == ["pitch", "speed", "world_pos[4]"]
            assert np.array_equal(got["count"], t[..., 0]) and np.array_equal(got["mean"], t[..., 1:4])
            assert np.array_equal(got["cov"], t[..., 4:].reshape(t.shape[:-1] + (3, 3)) / t[..., 0, None, None])
    for got, t in ((ex.histogram(0), _named("histograms", rows_, (15,))),
                   (ex.histogram(0, groups=True), _named("group_histograms", rows_, (G, 15)))):
        t = t.astype(np.int64)
        assert np.array_equal(got["counts"], t[..., 3:7]) and np.array_equal(got["nonfinite"], t[..., 0])
        assert np.array_equal(got["below"], t[..., 1]) and np.array_equal(got["above"], t[..., 2])
        assert np.array_equal(got["edges"], hists[0].edges)
    for got, t in ((ex.histogram(1), _named("histograms", rows_, (15,))),
                   (ex.histogram(1, groups=True), _named("group_histograms", rows_, (G, 15)))):
        t = t.astype(np.int64)
        assert np.array_equal(got["counts"], t[..., 9:15].reshape(t.shape[:-1] + (2, 3)))
        assert np.array_equal(got["nonfinite"], t[..., 7]) and np.array_equal(got["outside"], t[..., 8])
        assert all(np.array_equal(a, b) for a, b in zip(got["edges"], hists[1].edges))
    thr = _named("thresholds", [0], (M, 2, 26))[0]
    for i in range(2):
        got = ex.threshold(i)
        assert got["tick"].dtype == np.int64 and np.array_equal(got["tick"], thr[:, i, 0].astype(np.int64))
        for name, (lo, hi) in (("world_pos", (0, 7)), ("world_vel", (7, 13)), ("world_accel", (13, 19)), ("force", (19, 25))):
            assert np.array_equal(got[name], thr[:, i, 1 + lo:1 + hi])
    mom = _named("moments", [0], (M, E, 2, 3))[0]
    for pair, e, j, index in (("rocket.world_pos", 0, 0, 6), ("ball.channels", 1, 1, 1)):
        got = ex.moments(pair)
        n, mean, m2 = mom[:, e, [j], 0], mom[:, e, [j], 1], mom[:, e, [j], 2]
        assert list(got["index"]) == [index] and got["count"].dtype == np.int64
        assert np.array_equal(got["count"], n.astype(np.int64)) and np.array_equal(got["mean"], mean)
        assert np.array_equal(got["std"], np.sqrt(m2 / n)) and np.array_equal(got["rms"], np.sqrt(mean * mean + m2 / n))
    dw = _named("dwells", [0], (M, 1, 3))[0]
    got = ex.dwell(0)
    for f, k in enumerate(("rows", "first_tick", "last_tick")):
        assert got[k].dtype == np.int64 and np.array_equal(got[k], dw[:, 0, f].astype(np.int64))
    assert ex.retained == (4, 1) and ex.history_worlds("ball.world_pos").shape == (n_rows, 2, 7)
    assert ex.history_worlds("ball.inertia").shape == (n_rows, 2, 7)
    assert [r[0] for r in ex._globals_hist] == ([0, 3, 6, 9, 12, 15, 16] if route == "resident" else [0, 3, 6, 8])


# --------------------------------------------------------------------------- GPU helpers


def special_rows(M, E, seed):
    """[M, E, 25] rows: random non-unit quaternions and spread vectors, then rows with zero vectors, NaN, +-inf,
    squares that overflow and signed zeros."""
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (M, E, 25)) * rng.uniform(0.1, 50.0, (M, E, 1))
    x[..., :4] *= rng.uniform(0.2, 5.0, (M, E, 1))
    flat = np.zeros((10, 25)) if M * E < 10 else x.reshape(-1, 25)  # one body: only the random row
    flat[0, 7:13] = 0.0                          # at rest: atan2(0, 0) = 0, speed 0
    flat[1, 10] = np.nan
    flat[2, 4] = np.inf
    flat[3, 16] = -np.inf
    flat[4, 10:13] = (3e160, -2e160, 1e160)      # squares overflow: +inf
    flat[5, 10:13] = (-0.0, 0.0, -0.0)
    flat[5, 4:7] = (1.5, -2.0, -0.0)             # range 0 from the centre, alt -0.75 ...
    flat[6, :4] = (0.0, 0.0, 0.0, 0.0)           # a zero quaternion: NaN angles
    flat[7, 0] = np.nan
    flat[8, 6] = -3.0                            # dz = |(-3) - (-3)| = 0
    flat[9, 4:7] = (1e-300, 1e-300, 1e-300)      # underflowing squares
    return x


def ring_handle(mode, M, E, cap, seed, **kw):
    """state_handle with a full ring of `cap` samples and the special rows as the initial state"""
    x = special_rows(M, E, seed)
    return state_handle(x, mode, trajectory_every=1, trajectory_capacity=cap, trajectory_full=True, **kw), x


# --------------------------------------------------------------------------- GPU: channel values


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M, E", [(1, 1), (37, 3), (1000, 2)])
def test_channel_values_match_the_restatement(mode, M, E):
    need_gpu()
    ex, x = ring_handle(mode, M, E, 3, seed=M + E)
    with ex:
        ex.set_channels(records())
        assert ex.n_channels == len(CHANNELS)
        want, angle = ref_channels(x)
        n0 = ex.timings()["kernel_launches"]
        check_values(ex.state_channels(), want, angle)
        assert ex.timings()["kernel_launches"] - n0 == 2  # the channel pass, then the transpose
        ex.step(3)
        ex.sync()
        rows = ex.trajectory()
        got = ex.trajectory_channels()
        assert got.shape == (3, M, E, len(CHANNELS))
        want, _ = ref_channels(rows)
        check_values(got, want, angle)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_rocket_channel_values(mode):
    """A thrusting rocket's rows (unit quaternions from the integrator, real speeds)"""
    need_gpu()
    ex, _ = handle(ROCKET, 500, 2, mode, capacity=5, seed=2)
    with ex:
        ex.set_channels(records())
        ex.step(5)
        ex.sync()
        want, angle = ref_channels(ex.trajectory())
        check_values(ex.trajectory_channels(), want, angle)


# --------------------------------------------------------------------------- GPU: reductions of channel planes


def finite(v):
    return v[np.isfinite(v)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_channel_quantiles_and_histograms_are_numpys(mode):
    need_gpu()
    M, E = 3000, 2
    ex, x = ring_handle(mode, M, E, 2, seed=9)
    with ex:
        ex.set_channels(records())
        ch = ex.state_channels()
        q = ex.state_quantiles(LEVELS)
        assert q.shape == (E, 25 + len(CHANNELS), len(LEVELS))
        for e in range(E):
            for k in range(len(CHANNELS)):
                v = finite(ch[:, e, k])
                np.testing.assert_array_equal(q[e, 25 + k], np.quantile(v, LEVELS))
        specs = [(1, 25, 40, 0.0, 60.0), (0, 30, 16, 0.0, np.pi), (1, (25, 30), (8, 6), (0.0, 0.0), (80.0, np.pi))]
        h = ex.state_histograms(specs)
        v0 = ch[:, 1, 0]
        assert np.array_equal(h[3:43], np.histogram(finite(v0), bins=40, range=(0.0, 60.0))[0])
        assert h[0] == np.sum(~np.isfinite(v0))
        v1 = ch[:, 0, 5]
        assert np.array_equal(h[46:62], np.histogram(finite(v1), bins=16, range=(0.0, np.pi))[0])
        a, b = ch[:, 1, 0], ch[:, 1, 5]
        ok = np.isfinite(a) & np.isfinite(b)
        h2 = np.histogram2d(a[ok], b[ok], bins=(8, 6), range=((0.0, 80.0), (0.0, np.pi)))[0]
        assert np.array_equal(h[62 + 2:], h2.ravel())
        ex.set_world_groups([1000, 0, 2000])
        gq = ex.state_group_quantiles(LEVELS)
        for g, (lo, hi) in enumerate(((0, 1000), (1000, 1000), (1000, 3000))):
            for k in range(len(CHANNELS)):
                v = finite(ch[lo:hi, 0, k])
                want = np.quantile(v, LEVELS) if v.size else np.full(len(LEVELS), np.nan)
                np.testing.assert_array_equal(gq[g, 0, 25 + k], want)
        gh = ex.state_group_histograms(specs[:1])
        assert np.array_equal(gh[2, 3:], np.histogram(finite(ch[1000:, 1, 0]), bins=40, range=(0.0, 60.0))[0])


def _uploaded(ch, x, n_c):
    """x with the channel values in planes 0 .. n_c - 1 (world_pos, then world_vel)"""
    y = x.copy()
    y[..., :n_c] = ch
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_channel_stats_and_covariance_equal_a_handle_holding_the_values(mode):
    """Same values in the same shape give the same chunking and the same bits, plain and grouped"""
    need_gpu()
    M, E, n_c = 20_001, 2, len(CHANNELS)
    sizes = [3000, 0, 9000, 8001]
    ex, x = ring_handle(mode, M, E, 1, seed=11)
    with ex:
        ex.set_channels(records())
        ch = ex.state_channels()
        ex.set_world_groups(sizes)
        with state_handle(_uploaded(ch, x, n_c), mode) as ref:
            ref.set_world_groups(sizes)
            a, b = ex.state_stats(), ref.state_stats()
            assert a[:, 25:].tobytes() == b[:, :n_c].tobytes()
            a, b = ex.state_group_stats(), ref.state_group_stats()
            assert a[:, :, 25:].tobytes() == b[:, :, :n_c].tobytes()
            for sel_a, sel_b in (([25, 26, 30], [0, 1, 5]), ([32, 27], [7, 2])):
                assert ex.state_covariance(sel_a).tobytes() == ref.state_covariance(sel_b).tobytes()
                assert ex.state_group_covariance(sel_a).tobytes() == ref.state_group_covariance(sel_b).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_ring_tables_equal_the_state_route_sample_by_sample(mode):
    need_gpu()
    ex, _ = handle(ROCKET, 3000, 2, mode, capacity=3, seed=6)
    with ex:
        ex.set_channels(records())
        ex.set_world_groups([1000, 2000])
        specs = [(0, 25, 20, 0.0, 40.0), (1, (26, 30), (5, 5), (0.0, 0.0), (5e3, np.pi))]
        sel = [25, 4, 30]
        per = []
        for _ in range(3):
            ex.step(1)
            ex.sync()
            per.append((ex.state_stats(), ex.state_quantiles(LEVELS), ex.state_covariance(sel), ex.state_histograms(specs),
                        ex.state_group_stats(), ex.state_group_quantiles(LEVELS), ex.state_group_covariance(sel),
                        ex.state_group_histograms(specs), ex.state_channels()))
        ring = (ex.trajectory_stats(), ex.trajectory_quantiles(LEVELS), ex.trajectory_covariance(sel),
                ex.trajectory_histograms(specs), ex.trajectory_group_stats(), ex.trajectory_group_quantiles(LEVELS),
                ex.trajectory_group_covariance(sel), ex.trajectory_group_histograms(specs), ex.trajectory_channels())
        for s in range(3):
            for t, st in zip(ring, per[s]):
                assert t[s].tobytes() == st.tobytes()


# --------------------------------------------------------------------------- GPU: planes 0-24 keep their bits


def _all_tables(ex, sel, specs, ring):
    pre = "trajectory" if ring else "state"
    out = {}
    for kind, args in (("stats", ()), ("quantiles", (LEVELS,)), ("covariance", (sel,)), ("histograms", (specs,)),
                       ("group_stats", ()), ("group_quantiles", (LEVELS,)), ("group_covariance", (sel,)),
                       ("group_histograms", (specs,))):
        t = getattr(ex, f"{pre}_{kind}")(*args)
        if kind in ("stats", "quantiles", "group_stats", "group_quantiles"):
            t = np.ascontiguousarray(t[..., :25, :])
        out[kind] = t.tobytes()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_raw_planes_keep_their_bits_with_channels(mode):
    need_gpu()
    sel, specs = [4, 5, 10, 24], [(0, 6, 30, -5.0, 5.0), (1, (4, 5), (7, 7), (-3.0, -3.0), (3.0, 3.0))]
    thr = [(0, 6, False, 0.9), (1, 10, True, 0.0)]
    got = {}
    for arm in ("none", "channels", "cleared"):
        ex, _ = handle(ROCKET, 5000, 2, mode, capacity=4, seed=8)
        with ex:
            if arm != "none":
                ex.set_channels(records())
            if arm == "cleared":
                ex.set_channels([])
                assert ex.n_channels == 0
            ex.set_world_groups([1234, 0, 3766])
            ex.summary_begin(True, thr)
            ex.summary_add_state()
            ex.step(4)
            ex.sync()
            ex.summary_add_trajectory()
            t = _all_tables(ex, sel, specs, True)
            t.update({f"state_{k}": v for k, v in _all_tables(ex, sel, specs, False).items()})
            t["extrema"] = np.ascontiguousarray(ex.extrema()[..., :25, :]).tobytes()
            t["thresholds"] = ex.thresholds().tobytes()
            if arm != "channels":  # the full tables of the cleared handle are today's bytes
                t["full_stats"] = ex.trajectory_stats().tobytes()
                t["full_extrema"] = ex.extrema().tobytes()
            got[arm] = t
    for k, v in got["none"].items():
        assert got["cleared"][k] == v, k
        if not k.startswith("full_"):
            assert got["channels"][k] == v, k


# --------------------------------------------------------------------------- GPU: run summaries of channel planes


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_extrema_and_thresholds_of_channels_are_a_numpy_fold(mode):
    need_gpu()
    M, E, S = 700, 2, 6
    ex, _ = handle(ROCKET, M, E, mode, capacity=S, seed=3)
    with ex:
        ex.set_channels(records())
        # speed above 17 m/s, range below 400 m, pitch above 1.2 rad
        thr = [(0, 25, True, 17.0), (1, 26, False, 400.0), (0, 30, True, 1.2)]
        ex.summary_begin(True, thr)
        t0 = ex.tick
        ex.summary_add_state()
        rows = [ex.state_channels()]
        full = [sampled_state(ex)]
        ex.step(S)
        ex.sync()
        ex.summary_add_trajectory()
        rows += list(ex.trajectory_channels())
        full += list(ex.trajectory())
        v = np.stack(rows)  # [S + 1, M, E, n_c]
        x = np.stack(full)  # [S + 1, M, E, 25]
        ticks = t0 + np.arange(S + 1)
        ext = ex.extrema()
        assert ext.shape == (M, E, 25 + len(CHANNELS), 5)
        fin = np.isfinite(v)
        vmin, vmax = np.where(fin, v, np.inf), np.where(fin, v, -np.inf)
        any_f = fin.any(0)
        mn, mx = vmin.min(0), vmax.max(0)
        e = ext[:, :, 25:]
        assert np.array_equal(e[..., 0], np.where(any_f, mn, np.nan), equal_nan=True)
        assert np.array_equal(e[..., 1], np.where(any_f, mx, np.nan), equal_nan=True)
        assert np.array_equal(e[..., 2], np.where(any_f, ticks[np.argmin(vmin, 0)], -1))
        assert np.array_equal(e[..., 3], np.where(any_f, ticks[np.argmax(vmax, 0)], -1))
        nf = ~fin
        assert np.array_equal(e[..., 4], np.where(nf.any(0), ticks[np.argmax(nf, 0)], -1))
        th = ex.thresholds()
        for i, (ent, plane, above, val) in enumerate(thr):
            c = v[:, :, ent, plane - 25]
            fire = c > val if above else c < val
            first = np.argmax(fire, 0)
            fired = fire.any(0)
            assert np.array_equal(th[:, i, 0], np.where(fired, ticks[first], -1))
            want = x[first, np.arange(M), ent]  # the 25 raw planes at the firing row
            assert np.array_equal(th[fired, i, 1:], want[fired])
            assert np.all(np.isnan(th[~fired, i, 1:]))


# --------------------------------------------------------------------------- GPU: the C ABI


@pytest.mark.gpu
def test_set_channels_refusals_leave_the_setting_unchanged():
    need_gpu()
    good = records()[:2]
    N = _lib.CHANNEL_NORM
    A = _lib.CHANNEL_AXIS_ANGLE
    cases = [
        ([_lib.channel(N, 1, (0,))] * 9, "9 channels: at most 8"),
        ([_lib.channel(7, 1, (0,))], "channel 0: unknown kind 7"),
        ([_lib.channel(N, 0)], "channel 0: a norm of 0 planes, 1 to 3"),
        ([_lib.channel(N, 4, (0, 1, 2))], "channel 0: a norm of 4 planes, 1 to 3"),
        ([_lib.channel(N, 2, (3, 25))], "channel 0: plane 25, a row has 25"),
        ([_lib.channel(N, 3, (10, 11, 10))], "channel 0: plane 10 twice"),
        ([_lib.channel(N, 1, (4,), (np.nan,))], "channel 0: offset 0 is not finite"),
        ([_lib.channel(N, 1, (4,), (), (), np.inf)], "channel 0: r0 is not finite"),
        ([_lib.channel(A, 1, (10,), (1, 0, 0))], r"channel 0: an axis angle takes n = 0 \(fixed direction\) or 3"),
        ([_lib.channel(A, 3, (23,), (1, 0, 0))], r"channel 0: planes 23 .. 25 run past plane 24"),
        ([_lib.channel(A, 0, (), (0, 0, 0), (0, 0, 1))], "channel 0: the body axis is zero"),
        ([_lib.channel(A, 0, (), (1, np.inf, 0), (0, 0, 1))], "channel 0: the body axis is not finite"),
        ([_lib.channel(A, 0, (), (1, 0, 0), (0, 0, 0))], "channel 0: the direction is zero"),
        ([_lib.channel(A, 0, (), (1, 0, 0), (np.nan, 0, 1))], "channel 0: the direction is not finite"),
        ([good[0], _lib.channel(N, 1, (4,))], None),  # valid: placeholder replaced below
    ]
    bad_reserved = _lib.channel(N, 1, (4,))
    bad_reserved.reserved = 1
    cases[-1] = ([good[0], bad_reserved], "channel 1: reserved field is not 0")
    x = special_rows(64, 2, 1)
    with state_handle(x, "exact", trajectory_every=1, trajectory_capacity=2, trajectory_full=True) as ex:
        ex.set_channels(good)
        before = ex.state_channels()
        for recs, msg in cases:
            with pytest.raises(el.B200Error, match=msg) as e:
                ex.set_channels(recs)
            assert e.value.code == _lib.ERR_INVALID_ARGUMENT
            assert ex.n_channels == 2
        assert ex.state_channels().tobytes() == before.tobytes()
        ex.summary_begin(True)
        with pytest.raises(el.B200Error, match="set_channels after b200_sixdof_summary_begin"):
            ex.set_channels([])
        assert ex.n_channels == 2
        with pytest.raises(el.B200Error, match="threshold 0: plane 27, a row has 27"):
            ex.summary_begin(False, [(0, 27, True, 0.0)])
    with state_handle(x, "exact", trajectory_every=1, trajectory_capacity=2, trajectory_full=False) as ex:
        with pytest.raises(el.B200Error, match="B200_TRAJ_FULL trajectory ring: this one is 13 wide"):
            ex.set_channels(good)
    with state_handle(x, "exact") as ex:  # no ring: allowed
        ex.set_channels(good)
        assert ex.state_channels().shape == (64, 2, 2) and ex.trajectory_channels().shape == (0, 64, 2, 2)
        with pytest.raises(el.B200Error, match="covariance plane 0 is 27: the state has 27 planes"):
            ex.state_covariance([27])
        with pytest.raises(el.B200Error, match="covariance plane 0 is 25: the trajectory has 0 planes"):
            ex.trajectory_covariance([25])
        with pytest.raises(el.B200Error, match="histogram 0: plane 27, the state has 27 planes"):
            ex.state_histograms([(0, 27, 4, 0.0, 1.0)])
    L = _lib.lib()
    assert L.b200_sixdof_set_channels(None, None, 0) == _lib.ERR_INVALID_ARGUMENT
    assert L.b200_sixdof_channels(None) == 0


@pytest.mark.gpu
def test_launch_counts():
    """The channel pass runs before stats, quantiles and extrema whenever there are channels, and before covariance,
    histograms and thresholds only when they read a channel plane"""
    need_gpu()
    x = special_rows(500, 2, 4)
    with state_handle(x, "exact") as ex, state_handle(x, "exact") as ref:
        ex.set_channels(records()[:3])

        def launches(h, call):
            n0 = h.timings()["kernel_launches"]
            call(h)
            return h.timings()["kernel_launches"] - n0

        for call, extra in ((lambda h: h.state_stats(), 1), (lambda h: h.state_quantiles(LEVELS), 1),
                            (lambda h: h.state_covariance([4, 5]), 0), (lambda h: h.state_histograms([(0, 4, 8, 0, 1)]), 0)):
            assert launches(ex, call) == launches(ref, call) + extra
        assert launches(ex, lambda h: h.state_covariance([4, 26])) == launches(ref, lambda h: h.state_covariance([4, 5])) + 1
        assert launches(ex, lambda h: h.state_histograms([(0, 25, 8, 0, 1)])) == \
            launches(ref, lambda h: h.state_histograms([(0, 4, 8, 0, 1)])) + 1
        ex.summary_begin(False, [(0, 4, True, 0.0)])
        ref.summary_begin(False, [(0, 4, True, 0.0)])
        assert launches(ex, lambda h: h.summary_add_state()) == launches(ref, lambda h: h.summary_add_state())
    with state_handle(x, "exact") as ex, state_handle(x, "exact") as ref:
        ex.set_channels(records()[:3])
        ex.summary_begin(True)
        ref.summary_begin(True)
        assert launches(ex, lambda h: h.summary_add_state()) == launches(ref, lambda h: h.summary_add_state()) + 1


# --------------------------------------------------------------------------- GPU: Exec


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_exec_channels_equal_the_restatement_of_a_default_mode_exec(mode):
    need_gpu()
    M = 256
    w, sys_, params = rocket_world(M)
    chans = [el.Norm("speed", "world_vel", (3, 4, 5)), el.Norm("range", "world_pos", (4, 5)),
             el.AxisAngle("pitch", (-1.0, 0.0, 0.0), (0.0, 0.0, 1.0))]
    kw = dict(simulation_rate=120.0, telemetry_rate=30.0, math=mode, n_worlds=M, world_params=params)
    ens = w.build(sys_, **kw, ensemble=True, ensemble_ring=3, channels=chans, quantiles=LEVELS, extrema=True,
                  thresholds=[el.Threshold("rocket.channels", 0, above=5.0)],
                  histograms=[el.Histogram("rocket.channels", 0, range=(0.0, 40.0), bins=20)],
                  covariance=[("channels", (0, 1)), ("world_pos", (6,))])
    ens.run(40)
    ref = w.build(sys_, **kw)
    ref.run(40)
    rows = np.concatenate([ref.history_worlds(f"rocket.{c}") for c in ("world_pos", "world_vel")], -1)  # [T, M, 13]
    full = np.zeros(rows.shape[:-1] + (25,))
    full[..., :13] = rows
    sp, rg = norm_channel(full, (10, 11, 12)), norm_channel(full, (4, 5))
    s, t = angle_parts(full, (-1.0, 0.0, 0.0), d=(0.0, 0.0, 1.0))
    pitch = np.arctan2(s, t)
    q = ens.quantiles("rocket.channels")  # [rows, n_q, 3]
    assert q.shape == (rows.shape[0], len(LEVELS), 3)
    for r in range(rows.shape[0]):
        np.testing.assert_array_equal(q[r, :, 0], np.quantile(sp[r], LEVELS))
        np.testing.assert_array_equal(q[r, :, 1], np.quantile(rg[r], LEVELS))
        want = np.quantile(pitch[r], LEVELS)
        assert np.all(np.abs(q[r, :, 2] - want) <= ATAN2_ULP * np.spacing(np.abs(want)))
    st = ens.ensemble("rocket.channels")
    assert np.array_equal(st["max"][:, 0], sp.max(1)) and np.array_equal(st["min"][:, 1], rg.min(1))
    e = ens.extrema("rocket.channels")
    assert np.array_equal(e["max"][:, 0], sp.max(0))
    h = ens.histogram(0)
    assert np.array_equal(h["counts"][-1], np.histogram(sp[-1], bins=20, range=(0.0, 40.0))[0])
    assert ens.covariance("rocket")["planes"] == ["speed", "range", "world_pos[6]"]
    assert ens.channels == ["speed", "range", "pitch"]
    fire = sp > 5.0
    ticks = np.arange(rows.shape[0]) * ens.ticks_per_telemetry
    assert np.array_equal(ens.threshold(0)["tick"], np.where(fire.any(0), ticks[np.argmax(fire, 0)], -1))


# --------------------------------------------------------------------------- GPU: two gloo ranks

GLOO_M, GLOO_SIZES = 6001, [2000, 4001]


def _gloo_worker(rank, ws):
    from elodin_b200.sharding import gather_covariance, gather_ensemble, gather_histograms, shard_groups, shard_worlds

    w0, w1 = shard_worlds(GLOO_M, rank, ws)
    x = special_rows(GLOO_M, 2, 21)[w0:w1]
    with state_handle(np.ascontiguousarray(x), "exact") as ex:
        ex.set_channels(records())
        ex.set_world_groups(shard_groups(GLOO_SIZES, rank, ws))
        return (gather_ensemble(ex.state_stats()), gather_covariance(ex.state_covariance([25, 26, 31])),
                gather_histograms(ex.state_histograms([(0, 25, 16, 0.0, 80.0)])),
                gather_covariance(ex.state_group_covariance([25, 30])))


@pytest.mark.gpu
def test_two_gloo_ranks_merge_channel_tables():
    need_gpu()
    got = run_gloo(_gloo_worker, 2)
    x = special_rows(GLOO_M, 2, 21)
    with state_handle(x, "exact") as ex:
        ex.set_channels(records())
        ex.set_world_groups(GLOO_SIZES)
        hist = ex.state_histograms([(0, 25, 16, 0.0, 80.0)])
        cov = ex.state_covariance([25, 26, 31])
        st = ex.state_stats()
        gcov = ex.state_group_covariance([25, 30])
    for r in got:
        assert np.array_equal(r[2], hist)
        np.testing.assert_allclose(r[0], st, rtol=1e-12, equal_nan=True)
        np.testing.assert_allclose(r[1], cov, rtol=1e-9, atol=1e-9, equal_nan=True)
        np.testing.assert_allclose(r[3], gcov, rtol=1e-9, atol=1e-9, equal_nan=True)
        assert r[0].shape == st.shape and r[0][0, 25:, 0].tolist() == st[0, 25:, 0].tolist()  # counts exact
