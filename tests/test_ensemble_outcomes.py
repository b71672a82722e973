"""Outcomes of a Monte-Carlo batch: one value per world from the run summaries, a device column or host values
(b200_sixdof_set_outcomes, outcome_kernels.cu), reduced over the worlds by the existing ensemble reductions.

The CPU tests check every el.Outcome / outcomes= refusal before the handle exists, the struct and constants against
the header, the backend calls of an Exec with and without outcomes, and the value rules on hand tables against a
numpy restatement.  The GPU tests, in both math modes, hold outcome_values to the per-world tables of a rocket
campaign on both Exec routes and any ring size, every outcome table to the state table of a one-entity handle whose
planes hold the outcome values (and to numpy), group g to a handle over exactly its worlds, two halves merged to the
whole, and the refusals of the C ABI."""

import ctypes
import os
import subprocess

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200.executor import INERTIA, TICK, WORLD_POS, WORLD_VEL
from tests.ensemble_util import ROCKET, handle, need_gpu, no_device, rocket_world, two_body_world  # noqa: F401
from tests.test_ensemble_channels import _named, _RecordingFake
from tests.test_ensemble_histograms import state_handle
from tests.test_host_logic import _FakeBackend

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("exact", "fast")
LEVELS = (0.0, 0.01, 0.25, 0.5, 0.99, 1.0)
O = el.Outcome


# --------------------------------------------------------------------------- the numpy restatement of the value rules


def never_nan(ticks):
    """A tick field as an outcome: -1 ("never") is NaN."""
    t = np.array(ticks, dtype=np.float64)
    t[t == -1.0] = np.nan
    return t


def moment_outcomes(rec):
    """(count, mean, std, rms) of moment records [..., 3] = (n, mean, m2): Exec.moments' numpy operations."""
    n, mean, m2 = rec[..., 0], rec[..., 1], rec[..., 2]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        var = m2 / n
        return n, mean, np.sqrt(var), np.sqrt(mean * mean + var)


def bits(x):
    """f64 bits with every NaN made the same NaN (payloads are not part of the contract)."""
    x = np.array(x, dtype=np.float64)
    x[np.isnan(x)] = np.nan
    return x.view(np.uint64)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


# --------------------------------------------------------------------------- CPU: refusals before the handle


@pytest.mark.parametrize("make, exc, match", [
    (lambda: O("", "rocket.world_pos", 6, "max"), ValueError, "non-empty string"),
    (lambda: O("a", "rocket.world_pos", 7, "max"), ValueError, r"index 7 is not an integer in \[0, 7\)"),
    (lambda: O("a", "rocket.world_pos", 6, "median"), ValueError, "field 'median' is none of"),
    (lambda: O("a", "rocket.inertia", 6, "max"), _lib.B200ValueError, "component not found: rocket.inertia"),
    (lambda: O("a", "inertia", 6), _lib.B200ValueError, "component not found"),
    (lambda: O("a", "rocket.inertia", -1), ValueError, "not a non-negative integer"),
    (lambda: O.threshold("a", 0, "world_pos"), ValueError, "with an index"),
    (lambda: O.threshold("a", 0, "tick", 3), ValueError, "with an index"),
    (lambda: O.threshold("a", 0, "world_vel", 6), ValueError, r"\[0, 6\)"),
    (lambda: O.threshold("a", -1, "tick"), ValueError, "not a non-negative integer"),
    (lambda: O.dwell("a", 0, "ticks"), ValueError, "field 'ticks' is none of"),
    (lambda: O.values("a", [[1.0, 2.0]]), ValueError, "1-D array"),
    (lambda: O.values("a", ["x"]), ValueError, "1-D array of numbers"),
])
def test_outcome_constructors_refuse(make, exc, match):
    with pytest.raises(exc, match=match):
        make()


TWO = dict(n_worlds=4)


@pytest.mark.parametrize("kw, exc, match", [
    (dict(outcomes=[O("a", "rocket.inertia", 6)]), _lib.B200Error, r"^outcomes: need World.build\(..., ensemble=True\)"),
    (dict(ensemble=True, outcomes=[O("a", "rocket.world_pos", 6, "max")]), _lib.B200Error, "extrema=True"),
    (dict(ensemble=True, moments=[("world_pos", (5,))], outcomes=[O("a", "rocket.world_pos", 6, "rms")]),
     _lib.B200Error, r"moments=\[...\] selecting rocket.world_pos\[6\]"),
    (dict(ensemble=True, extrema=True, outcomes=[O("a", "rocket.channels", 0, "max")]), ValueError,
     "channel 0, this Exec has 0"),
    (dict(ensemble=True, thresholds=[el.Threshold("rocket.world_pos", 6, below=0.0)],
          outcomes=[O.threshold("a", 1, "tick")]), ValueError, "threshold 1, this Exec has 1"),
    (dict(ensemble=True, outcomes=[O.dwell("a", 0, "rows")]), ValueError, "dwell 0, this Exec has 0"),
    (dict(ensemble=True, outcomes=[O.values("a", np.zeros(3))]), ValueError, "3 values, this Exec has 4 worlds"),
    (dict(ensemble=True, outcomes=[O("a", "rocket.thrust", 0)]), _lib.B200ValueError,
     "component not found: rocket.thrust"),
    (dict(ensemble=True, outcomes=[O("a", "rocket.inertia", 7)]), ValueError, "index 7, rocket.inertia has 7"),
    (dict(ensemble=True, outcomes=[O("a", "nosuch.inertia", 0)]), _lib.B200ValueError, "component not found: nosuch"),
    (dict(ensemble=True, extrema=True, outcomes=[O("a", "nosuch.world_pos", 0, "min")]), _lib.B200ValueError,
     "component not found: nosuch.world_pos"),
    (dict(ensemble=True, outcomes=[O("a", "rocket.inertia", 6), O("a", "ball.inertia", 6)]), ValueError,
     "the name 'a' is used twice"),
    (dict(ensemble=True, outcomes=[O(f"m{k}", "rocket.inertia", 6) for k in range(26)]), ValueError,
     "26 outcomes: 1 to 25"),
    (dict(ensemble=True, outcomes=[]), ValueError, "0 outcomes: 1 to 25"),
    (dict(ensemble=True, outcomes=O("a", "rocket.inertia", 6)), TypeError, "outcomes take a sequence"),
    (dict(ensemble=True, outcomes=[("a", "rocket.inertia", 6)]), TypeError, "outcomes take el.Outcome objects"),
])
def test_build_refuses_outcomes_before_the_device(no_device, kw, exc, match):  # noqa: F811
    with pytest.raises(exc, match=match):
        two_body_world().build(el.six_dof(), **TWO, **kw)


def test_outcomes_come_last_in_the_ensemble_check(no_device):  # noqa: F811
    with pytest.raises(_lib.B200Error, match=r"^extrema, outcomes: need World.build"):
        two_body_world().build(el.six_dof(), extrema=True, outcomes=[O("a", "rocket.inertia", 6)])
    with pytest.raises(ValueError, match=r"^groups: need World.build"):  # unchanged
        two_body_world().build(el.six_dof(), groups=[1])


def test_valid_outcomes_reach_the_handle(no_device):  # noqa: F811
    outs = [O("apogee", "rocket.world_pos", 6, "max"), O("t", "rocket.world_pos", 6, "first_nonfinite_tick"),
            O("rms", "ball.channels", 0, "rms"), O("mass", "rocket.inertia", 6), O("z", "ball.world_pos", 6),
            O.threshold("t_hit", 0, "tick"), O.threshold("x_hit", 0, "world_pos", 4), O.dwell("settle", 0, "last_tick"),
            O.values("gain", np.arange(4))]
    with pytest.raises(AssertionError, match="handle is created"):
        two_body_world().build(el.six_dof(), n_worlds=4, ensemble=True, extrema=True,
                               channels=[el.Norm("speed", "world_vel", (3, 4, 5))], moments=[("channels", (0,))],
                               thresholds=[el.Threshold("rocket.world_pos", 6, below=0.0)],
                               dwells=[el.Threshold("rocket.world_pos", 6, above=1.0)], outcomes=outs)


# --------------------------------------------------------------------------- CPU: the C struct and constants


def test_outcome_struct_matches_header(tmp_path):
    st = _lib.Outcome
    assert ctypes.sizeof(st) == 40
    names = ("MAX_OUTCOMES", "OUTCOME_EXTREMA", "OUTCOME_THRESHOLD", "OUTCOME_MOMENT", "OUTCOME_DWELL",
             "OUTCOME_COLUMN", "OUTCOME_VALUES")
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200_sixdof.h"', 'int main(void) {',
           'printf("size %zu\\n", sizeof(b200_outcome));']
    src += [f'printf("{n} %u\\n", (unsigned)B200_{n});' for n in names]
    src += [f'printf("{f} %zu\\n", offsetof(b200_outcome, {f}));' for f, _ in st._fields_]
    src += ["return 0; }"]
    c = tmp_path / "outcome.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "outcome"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", str(c), "-I", os.path.join(ROOT, "include"), "-o", str(exe)],
                   check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(st)
    for n in names:
        assert int(got[n]) == getattr(_lib, n), n
    assert _lib.MAX_OUTCOMES == _lib.MAX_COV_PLANES
    for f, _ in st._fields_:
        assert int(got[f]) == getattr(st, f).offset, f


# --------------------------------------------------------------------------- CPU: backend calls through a fake


class _OutcomeFake(_RecordingFake):
    """The recording fake with the outcome calls: set_outcomes logged, outcome tables named like the others."""

    def set_outcomes(self, recs):
        self.n_out = len(recs)
        self._log("set_outcomes", [tuple(r[:5]) for r in recs])

    def outcome_stats(self):
        return _named("stats", [0], (self.n_out, 5))[0]

    def outcome_group_stats(self):
        return _named("group_stats", [0], (self.n_groups, self.n_out, 5))[0]

    def outcome_quantiles(self, q):
        return _named("quantiles", [0], (self.n_out, len(q)))[0]

    def outcome_covariance(self, planes):
        self._log("outcome_covariance", list(planes))
        return _named("covariance", [0], (1 + len(planes) + len(planes) ** 2,))[0]

    def outcome_histograms(self, specs):
        self._log("outcome_histograms", [tuple(np.asarray(v).tolist() if isinstance(v, tuple) else v for v in s)
                                         for s in specs])
        return _named("histograms", [0], (3 + specs[0][2][0],))[0]


def _calls(monkeypatch, **kw):
    from elodin_b200 import world as W

    monkeypatch.setattr(W, "B200Exec", _OutcomeFake)
    _FakeBackend.calls = []
    ex = two_body_world().build(el.six_dof(), simulation_rate=120.0, telemetry_rate=40.0, n_worlds=5, ensemble=True,
                                ensemble_ring=2, extrema=True, thresholds=[el.Threshold("rocket.world_pos", 6, below=0.0)],
                                groups=[2, 3], **kw)
    ex.run(7)
    return ex, list(_FakeBackend.calls)


def test_an_exec_with_outcomes_adds_only_set_outcomes_after_summary_begin(monkeypatch):
    _, plain = _calls(monkeypatch)
    gain = np.arange(5.0)
    outs = [O("apogee", "rocket.world_pos", 6, "max"), O("mass", "ball.inertia", 6), O.threshold("t", 0, "tick"),
            O.values("gain", gain)]
    ex, calls = _calls(monkeypatch, outcomes=outs)
    k = [c[0] for c in calls].index("set_outcomes")
    assert calls[k - 1][0] == "summary_begin" and calls[k + 1][0] == "set_world_groups"
    assert calls[k] == ("set_outcomes", [(_lib.OUTCOME_EXTREMA, 1, 6, 0), (_lib.OUTCOME_COLUMN, 6, 0, 1, "inertia"),
                                         (_lib.OUTCOME_THRESHOLD, 0, 0), (_lib.OUTCOME_VALUES, 0, 0, 0, 0)])
    assert calls[:k] + calls[k + 1:] == plain
    assert ex.outcomes == ["apogee", "mass", "t", "gain"]

    st = _named("stats", [0], (4, 5))[0]
    got = ex.outcome_stats()
    assert np.array_equal(got["count"], st[:, 0]) and np.array_equal(got["max"], st[:, 4])
    assert np.array_equal(got["std"], np.sqrt(st[:, 2] / st[:, 0]))
    g = _named("group_stats", [0], (2, 4, 5))[0]
    assert np.array_equal(ex.outcome_stats(groups=True)["mean"], g[..., 1])
    q = ex.outcome_quantiles([0.1, 0.9])
    assert np.array_equal(q, _named("quantiles", [0], (4, 2))[0].T)
    cov = ex.outcome_covariance(["gain", "apogee"])
    assert _FakeBackend.calls[-1] == ("outcome_covariance", [3, 0]) and cov["planes"] == ["gain", "apogee"]
    c = _named("covariance", [0], (7,))[0]
    assert np.array_equal(cov["mean"], c[1:3]) and np.array_equal(cov["cov"], c[3:].reshape(2, 2) / c[0])
    h = ex.outcome_histogram("t", (0.0, 30.0), bins=3)
    assert _FakeBackend.calls[-1] == ("outcome_histograms", [(0, [2], [3], [0.0], [30.0])])
    t = _named("histograms", [0], (6,))[0].astype(np.int64)
    assert np.array_equal(h["counts"], t[3:]) and h["below"] == t[1] and np.array_equal(h["edges"], np.linspace(0, 30, 4))
    with pytest.raises(ValueError, match="no finite, strictly increasing edges"):
        ex.outcome_histogram("t", (1.0, 1.0))
    with pytest.raises(_lib.B200ValueError, match="outcome not found: 'nosuch'"):
        ex.outcome_covariance(["nosuch"])


def test_accessors_without_outcomes_are_refused(monkeypatch):
    ex, _ = _calls(monkeypatch)
    for call, msg in ((ex.outcome_values, r"outcome_values\(\): build the Exec with World.build\(..., ensemble=True, "
                                          r"outcomes=\[...\]\)"),
                      (lambda: ex.outcome_stats(groups=True), r"outcome_stats\(groups=True\)"),
                      (lambda: ex.outcome_quantiles(0.5), "outcome_quantiles"),
                      (lambda: ex.outcome_histogram("a", (0, 1)), "outcome_histogram")):
        with pytest.raises(_lib.B200Error, match=msg) as e:
            call()
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT


def test_value_rules_on_hand_tables():
    """-1 ticks are NaN, every other field keeps its bits, and std / rms are Exec.moments' bits."""
    ext = np.array([[3.5, -0.0, 7.0, -1.0, -1.0], [np.nan, np.nan, -1.0, -1.0, 4.0]])
    assert same(never_nan(ext[:, 2:]), [[7.0, np.nan, np.nan], [np.nan, np.nan, 4.0]])
    assert bits(ext[:, 1])[0] == bits(-0.0)  # a signed zero keeps its sign
    rec = np.array([[3.0, 1.0 / 3.0, 2.0 / 7.0], [0.0, np.nan, np.nan], [5.0, 1e200, np.inf], [1.0, -2.5, 0.0]])
    n, mean, std, rms = moment_outcomes(rec)
    assert same(std, [np.sqrt((2.0 / 7.0) / 3.0), np.nan, np.inf, 0.0])
    assert same(rms, [np.sqrt((1.0 / 3.0) * (1.0 / 3.0) + (2.0 / 7.0) / 3.0), np.nan, np.inf, 2.5])


def test_moment_restatement_equals_exec_moments(monkeypatch):
    """The restatement the device is held to gives Exec.moments' std and rms bit for bit."""
    ex, _ = _calls(monkeypatch, moments=[("world_vel", (5,))])
    got = ex.moments("rocket.world_vel")
    rec = _named("moments", [0], (5, 2, 1, 3))[0][:, 0, 0]
    _, _, std, rms = moment_outcomes(rec)
    assert same(got["std"][:, 0], std) and same(got["rms"][:, 0], rms)


# --------------------------------------------------------------------------- GPU: a rocket campaign


def campaign(M, math, route, ring=None, groups=None):
    w, sys_, params = rocket_world(M)
    params["inertia"][1, 0, 6] = np.nan  # world 1 diverges
    if route == "host":
        sys_ = sys_ | el.host_system(lambda ctx: None)
    gain = np.linspace(0.5, 1.5, M)
    outs = [O("apogee", "rocket.world_pos", 6, "max"), O("t_apogee", "rocket.world_pos", 6, "max_tick"),
            O("t_nan", "rocket.world_pos", 6, "first_nonfinite_tick"), O("xmin", "rocket.world_pos", 4, "min"),
            O("t_xmin", "rocket.world_pos", 4, "min_tick"),
            O.threshold("t_hit", 0, "tick"), O.threshold("x_hit", 0, "world_pos", 4), O.threshold("q_hit", 0, "world_pos", 0),
            O.threshold("f_hit", 0, "force", 5), O.threshold("t_never", 1, "tick"),
            O("vz_n", "rocket.world_vel", 5, "count"), O("vz_mean", "rocket.world_vel", 5, "mean"),
            O("vz_std", "rocket.world_vel", 5, "std"), O("vz_rms", "rocket.world_vel", 5, "rms"),
            O.dwell("rows", 0, "rows"), O.dwell("first", 0, "first_tick"), O.dwell("last", 0, "last_tick"),
            O("mass", "rocket.inertia", 6), O("thrust", "rocket.thrust", 0), O("wind", "rocket.wind", 0),
            O("z_final", "rocket.world_pos", 6), O("vx_ball", "ball.world_vel", 3), O.values("gain", gain),
            O("ball_max", "ball.world_pos", 4, "max"), O("spd", "rocket.channels", 0, "max")]
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=40.0, n_worlds=M, math=math, world_params=params,
                 ensemble=True, ensemble_ring=ring, extrema=True, groups=groups,
                 channels=[el.Norm("speed", "world_vel", (3, 4, 5))],
                 thresholds=[el.Threshold("rocket.world_pos", 6, below=1.0), el.Threshold("rocket.world_pos", 6, above=1e9)],
                 moments=[("world_vel", (5,))], dwells=[el.Threshold("rocket.world_pos", 6, above=1.05)], outcomes=outs)
    ex.run(60)
    return ex, params, gain


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("route", ["resident", "host"])
def test_outcome_values_equal_the_per_world_tables(math, route):
    need_gpu()
    M = 37
    ex, params, gain = campaign(M, math, route)
    v = ex.outcome_values()
    x = ex.extrema("rocket.world_pos")
    assert same(v["apogee"], x["max"][:, 6]) and same(v["xmin"], x["min"][:, 4])
    for name, f, p in (("t_apogee", "max_tick", 6), ("t_nan", "first_nonfinite_tick", 6), ("t_xmin", "min_tick", 4)):
        assert same(v[name], never_nan(x[f][:, p])), name
    assert v["t_nan"][1] >= 0 and np.isnan(v["t_nan"][0])  # world 1 diverges after its initial row
    t0, t1 = ex.threshold(0), ex.threshold(1)
    assert same(v["t_hit"], never_nan(t0["tick"])) and same(v["x_hit"], t0["world_pos"][:, 4])
    assert same(v["q_hit"], t0["world_pos"][:, 0]) and same(v["f_hit"], t0["force"][:, 5])
    assert np.isnan(v["t_hit"][1]) and np.all(np.isnan(v["t_never"]))
    m = ex.moments("rocket.world_vel")
    assert same(v["vz_n"], m["count"][:, 0]) and same(v["vz_mean"], m["mean"][:, 0])
    assert same(v["vz_std"], m["std"][:, 0]) and same(v["vz_rms"], m["rms"][:, 0])
    d = ex.dwell(0)
    assert same(v["rows"], d["rows"]) and same(v["first"], never_nan(d["first_tick"]))
    assert same(v["last"], never_nan(d["last_tick"]))
    assert same(v["mass"], params["inertia"][:, 0, 6]) and same(v["thrust"], params["thrust"][:, 0, 0])
    assert same(v["wind"], params["wind"][:, 0, 0]) and same(v["gain"], gain)
    state = ex.backend.download(WORLD_POS)
    assert same(v["z_final"], state[:, 0, 6]) and same(v["vx_ball"], ex.backend.download(WORLD_VEL)[:, 1, 3])
    assert same(v["ball_max"], ex.extrema("ball.world_pos")["max"][:, 4])
    assert same(v["spd"], ex.extrema("rocket.channels")["max"][:, 0])
    # the same for any ring size
    ex1, _, _ = campaign(M, math, route, ring=1)
    v1 = ex1.outcome_values()
    assert all(same(v[k], v1[k]) for k in v)
    # the tables: the reductions of these values (the oracle itself is test_tables_equal_a_one_entity_state_handle)
    st = ex.outcome_stats()
    assert st["count"][ex.outcomes.index("t_never")] == 0 and st["count"][ex.outcomes.index("mass")] == M - 1
    assert st["count"][ex.outcomes.index("t_hit")] == np.sum(np.isfinite(v["t_hit"]))


def _state_of(values):
    """[M, 1, 25] state rows whose first P planes are the outcome values [M, P] (the rest 0)."""
    M, P = values.shape
    x = np.zeros((M, 1, 25))
    x[:, 0, :P] = values
    return x


def _random_values(M, P, seed):
    rng = np.random.default_rng(seed)
    v = rng.normal(0.0, 1.0, (M, P)) * rng.uniform(0.1, 100.0, (1, P))
    v[rng.random((M, P)) < 0.05] = np.nan
    v[rng.random((M, P)) < 0.01] = np.inf
    v[:, 1] = np.round(v[:, 1])          # ties
    if M > 3:
        v[:3, 2] = -0.0
    return v


def _specs(P):
    return [(0, (0,), (16,), (-50.0,), (50.0,)), (0, (1, 3), (5, 7), (-3.0, -40.0), (3.0, 40.0)),
            (0, (P - 1,), (1,), (-1.0,), (1.0,))]


def _values_handle(values, math, E=1, groups=None, groups_first=False):
    """A handle of E entities whose outcomes are `values` [M, P]: COLUMN outcomes of the last entity's world_pos,
    world_vel and inertia planes (the values written there), then VALUES outcomes; `groups` set after the outcomes, or
    before them with `groups_first`."""
    M, P = values.shape
    x = np.zeros((M, E, 25))
    ine = np.tile(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 1))
    n_col = min(P, 14)
    x[:, E - 1, :13] = values[:, :13] if n_col >= 13 else np.pad(values[:, :n_col], ((0, 0), (0, 13 - n_col)))
    if n_col == 14:
        ine[:, E - 1, 6] = values[:, 13]
    ex = el.B200Exec(E, M, 0.01, None, [], "rk4", math)
    ex.set_state(x[..., :7], x[..., 7:13], ine)
    outs = [(_lib.OUTCOME_COLUMN, k if k < 7 else k - 7, 0, E - 1, WORLD_POS if k < 7 else WORLD_VEL) for k in range(min(n_col, 13))]
    if n_col == 14:
        outs.append((_lib.OUTCOME_COLUMN, 6, 0, E - 1, INERTIA))
    outs += [(_lib.OUTCOME_VALUES, 0, 0, 0, 0, values[:, k]) for k in range(n_col, P)]
    if groups is not None and groups_first:
        ex.set_world_groups(groups)
    ex.set_outcomes(outs)
    if groups is not None and not groups_first:
        ex.set_world_groups(groups)
    return ex


def _launches(ex, call):
    n0 = ex.timings()["kernel_launches"]
    got = call()
    return got, ex.timings()["kernel_launches"] - n0


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
@pytest.mark.parametrize("M", [1, 255, 256, 257, 8192, 8193])
def test_tables_equal_a_one_entity_state_handle(math, M):
    need_gpu()
    P = 25
    values = _random_values(M, P, seed=M)
    ex = _values_handle(values, math, E=3 if M in (257, 8193) else 1)
    st = state_handle(_state_of(values), math)
    assert same(ex.outcome_values(), values)
    (got, n_out), (want, n_st) = _launches(ex, ex.outcome_stats), _launches(st, st.state_stats)
    assert same(got, want[0, :P]) and n_out == n_st + 1  # + the value pass
    q = ex.outcome_quantiles(LEVELS)
    assert same(q, st.state_quantiles(LEVELS)[0, :P])
    for k in range(P):
        fin = values[:, k][np.isfinite(values[:, k])]
        ref = np.quantile(fin, LEVELS) if fin.size else np.full(len(LEVELS), np.nan)
        assert np.array_equal(np.abs(q[k]), np.abs(ref), equal_nan=True), k  # numpy may order -0 / +0 either way
    sel = list(range(P))[::-1]
    assert same(ex.outcome_covariance(sel), st.state_covariance(sel)[0])
    h = ex.outcome_histograms(_specs(P))
    assert same(h, st.state_histograms(_specs(P)))
    fin = values[:, 0][np.isfinite(values[:, 0])]
    assert np.array_equal(h[3:19], np.histogram(fin, 16, (-50.0, 50.0))[0])
    both = np.isfinite(values[:, 1]) & np.isfinite(values[:, 3])
    h2 = np.histogram2d(values[both, 1], values[both, 3], (5, 7), ((-3.0, 3.0), (-40.0, 40.0)))[0]
    assert np.array_equal(h[19 + 2:19 + 2 + 35].reshape(5, 7), h2)
    # grouped: the same bits as the state's grouped tables
    sizes = [0, M // 3, M - M // 3] if M > 1 else [1]
    ex.set_world_groups(sizes)
    st.set_world_groups(sizes)
    assert same(ex.outcome_group_stats(), st.state_group_stats()[:, 0, :P])
    assert same(ex.outcome_group_quantiles(LEVELS), st.state_group_quantiles(LEVELS)[:, 0, :P])
    assert same(ex.outcome_group_covariance(sel), st.state_group_covariance(sel)[:, 0])
    assert same(ex.outcome_group_histograms(_specs(P)), st.state_group_histograms(_specs(P)))


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_group_tables_equal_a_handle_over_the_group(math):
    need_gpu()
    M, P, sizes = 9000, 6, [0, 300, 57, 8643]
    values = _random_values(M, P, seed=3)
    ex = _values_handle(values, math, E=3, groups=sizes)
    sel = [4, 0, 2]
    g = (ex.outcome_group_stats(), ex.outcome_group_quantiles(LEVELS), ex.outcome_group_covariance(sel),
         ex.outcome_group_histograms(_specs(P)))
    # groups set before the outcomes: set_outcomes builds the one-entity group tables itself
    first = _values_handle(values, math, E=3, groups=sizes, groups_first=True)
    for a, b in zip(g, (first.outcome_group_stats(), first.outcome_group_quantiles(LEVELS),
                        first.outcome_group_covariance(sel), first.outcome_group_histograms(_specs(P)))):
        assert same(a, b)
    w0 = 0
    for k, n in enumerate(sizes):
        if n:
            sub = _values_handle(values[w0:w0 + n], math, E=2)
            want = (sub.outcome_stats(), sub.outcome_quantiles(LEVELS), sub.outcome_covariance(sel),
                    sub.outcome_histograms(_specs(P)))
            for a, b in zip(g, want):
                assert same(a[k], b), k
        else:
            assert np.all(g[0][k][:, 0] == 0) and np.all(np.isnan(g[1][k])) and np.all(g[3][k] == 0)
        w0 += n


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_halves_merge_into_the_whole(math):
    need_gpu()
    M, P = 4099, 5
    values = _random_values(M, P, seed=11)
    whole = _values_handle(values, math)
    a, b = _values_handle(values[:2000], math), _values_handle(values[2000:], math)
    st = el.merge_stats([a.outcome_stats(), b.outcome_stats()])
    want = whole.outcome_stats()
    assert np.array_equal(st[:, [0, 3, 4]], want[:, [0, 3, 4]], equal_nan=True)
    assert np.allclose(st[:, 1:3], want[:, 1:3], rtol=1e-11, atol=0)
    sel = [0, 2, 4]
    cv = el.merge_covariance([a.outcome_covariance(sel), b.outcome_covariance(sel)])
    cw = whole.outcome_covariance(sel)
    assert cv[0] == cw[0] and np.allclose(cv[1:], cw[1:], rtol=1e-11, atol=1e-9)
    hs = el.merge_histograms([a.outcome_histograms(_specs(P)), b.outcome_histograms(_specs(P))])
    assert np.array_equal(hs, whole.outcome_histograms(_specs(P)))


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_index_7_entity_2_and_channel_extrema(math):
    """Threshold and dwell 7, outcomes on entity 2 of 3, and extrema of a channel plane, against the downloads."""
    need_gpu()
    M, N = 300, 3
    ex, _ = handle(ROCKET, M, N, math, capacity=4, seed=5)
    ex.set_channels([_lib.channel(_lib.CHANNEL_NORM, 3, (10, 11, 12))])
    conds = [(k % N, 4 + k % 3, k % 2 == 0, 0.5 * k - 1.0) for k in range(8)]
    ex.summary_begin(True, conds, moments=[25, 6], dwells=conds[::-1])
    for _ in range(5):
        ex.step(3)
        ex.summary_add_state()
    outs = [(_lib.OUTCOME_THRESHOLD, 0, 7), (_lib.OUTCOME_THRESHOLD, 5, 7), (_lib.OUTCOME_DWELL, 0, 7),
            (_lib.OUTCOME_DWELL, 1, 7), (_lib.OUTCOME_DWELL, 2, 7), (_lib.OUTCOME_EXTREMA, 1, 25, 2),
            (_lib.OUTCOME_EXTREMA, 4, 25, 2), (_lib.OUTCOME_EXTREMA, 2, 5, 2), (_lib.OUTCOME_MOMENT, 3, 0, 2),
            (_lib.OUTCOME_MOMENT, 2, 1, 1), (_lib.OUTCOME_COLUMN, 0, 0, 2, "thrust"), (_lib.OUTCOME_COLUMN, 2, 0, 2, "wind")]
    ex.set_outcomes(outs)
    v = ex.outcome_values()
    thr, dw, ext, mom = ex.thresholds(), ex.dwells(), ex.extrema(), ex.moments()
    assert same(v[:, 0], never_nan(thr[:, 7, 0])) and same(v[:, 1], thr[:, 7, 5])
    assert same(v[:, 2], dw[:, 7, 0]) and same(v[:, 3], never_nan(dw[:, 7, 1])) and same(v[:, 4], never_nan(dw[:, 7, 2]))
    assert same(v[:, 5], ext[:, 2, 25, 1]) and same(v[:, 6], never_nan(ext[:, 2, 25, 4]))
    assert same(v[:, 7], never_nan(ext[:, 2, 5, 2]))
    assert same(v[:, 8], moment_outcomes(mom[:, 2, 0])[3]) and same(v[:, 9], moment_outcomes(mom[:, 1, 1])[2])
    assert same(v[:, 10], ex.download(el.component_id("thrust"))[:, 2, 0])
    assert same(v[:, 11], ex.download(el.component_id("wind"))[:, 2, 2])


def _refused(call, code, match):
    with pytest.raises(_lib.B200Error, match=match) as e:
        call()
    assert e.value.code == code


@pytest.mark.gpu
def test_abi_refusals():
    need_gpu()
    M, N = 40, 2
    ex, _ = handle(ROCKET, M, N, "exact", capacity=2)
    INV = _lib.ERR_INVALID_ARGUMENT
    _refused(ex.outcome_stats, INV, "no outcomes: call b200_sixdof_set_outcomes first")
    _refused(lambda: ex.set_outcomes([(_lib.OUTCOME_EXTREMA, 1, 6, 0)]), INV, "outcome 0: the summary in force has no extrema")
    ex.summary_begin(True, [(0, 6, False, 0.0)])
    good = [(_lib.OUTCOME_THRESHOLD, 0, 0), (_lib.OUTCOME_EXTREMA, 1, 6, 1), (_lib.OUTCOME_VALUES, 0, 0, 0, 0, np.arange(M))]
    ex.set_outcomes(good)
    before = ex.outcome_values()
    bad = [
        ([(9, 0, 0)], INV, "outcome 0: unknown kind 9"),
        ([(_lib.OUTCOME_EXTREMA, 5, 6, 0)], INV, "outcome 0: field 5, kind 1 has fields 0 to 4"),
        ([(_lib.OUTCOME_EXTREMA, 0, 25, 0)], INV, "extrema plane 25, a row has 25"),
        ([(_lib.OUTCOME_EXTREMA, 0, 6, 2)], INV, "entity row 2"),
        ([(_lib.OUTCOME_THRESHOLD, 26, 0)], INV, "field 26"),
        ([(_lib.OUTCOME_THRESHOLD, 0, 0, 1)], INV, "its kind takes none"),
        ([(_lib.OUTCOME_THRESHOLD, 0, 1)], INV, "threshold 1, the summary in force has 1"),
        ([(_lib.OUTCOME_DWELL, 0, 0)], INV, "dwell 0, the summary in force has 0"),
        ([(_lib.OUTCOME_MOMENT, 0, 0)], INV, "moment slot 0, the summary in force has 0"),
        ([(_lib.OUTCOME_COLUMN, 0, 0, 0, TICK)], INV, "is global"),
        ([(_lib.OUTCOME_COLUMN, 7, 0, 0, INERTIA)], INV, "plane 7, the column has 7"),
        ([(_lib.OUTCOME_COLUMN, 0, 0, 0, 12345)], _lib.ERR_COMPONENT_NOT_FOUND, "component 0x0000000000003039 not found"),
        ([(_lib.OUTCOME_VALUES, 0, 0)], INV, "outcome 0: null values"),
        ([(_lib.OUTCOME_THRESHOLD, 0, 0, 0, 0, np.zeros(M))], INV, "values given"),
        ([(_lib.OUTCOME_COLUMN, 0, 1, 0, INERTIA)], INV, "index 1, a column outcome takes 0"),
        ([(_lib.OUTCOME_THRESHOLD, 0, 0)] * 26, INV, "26 outcomes: at most 25"),
    ]
    for outs, code, match in bad:
        _refused(lambda: ex.set_outcomes(outs), code, match)
    r = _lib.Outcome(_lib.OUTCOME_THRESHOLD, 0, 0, 1)
    _refused(lambda: ex.set_outcomes([r]), INV, "reserved field is not 0")
    assert ex.n_outcomes == 3 and same(ex.outcome_values(), before)  # the previous set stays in force
    # entry checks: bytes, histogram entity and plane, covariance plane
    _refused(lambda: ex._reduce("stats", "outcome", (), (3, 4)), _lib.ERR_VALUE_SIZE_MISMATCH, "outcome statistics are 120 bytes")
    _refused(lambda: ex.outcome_histograms([(1, (0,), (4,), (0.0,), (1.0,))]), INV, "histogram 0: entity 1 of 1")
    _refused(lambda: ex.outcome_histograms([(0, (3,), (4,), (0.0,), (1.0,))]), INV, "plane 3, the outcome has 3 planes")
    _refused(lambda: ex.outcome_covariance([0, 3]), INV, "covariance plane 1 is 3: the outcome has 3 planes")
    _refused(ex.outcome_group_stats, INV, "grouped outcome: call b200_sixdof_set_world_groups first")
    # a summary_start that drops the threshold an outcome names: every entry refuses, naming it
    ex.summary_begin(True)
    for call in (ex.outcome_values, ex.outcome_stats, lambda: ex.outcome_quantiles(0.5), lambda: ex.outcome_covariance([0]),
                 lambda: ex.outcome_histograms([(0, (0,), (4,), (0.0,), (1.0,))])):
        _refused(call, INV, "outcome 0: threshold 0, the summary in force has 0")
    ex.set_outcomes([])
    assert ex.n_outcomes == 0
    _refused(ex.outcome_values, INV, "no outcomes")
