"""Sobol indices of a Saltelli campaign (monte_carlo.saltelli, b200_sixdof_outcome_[group_]sobol, sobol_kernels.cu):
per group and output, the first-order and total indices from the covariance record of the derived planes, and the
bootstrap spreads of the restated draw stream.

The CPU tests check the constants and prototypes against the header, the design's layout and its order under
plan_groups, the numpy restatement of the estimator against SALib's raw formulas and against analytic indices, the
vectorised draw stream against Python integers, and every Exec refusal before the backend is reached.  The GPU tests
hold the point estimates bit for bit to executor.sobol_indices on the covariance of a handle whose worlds are the
samples, the spreads to a numpy bootstrap of the same draws, and check incomplete samples, the edges, groups against a
handle over their worlds, reproducibility, side effects, launches, the C ABI's refusals and the rocket campaign."""

import ctypes
import math
import os
import re
from statistics import NormalDist

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib, monte_carlo
from elodin_b200.executor import sobol_indices
from tests.ensemble_util import need_gpu, two_body_world
from tests.test_ensemble_outcomes import _OutcomeFake
from tests.test_host_logic import _FakeBackend
from tests.test_outcome_rank_correlation import _only_values, _refused, same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("exact", "fast")
GOLDEN = 0x9E3779B97F4A7C15
MASK = (1 << 64) - 1


# --------------------------------------------------------------------------- the numpy restatement


def mix_int(z: int) -> int:
    z ^= z >> 30
    z = (z * 0xBF58476D1CE4E5B9) & MASK
    z ^= z >> 27
    z = (z * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


def mix(z):
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = z ^ (z >> np.uint64(30))
        z = z * np.uint64(0xBF58476D1CE4E5B9)
        z = z ^ (z >> np.uint64(27))
        z = z * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def umulhi(x, n: int):
    """(x * n) >> 64 for uint64 x and 0 <= n < 2^32."""
    x = np.asarray(x, dtype=np.uint64)
    n = np.uint64(n)
    with np.errstate(over="ignore"):
        hi, lo = (x >> np.uint64(32)) * n, (x & np.uint64(0xFFFFFFFF)) * n
        return (hi + (lo >> np.uint64(32))) >> np.uint64(32)


def draws(seed: int, r: int, n: int):
    """The complete-list positions of resample r's n draws."""
    t = np.arange(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = mix(np.uint64(seed % (1 << 64)) + np.uint64(GOLDEN) * ((np.uint64(r) << np.uint64(32)) + t + np.uint64(1)))
    return umulhi(x, n).astype(np.int64)


def planes(y, d):
    """(a, b, D [N, d], complete [N]) of a Saltelli layout's values y [N (d + 2)]."""
    Y = np.asarray(y, dtype=np.float64).reshape(-1, d + 2)
    a, b = Y[:, 0], Y[:, -1]
    with np.errstate(invalid="ignore", over="ignore"):
        D = Y[:, 1:d + 1] - a[:, None]
    ok = np.isfinite(a) & np.isfinite(b) & np.all(np.isfinite(D), axis=1)
    return a, b, D, ok


def ref_bootstrap(y, d, B, seed, means):
    """(S1_sd [d], ST_sd [d], n_boot_ok) of the contract's bootstrap over y [N (d + 2)], shifted by the point record's
    means [d + 2]."""
    a, b, D, ok = planes(y, d)
    c = np.flatnonzero(ok)
    n = c.size
    S1 = np.full((B, d), np.nan)
    ST = np.full((B, d), np.nan)
    good = 0
    for r in range(B):
        if n == 0:
            continue
        j = c[draws(seed, r, n)]
        ap, bp, Dp = a[j] - means[0], b[j] - means[1], D[j] - means[2:]
        ea, eb = ap.sum() / n, bp.sum() / n
        va, vb = (ap * ap).sum() / n - ea * ea, (bp * bp).sum() / n - eb * eb
        dm = (means[0] + ea) - (means[1] + eb)
        V = (va + vb) * 0.5 + dm * dm * 0.25
        good += V > 0
        if n < 2 or not V > 0:
            continue
        eD = Dp.sum(0) / n
        mD = means[2:]
        EbD = (bp[:, None] * Dp).sum(0) / n + means[1] * eD + mD * eb + means[1] * mD
        EDD = (Dp * Dp).sum(0) / n + 2 * mD * eD + mD * mD
        S1[r], ST[r] = EbD / V, EDD / (2 * V)

    def sd(x):
        out = np.full(d, np.nan)
        for i in range(d):
            v = x[:, i][np.isfinite(x[:, i])]
            if v.size >= 2:
                out[i] = v.std(ddof=1)
        return out

    return sd(S1), sd(ST), good


def cov_record(y, d):
    """The covariance record [1 + q + q*q] of the derived planes in numpy (for the CPU tests)."""
    a, b, D, ok = planes(y, d)
    P = np.column_stack([a, b, D])[ok]
    n = P.shape[0]
    m = P.mean(0) if n else np.full(d + 2, np.nan)
    M = (P - m).T @ (P - m) if n else np.full((d + 2, d + 2), np.nan)
    return np.concatenate([[n], m, M.ravel()])


def ishigami(X, a=7.0, b=0.1):
    return np.sin(X[:, 0]) + a * np.sin(X[:, 1]) ** 2 + b * X[:, 2] ** 4 * np.sin(X[:, 0])


ISHIGAMI_S1 = np.array([0.3139, 0.4424, 0.0])
ISHIGAMI_ST = np.array([0.5576, 0.4424, 0.2437])


def ishigami_spec(n, method="random", seed=3):
    u = {"dist": "uniform", "min": -math.pi, "max": math.pi}
    return {"monte_carlo": {"n_samples": n, "method": method, "seed": seed,
                            "variables": {"x1": u, "x2": u, "x3": u, "z": {"dist": "fixed", "value": 1.5}}}}


def design_X(design):
    return np.array([[r[f"param.{k}"] for k in design.inputs] for r in design.rows])


def layout(A, B):
    """The Saltelli layout [N (d + 2), d] of base matrices A, B [N, d] in numpy."""
    N, d = A.shape
    X = np.repeat(A[:, None, :], d + 2, axis=1)
    X[:, -1] = B
    for i in range(d):
        X[:, 1 + i, i] = B[:, i]
    return X.reshape(-1, d)


def record_split(t, d):
    return t[..., 0], t[..., 1], t[..., 2], t[..., 3:3 + d], t[..., 3 + d:3 + 2 * d], t[..., 3 + 2 * d:3 + 3 * d], \
        t[..., 3 + 3 * d:]


# --------------------------------------------------------------------------- CPU


def test_header_constants_and_prototypes():
    h = open(os.path.join(ROOT, "include", "b200_sixdof.h")).read()
    for name in ("b200_sixdof_outcome_sobol", "b200_sixdof_outcome_group_sobol"):
        m = re.search(name + r"\(([^)]*)\)", h)
        assert m and len(m.group(1).split(",")) == 8, name
        assert name in _lib.SYMBOLS
    assert int(re.search(r"#define B200_MAX_SOBOL_INPUTS (\d+)u", h).group(1)) == _lib.MAX_SOBOL_INPUTS == 23
    assert int(re.search(r"#define B200_MAX_SOBOL_RESAMPLES (\d+)u", h).group(1)) == _lib.MAX_SOBOL_RESAMPLES == 10000
    assert monte_carlo.MAX_SOBOL_INPUTS == _lib.MAX_SOBOL_INPUTS == _lib.MAX_COV_PLANES - 2
    L = _lib.lib()
    for name in ("sobol", "group_sobol"):
        fn = getattr(L, f"b200_sixdof_outcome_{name}")
        assert len(fn.argtypes) == 8 and fn.argtypes[2:5] == [ctypes.c_uint32] * 3
        assert fn.argtypes[5] is ctypes.c_uint64 and fn.argtypes[7] is ctypes.c_uint64


def test_design_layout_and_order():
    spec = {"sim_sweep": {"gain": [0.9, 1.1]}, "meta_sweep": {"label": ["a", "b"]},
            "monte_carlo": {"n_samples": 5, "method": "lhs", "seed": 11, "variables": {
                "m": {"dist": "uniform", "min": 1, "max": 2}, "c": {"dist": "fixed", "value": 4.0},
                "k": {"dist": "normal", "mean": 0, "std": 2}, "ch": {"dist": "choice", "values": [1, 2, 3]},
                "lg": {"dist": "loguniform", "min": 1e-3, "max": 1.0}}}}
    des = monte_carlo.saltelli(spec)
    assert des.inputs == ["ch", "k", "lg", "m"] and des.n_base == 5
    d, q = 4, 6
    assert len(des.rows) == 2 * 2 * 5 * q
    for i, r in enumerate(des.rows):
        assert r["run_id"] == f"run_{i:07}" and r["seed"] == i + 1 and r["param.c"] == 4.0
    X = design_X(des).reshape(4, 5, q, d)
    for p in range(4):
        for j in range(5):
            A, B = X[p, j, 0], X[p, j, -1]
            for i in range(d):
                want = A.copy()
                want[i] = B[i]
                assert np.array_equal(X[p, j, 1 + i], want)
        assert np.array_equal(X[p], X[0])  # the same samples at every sweep point
    # the sweep x meta x block order of materialize, and plan_groups by the sim key keeps it
    pts = [(r["param.gain"], r["meta.label"]) for r in des.rows[::5 * q]]
    assert pts == [(0.9, "a"), (0.9, "b"), (1.1, "a"), (1.1, "b")]
    rows, sizes, keys = monte_carlo.plan_groups(des.rows, ["param.gain"])
    assert rows == des.rows and sizes == [2 * 5 * q] * 2 and keys == [{"param.gain": 0.9}, {"param.gain": 1.1}]
    assert monte_carlo.saltelli(spec) == des
    # the unit samples are materialize's draws of 2d columns: A and B map them through each distribution
    import random
    units = monte_carlo._unit_samples(5, 2 * d, "lhs", random.Random(11))
    variables = spec["monte_carlo"]["variables"]
    for j in range(5):
        for i, k in enumerate(des.inputs):
            assert X[0, j, 0, i] == monte_carlo._draw(variables[k], units[j][i])
            assert X[0, j, -1, i] == monte_carlo._draw(variables[k], units[j][d + i])
    other = monte_carlo.saltelli(spec, n_base=3)
    assert other.n_base == 3 and len(other.rows) == 4 * 3 * q
    rnd = monte_carlo.saltelli(ishigami_spec(4))
    assert rnd.inputs == ["x1", "x2", "x3"] and len(rnd.rows) == 20 and all(r["param.z"] == 1.5 for r in rnd.rows)


def test_design_refusals_and_materialize_unchanged(tmp_path):
    import json

    fixed = {"monte_carlo": {"n_samples": 4, "variables": {"a": {"dist": "fixed", "value": 1}}}}
    with pytest.raises(ValueError, match=r"no dispersed .*\['a'\]"):
        monte_carlo.saltelli(fixed)
    with pytest.raises(ValueError, match="no dispersed"):
        monte_carlo.saltelli({})
    many = {"monte_carlo": {"variables": {f"v{k:02}": {"dist": "uniform", "min": 0, "max": 1} for k in range(24)}}}
    with pytest.raises(ValueError, match=r"24 dispersed variables \['v00'.*at most 23"):
        monte_carlo.saltelli(many)
    with pytest.raises(ValueError, match=r"n_base must be >= 1 \(got 0\) for the inputs \['x1', 'x2', 'x3'\]"):
        monte_carlo.saltelli(ishigami_spec(4), n_base=0)
    with pytest.raises(ValueError, match="missing"):
        monte_carlo.saltelli({"monte_carlo": {"variables": {"u": {"dist": "uniform", "min": 0}}}})
    import tomllib

    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "mc_plans.json")))
    for name, case in golden.items():  # materialize still gives the reference's plans byte for byte
        path = os.path.join(str(tmp_path), f"{name}.csv")
        spec = tomllib.loads(case["spec"])
        monte_carlo.write_plan(monte_carlo.materialize(spec), path)
        assert open(path).read() == case["plan_csv"], name
        variables = (spec.get("monte_carlo") or {}).get("variables", {})
        dispersed = sum(str(v.get("dist", "fixed")) != "fixed" for v in variables.values())
        if dispersed > 23:
            with pytest.raises(ValueError, match=f"{dispersed} dispersed variables"):
                monte_carlo.saltelli(spec)
        elif dispersed:
            des = monte_carlo.saltelli(spec, n_base=2)
            plain = monte_carlo.materialize(spec)
            assert len(des.rows) * len(plain) // len(des.rows) == len(plain)
            assert len(des.rows) == len(plain) // int(spec["monte_carlo"].get("n_samples", 1)) * 2 * (len(des.inputs) + 2)


def salib(fA, fB, fAB):
    """SALib's raw first-order (Saltelli 2010) and total (Jansen) formulas."""
    V = np.var(np.r_[fA, fB])
    return np.mean(fB[:, None] * (fAB - fA[:, None]), axis=0) / V, 0.5 * np.mean((fA[:, None] - fAB) ** 2, axis=0) / V


def _analytic(X, f, d, S1, ST, boot=100):
    y = f(X)
    rec = cov_record(y, d)
    n, V, s1, st = sobol_indices(rec, d)
    Y = y.reshape(-1, d + 2)
    w1, wt = salib(Y[:, 0], Y[:, -1], Y[:, 1:d + 1])
    assert np.allclose(s1, w1, rtol=0, atol=1e-12) and np.allclose(st, wt, rtol=0, atol=1e-12)
    sd1, sdt, good = ref_bootstrap(y, d, boot, 5, rec[1:d + 3])
    assert good == boot
    z = NormalDist().inv_cdf(0.975)
    assert np.all(np.abs(s1 - S1) <= 3 * z * sd1 + 1e-3), (s1, S1, sd1)
    assert np.all(np.abs(st - ST) <= 3 * z * sdt + 1e-3), (st, ST, sdt)


def test_restated_estimator_on_analytic_cases():
    des = monte_carlo.saltelli(ishigami_spec(1 << 12))
    _analytic(design_X(des), ishigami, 3, ISHIGAMI_S1, ISHIGAMI_ST)
    c = np.array([1.0, 2.0, 0.5, 3.0])
    share = c ** 2 / np.sum(c ** 2)
    u = {"dist": "normal", "mean": 0.0, "std": 1.0}
    spec = {"monte_carlo": {"n_samples": 1 << 12, "method": "lhs", "seed": 2, "variables": {f"x{i}": u for i in range(4)}}}
    _analytic(design_X(monte_carlo.saltelli(spec)), lambda X: 10.0 + X @ c, 4, share, share)
    # the contract's edges: n < 2 and a constant output
    one = cov_record(np.arange(5.0), 3)
    n, V, s1, st = sobol_indices(one, 3)
    assert n == 1 and np.isnan(V) and np.all(np.isnan(s1)) and np.all(np.isnan(st))
    n, V, s1, st = sobol_indices(cov_record(np.full(50, 2.0), 3), 3)
    assert n == 10 and V == 0 and np.all(np.isnan(s1)) and np.all(np.isnan(st))


def test_draw_stream_vectorised_equals_python_integers():
    for n in (1, 2, 7, 1000, (1 << 31) + 11, (1 << 32) - 1):
        for seed in (0, 12345, (1 << 64) - 1):
            for r in (0, 1, 9999):
                t = min(n, 64)
                got = draws(seed, r, n)[:t] if n < 4096 else _draws_head(seed, r, n, t)
                want = [(mix_int((seed + GOLDEN * ((r << 32) + k + 1)) & MASK) * n) >> 64 for k in range(t)]
                assert got.tolist() == want, (n, seed, r)
    assert int(mix(np.uint64(1))) == mix_int(1)


def _draws_head(seed, r, n, t):
    k = np.arange(t, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = mix(np.uint64(seed) + np.uint64(GOLDEN) * ((np.uint64(r) << np.uint64(32)) + k + np.uint64(1)))
    return umulhi(x, n).astype(np.int64)


class _SobolFake(_OutcomeFake):
    def outcome_sobol(self, planes, d, n_boot, seed):
        self._log("outcome_sobol", [list(planes), d, n_boot, seed])
        return np.tile(np.arange(3 + 4 * d, dtype=np.float64), (len(planes), 1))

    def outcome_group_sobol(self, planes, d, n_boot, seed):
        self._log("outcome_group_sobol", [list(planes), d, n_boot, seed])
        return np.tile(np.arange(3 + 4 * d, dtype=np.float64), (self.n_groups, len(planes), 1))


O = el.Outcome
OUTS = [O("apogee", "rocket.world_pos", 6, "max"), O.threshold("t", 0, "tick"), O.values("gain", np.arange(10.0))]


def _exec(monkeypatch, **kw):
    from elodin_b200 import world as W

    monkeypatch.setattr(W, "B200Exec", _SobolFake)
    _FakeBackend.calls = []
    args = dict(simulation_rate=120.0, telemetry_rate=40.0, n_worlds=10, ensemble=True, ensemble_ring=2, extrema=True,
                thresholds=[el.Threshold("rocket.world_pos", 6, below=0.0)])
    args.update(kw)
    ex = two_body_world().build(el.six_dof(), **args)
    ex.run(7)
    return ex


def test_exec_refusals_before_any_backend_call(monkeypatch):
    ex = _exec(monkeypatch, outcomes=OUTS, groups=[5, 5])
    n0 = len(_FakeBackend.calls)
    ins = ["x", "y", "z"]  # d = 3: blocks of 5 worlds
    cases = [
        (lambda: ex.outcome_sobol([], ["apogee"]), ValueError, "1 to 23 distinct names"),
        (lambda: ex.outcome_sobol(["x", "x"], ["apogee"]), ValueError, "1 to 23 distinct names"),
        (lambda: ex.outcome_sobol([f"v{k}" for k in range(24)], ["apogee"]), ValueError, "1 to 23 distinct"),
        (lambda: ex.outcome_sobol(ins, []), ValueError, "1 to 25 distinct outcome names"),
        (lambda: ex.outcome_sobol(ins, ["t", "t"]), ValueError, "1 to 25 distinct outcome names"),
        (lambda: ex.outcome_sobol(ins, ["nosuch"]), _lib.B200ValueError, "outcome not found: 'nosuch'"),
        (lambda: ex.outcome_sobol(ins, ["t"], bootstrap=-1), ValueError, r"bootstrap = -1, an int in \[0, 10000\]"),
        (lambda: ex.outcome_sobol(ins, ["t"], bootstrap=10001), ValueError, "bootstrap = 10001"),
        (lambda: ex.outcome_sobol(ins, ["t"], bootstrap=True), ValueError, "bootstrap = True"),
        (lambda: ex.outcome_sobol(ins, ["t"], level=1.0), ValueError, r"level = 1.0, a number in \(0, 1\)"),
        (lambda: ex.outcome_sobol(ins, ["t"], level=0), ValueError, "level = 0"),
        (lambda: ex.outcome_sobol(ins, ["t"], seed=1.5), TypeError, "seed = 1.5, an int"),
        (lambda: ex.outcome_sobol(["x"], ["t"]), ValueError, "blocks of 3 worlds, but the batch has 10 worlds"),
        (lambda: ex.outcome_sobol(["x", "y"], ["t"], groups=True), ValueError, "blocks of 4 worlds, but a group has 5"),
    ]
    for call, exc, match in cases:
        with pytest.raises(exc, match=match):
            call()
    assert len(_FakeBackend.calls) == n0
    plain = _exec(monkeypatch, outcomes=OUTS)
    with pytest.raises(_lib.B200Error, match=r"outcome_sobol\(groups=True\).*groups=\[...\]"):
        plain.outcome_sobol(ins, ["t"], groups=True)
    ex._pg = object()
    n0 = len(_FakeBackend.calls)
    with pytest.raises(_lib.B200Error, match="world-sharded campaign are not supported") as e:
        ex.outcome_sobol(ins, ["t"])
    assert e.value.code == _lib.ERR_UNSUPPORTED and len(_FakeBackend.calls) == n0


def test_an_exec_that_never_asks_makes_the_same_calls(monkeypatch):
    _exec(monkeypatch, outcomes=OUTS, groups=[5, 5])
    before = list(_FakeBackend.calls)
    assert not any("sobol" in c[0] for c in before)
    ex = _exec(monkeypatch, outcomes=OUTS, groups=[5, 5])
    assert _FakeBackend.calls == before
    s = ex.outcome_sobol(["x", "y", "z"], ["gain", "apogee"], bootstrap=7, level=0.9, seed=-1)
    assert _FakeBackend.calls == before + [("outcome_sobol", [[2, 0], 3, 7, -1])]
    z = NormalDist().inv_cdf(0.95)
    assert s["S1"].shape == (2, 3) and np.all(s["S1"] == [3, 4, 5]) and np.all(s["ST"] == [6, 7, 8])
    assert np.allclose(s["S1_conf"], z * np.array([9, 10, 11])) and np.allclose(s["ST_conf"], z * np.array([12, 13, 14]))
    assert np.all(s["count"] == 0) and np.all(s["var"] == 1) and s["inputs"] == ["x", "y", "z"]
    g = ex.outcome_sobol(["x", "y", "z"], "t", groups=True, bootstrap=0)
    assert _FakeBackend.calls[-1] == ("outcome_group_sobol", [[1], 3, 0, 0])
    assert g["S1"].shape == (2, 1, 3) and g["count"].shape == (2, 1) and g["outputs"] == ["t"]


# --------------------------------------------------------------------------- GPU


def _values_handle(y, math_mode="exact", groups=None):
    y = np.asarray(y, dtype=np.float64)
    return _only_values(y if y.ndim == 2 else y[:, None], math_mode, groups)


def _check_point(ex, t, Y, d, sizes=None):
    """t [G or none, p, rec] equals sobol_indices of the outcome covariance of a handle whose VALUES outcomes are the
    derived planes of Y [W, p], with n_worlds = samples and the same groups, bit for bit."""
    p = Y.shape[1]
    recs = []
    for k in range(p):
        a, b, D, ok = planes(Y[:, k], d)
        P = np.column_stack([a, b, D])
        P[~ok] = np.nan
        h = _values_handle(P, "exact", None if sizes is None else [s // (d + 2) for s in sizes])
        cov = h.outcome_covariance(list(range(d + 2))) if sizes is None else h.outcome_group_covariance(list(range(d + 2)))
        recs.append(cov)
        n, V, s1, st = sobol_indices(cov, d)
        got = t[..., k, :]
        assert same(got[..., 0], n) and same(got[..., 1], V), k
        assert same(got[..., 3:3 + d], s1) and same(got[..., 3 + d:3 + 2 * d], st), k
    return recs


def _check_boot(t, Y, d, B, seed, recs, sizes=None):
    p = Y.shape[1]
    q = d + 2
    o = 0
    for g, W in enumerate([Y.shape[0]] if sizes is None else sizes):
        for k in range(p):
            rec = recs[k] if sizes is None else recs[k][g]
            sd1, sdt, good = ref_bootstrap(Y[o:o + W, k], d, B, seed, rec[1:q + 1])
            got = t[k] if sizes is None else t[g, k]
            assert got[2] == good, (g, k)
            for want, have in ((sd1, got[3 + 2 * d:3 + 3 * d]), (sdt, got[3 + 3 * d:])):
                assert np.array_equal(np.isnan(want), np.isnan(have)), (g, k, want, have)
                assert np.allclose(have, want, rtol=1e-9, atol=0, equal_nan=True), (g, k, want, have)
        o += W


def _launches(ex, call, sample_groups, B, slices=1):
    n0 = ex.timings()["kernel_launches"]
    out = call()
    merge = any(n > 64 for n in sample_groups)
    assert ex.timings()["kernel_launches"] - n0 == 1 + 1 + merge + slices * (3 if B else 1)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_point_estimates_bit_for_bit_and_bootstrap(math):
    need_gpu()
    for N in (1, 2, 3, 100, 4096):
        des = monte_carlo.saltelli(ishigami_spec(N))
        y = ishigami(design_X(des))
        Y = np.column_stack([y, 3.0 * y + 1e5, np.cos(y)])
        ex = _values_handle(Y, math)
        B = 64
        t = _launches(ex, lambda: ex.outcome_sobol([0, 1, 2], 3, B, 99), [N], B)
        recs = _check_point(ex, t, Y, 3)
        _check_boot(t, Y, 3, B, 99, recs)
        if N == 4096:
            z = NormalDist().inv_cdf(0.975)
            _, _, _, S1, ST, s1, st = record_split(t[0], 3)
            assert np.all(np.abs(S1 - ISHIGAMI_S1) <= 3 * z * s1 + 1e-3), (S1, s1)
            assert np.all(np.abs(ST - ISHIGAMI_ST) <= 3 * z * st + 1e-3), (ST, st)
    A = np.random.default_rng(1).uniform(-np.pi, np.pi, (1 << 16, 3))
    B_ = np.random.default_rng(2).uniform(-np.pi, np.pi, (1 << 16, 3))
    y = ishigami(layout(A, B_))
    ex = _values_handle(y, math)
    t = ex.outcome_sobol([0], 3, 20, 5)
    _check_boot(t, y[:, None], 3, 20, 5, _check_point(ex, t, y[:, None], 3))
    _, _, _, S1, ST, s1, st = record_split(t[0], 3)
    assert np.all(np.abs(S1 - ISHIGAMI_S1) <= 3 * 1.96 * s1 + 1e-3) and np.all(np.abs(ST - ISHIGAMI_ST) <= 3 * 1.96 * st + 1e-3)


@pytest.mark.gpu
def test_incomplete_samples_per_output():
    need_gpu()
    rng = np.random.default_rng(4)
    d, N = 4, 300
    y = layout(rng.normal(size=(N, d)), rng.normal(size=(N, d))) @ np.array([1.0, -2.0, 0.5, 0.0])
    Y = np.column_stack([y, y * y, np.exp(y)])
    q = d + 2
    Y[0 * q + 0, 0] = np.nan          # A of sample 0, output 0
    Y[1 * q + q - 1, 0] = np.inf      # B of sample 1
    Y[2 * q + 3, 0] = -np.inf         # one AB world of sample 2
    Y[5 * q + 2, 1] = np.nan          # output 1: sample 5 only
    Y[7 * q + 1, 2] = 1e308           # output 2: f(AB) - f(A) overflows nowhere, finite: complete
    Y[8 * q + 0, 2] = -1e308
    Y[8 * q + 1, 2] = 1e308           # output 2: the difference overflows: incomplete
    ex = _values_handle(Y)
    t = ex.outcome_sobol([0, 1, 2], d, 30, 1)
    assert t[0, 0] == N - 3 and t[1, 0] == N - 1 and t[2, 0] == N - 1
    recs = _check_point(ex, t, Y, d)
    _check_boot(t, Y, d, 30, 1, recs)


@pytest.mark.gpu
def test_edges():
    need_gpu()
    rng = np.random.default_rng(6)
    # a constant output, n = 0 and n = 1 in groups; B = 0 and B = 1
    d, q = 2, 4
    y = rng.normal(size=q * 40)
    Y = np.column_stack([y, np.full_like(y, 2.5), y.copy(), y.copy()])
    Y[:q * 10, 2] = np.nan  # group 0 of output 2: n = 0
    Y[q * 10:q * 19, 3] = np.nan  # group 1 of output 3: n = 1
    sizes = [q * 10, q * 10, q * 20]
    ex = _values_handle(Y, groups=sizes)
    for B in (0, 1, 5):
        t = _launches(ex, lambda: ex.outcome_group_sobol([0, 1, 2, 3], d, B, 3), [10, 10, 20], B)
        recs = _check_point(ex, t, Y, d, sizes)
        n, V, ok, S1, ST, s1, st = record_split(t, d)
        assert np.all(V[:, 1] == 0) and np.all(np.isnan(S1[:, 1])) and np.all(np.isnan(ST[:, 1]))
        assert n[0, 2] == 0 and np.isnan(V[0, 2]) and np.all(np.isnan(S1[0, 2]))
        assert n[1, 3] == 1 and np.isnan(V[1, 3]) and np.all(np.isnan(ST[1, 3]))
        if B < 2:
            assert np.all(np.isnan(s1)) and np.all(np.isnan(st))
        if B == 0:
            assert np.all(ok == 0)
        else:
            _check_boot(t, Y, d, B, 3, recs, sizes)
    # d = 1 and d = 23, 25 outputs
    for d in (1, 23):
        q = d + 2
        N = 64 if d == 23 else 500
        A, B_ = rng.uniform(size=(N, d)), rng.uniform(size=(N, d))
        X = layout(A, B_)
        c = rng.normal(size=d)
        Y = np.column_stack([np.sin(3 * X @ c + k) + 0.1 * k * X[:, 0] ** 2 for k in range(25)])
        ex = _values_handle(Y)
        t = ex.outcome_sobol(list(range(25))[::-1], d, 8, 2)
        recs = _check_point(ex, t, Y[:, ::-1], d)
        _check_boot(t, Y[:, ::-1], d, 8, 2, recs)


@pytest.mark.gpu
def test_groups_equal_a_handle_over_their_worlds_and_slices():
    need_gpu()
    rng = np.random.default_rng(8)
    d, q = 23, 25
    sizes = [q * 50, 0, q * 7, q * 51]
    W = sum(sizes)
    X = rng.uniform(size=(W, d))
    Y = np.column_stack([np.sin(X @ rng.normal(size=d)) * (1 + k) + X[:, k % d] ** 2 for k in range(25)])
    Y[rng.random(Y.shape) < 0.002] = np.nan
    ex = _values_handle(Y, groups=sizes)
    B = 10000  # 25 outputs x 4 groups of 3.7 MB tasks: two slices of the bootstrap scratch
    t = _launches(ex, lambda: ex.outcome_group_sobol(list(range(25)), d, B, 17), [50, 0, 7, 51], B, slices=2)
    o = 0
    for g, n in enumerate(sizes):
        if n:
            alone = _values_handle(Y[o:o + n])
            assert same(t[g], alone.outcome_sobol(list(range(25)), d, B, 17)), g
        else:
            assert np.all(t[g, :, 0] == 0) and np.all(np.isnan(t[g, :, 3:]))
        o += n
    _check_boot(t[:, :2], Y[:, :2], d, B, 17, _check_point(ex, t[:, :2], Y[:, :2], d, sizes), sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_reproducible_without_side_effects_and_abi(math):
    need_gpu()
    import torch

    rng = np.random.default_rng(2)
    d, q, N = 3, 5, 2000
    y = ishigami(layout(rng.uniform(-np.pi, np.pi, (N, d)), rng.uniform(-np.pi, np.pi, (N, d))))
    Y = np.column_stack([y, -y, rng.normal(size=y.size)])
    sizes = [q * 700, q * 1300]
    ex = _values_handle(Y, math, groups=sizes)
    vals = ex.outcome_values()
    cov = ex.outcome_group_covariance([0, 1, 2])
    ranks = ex.outcome_group_ranks([0, 1])
    want = ex.outcome_group_sobol([2, 0], d, 50, 7)
    assert same(ex.outcome_group_sobol([2, 0], d, 50, 7), want)
    assert not same(ex.outcome_group_sobol([2, 0], d, 50, 8)[..., 3 + 2 * d:], want[..., 3 + 2 * d:])
    dev = torch.empty(want.size, dtype=torch.float64, device="cuda")
    ex._reduce("group_sobol", "outcome", ex._selection([2, 0]) + (d, 50, 7), want.shape, dev.data_ptr())
    torch.cuda.synchronize()
    assert same(dev.cpu().numpy().reshape(want.shape), want)
    s = torch.cuda.Stream()
    ex.set_stream(s.cuda_stream)
    with torch.cuda.stream(s):
        dev2 = torch.full((want.size,), 5.0, dtype=torch.float64, device="cuda")
        ex._reduce("group_sobol", "outcome", ex._selection([2, 0]) + (d, 50, 7), want.shape, dev2.data_ptr())
        back = dev2.cpu()
    assert same(back.numpy().reshape(want.shape), want)
    ex.set_stream(None)
    assert same(ex.outcome_values(), vals) and same(ex.outcome_group_covariance([0, 1, 2]), cov)
    assert same(ex.outcome_group_ranks([0, 1]), ranks)
    # the C ABI's refusals, the handle usable after each
    L, h = ex._L, ex._h
    out = np.empty(4096)
    u32p = ctypes.POINTER(ctypes.c_uint32)
    INV = _lib.ERR_INVALID_ARGUMENT

    def call(name, pl, d_, B, nbytes):
        arr = (ctypes.c_uint32 * max(len(pl), 1))(*pl)
        fn = getattr(L, f"b200_sixdof_outcome_{name}")
        return lambda: _lib.check(fn(h, ctypes.cast(arr, u32p), len(pl), d_, B, 0, ctypes.c_void_p(out.ctypes.data), nbytes))

    rec = lambda d_, p=1, G=1: G * p * (3 + 4 * d_) * 8
    _refused(call("sobol", [], 3, 0, rec(3, 0)), INV, "0 sobol planes: 1 to 3")
    _refused(call("sobol", [0, 0], 3, 0, rec(3, 2)), INV, "sobol plane 0 listed twice")
    _refused(call("sobol", [3], 3, 0, rec(3)), INV, "sobol plane 0 is 3: the outcome has 3 planes")
    _refused(call("sobol", [0], 0, 0, rec(0)), INV, "sobol: 0 inputs, 1 to 23")
    _refused(call("sobol", [0], 24, 0, rec(24)), INV, "sobol: 24 inputs, 1 to 23")
    _refused(call("sobol", [0], 4, 0, rec(4)), INV, "sobol: the batch has 10000 worlds, not a multiple of d \\+ 2 = 6")
    _refused(call("group_sobol", [0], 1, 0, rec(1, 1, 2)), INV, "group 0 has 3500 worlds, not a multiple of d \\+ 2 = 3")
    _refused(call("sobol", [0], 3, 10001, rec(3)), INV, "sobol: 10001 resamples, at most 10000")
    _refused(call("sobol", [0], 3, 0, rec(3) + 8), _lib.ERR_VALUE_SIZE_MISMATCH, f"outcome sobol records are {rec(3)} bytes")
    assert same(ex.outcome_group_sobol([2, 0], d, 50, 7), want)
    ex2 = el.B200Exec(1, 10, 0.01, None, [], "rk4", "exact")
    _refused(lambda: ex2.outcome_sobol([0], 3, 0, 0), INV, "no outcomes: call b200_sixdof_set_outcomes first")
    _refused(lambda: _values_handle(Y).outcome_group_sobol([0], 3, 0, 0), INV, "grouped outcome sobol")


@pytest.mark.gpu
def test_four_million_worlds():
    need_gpu()
    rng = np.random.default_rng(12)
    d, N = 2, 1 << 20
    X = layout(rng.uniform(size=(N, d)), rng.uniform(size=(N, d)))
    y = 1e5 + 10.0 * (X[:, 0] + 2.0 * X[:, 1] + X[:, 0] * X[:, 1])
    ex = _values_handle(y)
    assert ex.n_worlds == 1 << 22
    t = _launches(ex, lambda: ex.outcome_sobol([0], d, 10, 3), [N], 10)
    _check_boot(t, y[:, None], d, 10, 3, _check_point(ex, t, y[:, None], d))


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_rocket_campaign(math):
    need_gpu()
    import importlib.util

    spec = importlib.util.spec_from_file_location("rocket_sobol", os.path.join(ROOT, "examples", "rocket_sobol.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    design, ex, s, sens = mod.campaign(n_base=512, bootstrap=100, seed=1, math_mode=math)
    iaz, y = design.inputs.index("wind_az"), s["outputs"].index("impact_y")
    landed = s["count"][:, y] >= 100
    assert landed.any(), s["count"]
    assert np.all(s["ST"][landed, y, iaz] > 0.2), s["ST"][:, y]
    assert np.all(np.isfinite(s["ST_conf"][landed, y]))
    assert abs(sens["prcc"][y, iaz]) < 0.1, sens["prcc"][y]
