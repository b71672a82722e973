"""Rank correlation of a Monte-Carlo batch (b200_sixdof_outcome_[group_]ranks and _rank_correlation, rank_kernels.cu):
per group, the midrank of every complete world (all selected outcomes finite) in each selected outcome, and the
Spearman correlation of those ranks through the covariance kernels.

The CPU tests check the constants and prototypes against the header, the numpy restatement of the midranks on hand
cases, every Exec refusal before the backend is reached (a world-sharded build included), that an Exec which never
asks for ranks makes the backend calls it made before, and the PRCC helper against an independent restatement by rank
regressions.  The GPU tests, in both math modes, hold every rank to scipy.stats.rankdata bit for bit on a rocket
campaign and on adversarial planes at every route edge and over several scratch slices, the read bound, rho to the
numpy formula on the covariance of a handle holding the downloaded ranks (bit for bit) and to scipy.stats.spearmanr,
each group to a handle over its worlds, the absence of side effects, and the C ABI's refusals, destinations and a
caller stream."""

import ctypes
import os
import re
import warnings

import numpy as np
import pytest
import scipy.stats

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200.executor import partial_rank_correlation, rank_correlation
from tests.ensemble_util import need_gpu, two_body_world
from tests.test_ensemble_outcomes import _OutcomeFake, campaign
from tests.test_host_logic import _FakeBackend

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("exact", "fast")
O = el.Outcome
READ_BOUND = 7  # include/b200_sixdof.h: at most 7 reads of a task's plane on any data


# --------------------------------------------------------------------------- the numpy restatement


def ref_ranks(values, sizes=None):
    """[M, p] midranks of values [M, p] within each group of `sizes` (default: one group) over the worlds whose p
    values are all finite; NaN elsewhere."""
    values = np.asarray(values, dtype=np.float64)
    M, p = values.shape
    out = np.full((M, p), np.nan)
    ok = np.all(np.isfinite(values), axis=1)
    o = 0
    for n in ([M] if sizes is None else sizes):
        w = np.arange(o, o + n)[ok[o:o + n]]
        for j in range(p):
            if w.size:
                out[w, j] = scipy.stats.rankdata(values[w, j], method="average")
        o += n
    return out


def bits(x):
    x = np.array(x, dtype=np.float64)
    x[np.isnan(x)] = np.nan
    return x.view(np.uint64)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


def lstsq_prcc(ranks_in, rank_out):
    """PRCC of each input by the definition: the Pearson correlation of the residuals of input i and of the output
    after a least-squares regression of each on the other inputs' ranks (and a constant); NaN where the regressors and
    the column are collinear."""
    n, k = ranks_in.shape
    out = np.full(k, np.nan)
    for i in range(k):
        X = np.column_stack([np.ones(n), np.delete(ranks_in, i, axis=1)])
        full = np.column_stack([X, ranks_in[:, i], rank_out])
        if np.linalg.matrix_rank(full) < full.shape[1]:
            continue
        ri = ranks_in[:, i] - X @ np.linalg.lstsq(X, ranks_in[:, i], rcond=None)[0]
        ry = rank_out - X @ np.linalg.lstsq(X, rank_out, rcond=None)[0]
        out[i] = np.corrcoef(ri, ry)[0, 1]
    return out


def test_reference_midranks_on_hand_cases():
    nan, inf, tiny = np.nan, np.inf, 5e-324
    r = ref_ranks(np.array([[2.0], [1.0], [2.0], [3.0], [2.0]]))  # a tie run of three: ranks 2, 3, 4 -> 3
    assert list(r[:, 0]) == [3.0, 1.0, 3.0, 5.0, 3.0]
    r = ref_ranks(np.array([[-0.0], [0.0], [tiny], [-tiny], [0.0]]))  # -0 ties with +0
    assert list(r[:, 0]) == [3.0, 3.0, 5.0, 1.0, 3.0]
    v = np.array([[1.0, 5.0], [nan, 1.0], [3.0, inf], [2.0, 0.0], [-inf, 2.0], [0.5, 9.0]])
    r = ref_ranks(v)  # a non-finite value drops its world from both planes
    assert np.all(np.isnan(r[[1, 2, 4]])) and list(r[[0, 3, 5], 0]) == [2.0, 3.0, 1.0]
    assert list(r[[0, 3, 5], 1]) == [2.0, 1.0, 3.0]
    assert list(ref_ranks(np.full((4, 1), 7.0))[:, 0]) == [2.5] * 4  # a constant plane
    assert ref_ranks(np.zeros((0, 2))).shape == (0, 2)
    assert np.all(np.isnan(ref_ranks(np.array([[4.0, nan]]))))  # n = 0
    assert list(ref_ranks(np.array([[4.0, 1.0]]))[0]) == [1.0, 1.0]  # n = 1
    r = ref_ranks(np.array([[3.0], [1.0], [2.0], [1.0]]), sizes=[2, 0, 2])  # within each group
    assert list(r[:, 0]) == [2.0, 1.0, 2.0, 1.0]
    # the record: n = 1 and n = 0 give NaN rho; a constant plane its row and column
    cov = np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 0.0])
    assert np.all(np.isnan(rank_correlation(cov, 2)[1:]))
    c3 = np.array([3.0, 2.0, 2.0, 0.0, 0.0, 0.0, 2.0])  # plane 0 constant
    rec = rank_correlation(c3, 2)
    assert rec[0] == 3.0 and np.all(np.isnan(rec[1:4])) and rec[4] == 1.0


def test_header_constants_and_prototypes():
    h = open(os.path.join(ROOT, "include", "b200_sixdof.h")).read()
    for name, args in (("b200_sixdof_outcome_ranks", 5), ("b200_sixdof_outcome_group_ranks", 5),
                       ("b200_sixdof_outcome_rank_correlation", 5), ("b200_sixdof_outcome_group_rank_correlation", 5),
                       ("b200_sixdof_rank_reads", 1)):
        m = re.search(name + r"\(([^)]*)\)", h)
        assert m and len(m.group(1).split(",")) == args, name
        assert name in _lib.SYMBOLS, name
    assert int(re.search(r"#define B200_MAX_OUTCOMES (\d+)u", h).group(1)) == _lib.MAX_OUTCOMES == 25
    L = _lib.lib()
    for name in ("ranks", "group_ranks", "rank_correlation", "group_rank_correlation"):
        fn = getattr(L, f"b200_sixdof_outcome_{name}")
        assert len(fn.argtypes) == 5 and fn.argtypes[2] is ctypes.c_uint32 and fn.argtypes[4] is ctypes.c_uint64
    assert L.b200_sixdof_rank_reads.restype is ctypes.c_double


def test_prcc_helper_equals_rank_regressions():
    rng = np.random.default_rng(11)
    for trial in range(60):
        n = int(rng.integers(8, 80))
        k = int(rng.integers(1, 5))
        X = rng.normal(size=(n, k))
        if trial % 3 == 0:
            X[:, 0] = np.round(X[:, 0])  # ties
        y = X @ rng.normal(size=k) + rng.normal(scale=0.5, size=n)
        if trial % 10 == 1 and k >= 2:
            X[:, 1] = X[:, 0]  # a singular rank correlation matrix
        ranks = np.column_stack([scipy.stats.rankdata(c) for c in np.column_stack([X, y]).T])
        R = np.corrcoef(ranks, rowvar=False)
        got = partial_rank_correlation(R)
        want = lstsq_prcc(ranks[:, :k], ranks[:, k])
        assert np.array_equal(np.isnan(got), np.isnan(want)), trial
        assert np.allclose(got, want, atol=1e-10, rtol=0, equal_nan=True), (trial, got, want)
        if k == 1:
            assert np.allclose(got, R[0, 1], atol=1e-12)
    assert np.all(np.isnan(partial_rank_correlation(np.array([[1.0, np.nan], [np.nan, 1.0]]))))
    G = np.stack([np.eye(3), np.ones((3, 3))])  # a leading axis; the second is singular
    got = partial_rank_correlation(G)
    assert got.shape == (2, 2) and np.all(got[0] == 0.0) and np.all(np.isnan(got[1]))


# --------------------------------------------------------------------------- CPU: Exec through a fake backend


class _RankFake(_OutcomeFake):
    """The outcome fake with the rank calls logged; the correlation is the identity, ranks name their plane."""

    def outcome_ranks(self, planes):
        self._log("outcome_ranks", list(planes))
        return np.tile(np.asarray(planes, dtype=np.float64), (5, 1))

    def outcome_group_ranks(self, planes):
        self._log("outcome_group_ranks", list(planes))
        return np.tile(np.asarray(planes, dtype=np.float64), (5, 1))

    def _corr(self, name, planes, G=None):
        self._log(name, list(planes))
        p = len(planes)
        rec = np.concatenate([[5.0], (0.5 * np.eye(p) + 0.5 * np.ones((p, p))).ravel()])
        return rec if G is None else np.tile(rec, (G, 1))

    def outcome_rank_correlation(self, planes):
        return self._corr("outcome_rank_correlation", planes)

    def outcome_group_rank_correlation(self, planes):
        return self._corr("outcome_group_rank_correlation", planes, self.n_groups)


def _exec(monkeypatch, **kw):
    from elodin_b200 import world as W

    monkeypatch.setattr(W, "B200Exec", _RankFake)
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
    cases = [
        (lambda: ex.outcome_ranks(["apogee", "apogee"]), ValueError, "distinct outcome names"),
        (lambda: ex.outcome_ranks([]), ValueError, "1 or more distinct"),
        (lambda: ex.outcome_ranks(["nosuch"]), _lib.B200ValueError, "outcome not found: 'nosuch'"),
        (lambda: ex.outcome_ranks(groups=True), _lib.B200Error, r"outcome_ranks\(groups=True\).*groups=\[...\]"),
        (lambda: ex.outcome_rank_correlation(["gain"]), ValueError, "2 or more distinct"),
        (lambda: ex.outcome_rank_correlation(["gain", "gain"]), ValueError, "2 or more distinct"),
        (lambda: ex.outcome_rank_correlation(["gain", "x"]), _lib.B200ValueError, "outcome not found: 'x'"),
        (lambda: ex.outcome_rank_correlation(groups=True), _lib.B200Error, r"outcome_rank_correlation\(groups=True\)"),
        (lambda: ex.outcome_sensitivity([], ["apogee"]), ValueError, "non-empty and disjoint"),
        (lambda: ex.outcome_sensitivity(["gain"], []), ValueError, "non-empty and disjoint"),
        (lambda: ex.outcome_sensitivity(["gain", "t"], ["t"]), ValueError, "non-empty and disjoint"),
        (lambda: ex.outcome_sensitivity(["gain"] * 2, ["t"]), ValueError, "distinct outcome names"),
        (lambda: ex.outcome_sensitivity([f"i{k}" for k in range(20)], [f"o{k}" for k in range(6)]), ValueError,
         "26 names, at most 25"),
        (lambda: ex.outcome_sensitivity(["gain"], ["nosuch"]), _lib.B200ValueError, "outcome not found"),
        (lambda: ex.outcome_sensitivity(["gain"], ["t"], groups=True), _lib.B200Error, r"outcome_sensitivity\(groups=True\)"),
    ]
    for call, exc, match in cases:
        with pytest.raises(exc, match=match):
            call()
    assert len(_FakeBackend.calls) == n0
    plain = _exec(monkeypatch)
    with pytest.raises(_lib.B200Error, match=r"outcome_ranks\(\): build the Exec with .*outcomes=\[...\]"):
        plain.outcome_ranks()
    # a world-sharded build: all three refused, before any backend call
    ex._pg = object()
    n0 = len(_FakeBackend.calls)
    for call in (lambda: ex.outcome_ranks(), lambda: ex.outcome_rank_correlation(),
                 lambda: ex.outcome_sensitivity(["gain"], ["apogee"])):
        with pytest.raises(_lib.B200Error, match="world-sharded campaign are not supported") as e:
            call()
        assert e.value.code == _lib.ERR_UNSUPPORTED
    assert len(_FakeBackend.calls) == n0


def test_an_exec_that_never_asks_makes_the_same_calls(monkeypatch):
    """The rank entries add no backend call of their own to an Exec's run; asking adds exactly one."""
    _exec(monkeypatch, outcomes=OUTS, groups=[2, 3])
    before = list(_FakeBackend.calls)
    assert not any("rank" in c[0] for c in before)
    from tests.test_ensemble_outcomes import _calls

    _, with_outcomes = _calls(monkeypatch, outcomes=OUTS)
    assert not any("rank" in c[0] for c in with_outcomes)
    ex = _exec(monkeypatch, outcomes=OUTS, groups=[2, 3])
    assert _FakeBackend.calls == before
    r = ex.outcome_ranks(["gain", "apogee"])
    assert _FakeBackend.calls == before + [("outcome_ranks", [2, 0])]
    assert list(r) == ["gain", "apogee"] and np.all(r["gain"] == 2.0) and np.all(r["apogee"] == 0.0)
    c = ex.outcome_rank_correlation(groups=True)
    assert _FakeBackend.calls[-1] == ("outcome_group_rank_correlation", [0, 1, 2])
    assert c["rho"].shape == (2, 3, 3) and c["count"].shape == (2,) and c["names"] == ["apogee", "t", "gain"]
    s = ex.outcome_sensitivity(["gain", "t"], "apogee")
    assert _FakeBackend.calls[-1] == ("outcome_rank_correlation", [2, 1, 0])
    assert s["rho"].shape == (1, 2) and np.all(s["rho"] == 0.5) and s["inputs"] == ["gain", "t"]
    # R = 0.5 off the diagonal, 3 x 3: prcc = (0.5 - 0.5 * 0.5) / (1 - 0.5 * 0.5) = 1 / 3
    assert np.allclose(s["prcc"], 1 / 3) and s["outputs"] == ["apogee"]
    g = ex.outcome_sensitivity(["gain"], ["apogee", "t"], groups=True)
    assert g["rho"].shape == (2, 2, 1) and np.allclose(g["prcc"], g["rho"])  # one input: prcc = rho


# --------------------------------------------------------------------------- GPU


def _only_values(values, math, groups=None):
    """A handle of one entity whose outcomes are VALUES outcomes holding `values` [M, p]."""
    M, p = values.shape
    ex = el.B200Exec(1, M, 0.01, None, [], "rk4", math)
    ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, np.ascontiguousarray(values[:, j])) for j in range(p)])
    if groups is not None:
        ex.set_world_groups(groups)
    return ex


def _check_rho(ex, values, planes, math, sizes=None):
    """rho of the device equals the numpy formula on the covariance of a handle holding the downloaded ranks, bit for
    bit, and scipy.stats.spearmanr over the complete worlds to 1e-12."""
    p = len(planes)
    if sizes is None:
        got = ex.outcome_rank_correlation(planes)
        ranks = ex.outcome_ranks(planes)
        cov = _only_values(ranks, math).outcome_covariance(list(range(p)))
    else:
        got = ex.outcome_group_rank_correlation(planes)
        ranks = ex.outcome_group_ranks(planes)
        cov = _only_values(ranks, math, sizes).outcome_group_covariance(list(range(p)))
    assert same(got, rank_correlation(cov, p))
    sel = values[:, planes]
    o = 0
    for g, n in enumerate([values.shape[0]] if sizes is None else sizes):
        rec = got if sizes is None else got[g]
        x = sel[o:o + n]
        x = x[np.all(np.isfinite(x), axis=1)]
        assert rec[0] == x.shape[0]
        if x.shape[0] >= 2:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")  # spearmanr warns on a constant column
                st = scipy.stats.spearmanr(x).statistic
            want = np.array([[1.0, st], [st, 1.0]]) if p == 2 else np.array(st)
            for j in range(p):
                if np.all(x[:, j] == x[0, j]):
                    want[j, :] = want[:, j] = np.nan
            rho = rec[1:].reshape(p, p)
            assert np.allclose(rho, want, atol=1e-12, rtol=0, equal_nan=True), (g, rho, want)
        else:
            assert np.all(np.isnan(rec[1:]))
        o += n
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_rocket_campaign_ranks_and_rho(math):
    need_gpu()
    M = 300
    sizes = [100, 37, 163]
    ex, _, _ = campaign(M, math, "resident", groups=sizes)
    v = ex.outcome_values()
    names = ["mass", "wind", "thrust", "gain", "apogee", "xmin", "t_hit", "rows", "vz_std"]
    vals = np.stack([v[n] for n in names], axis=1)
    be = ex.backend
    planes = [ex.outcomes.index(n) for n in names]
    assert same(be.outcome_ranks(planes), ref_ranks(vals))
    assert same(be.outcome_group_ranks(planes), ref_ranks(vals, sizes))
    assert be.rank_reads() == 1.0  # small groups: one read
    for j, n in enumerate(names):  # each plane alone: its own finite worlds
        assert same(be.outcome_ranks([planes[j]])[:, 0], ref_ranks(vals[:, [j]])[:, 0]), n
    _check_rho(be, np.stack([v[n] for n in ex.outcomes], axis=1), planes, math)
    _check_rho(be, np.stack([v[n] for n in ex.outcomes], axis=1), planes, math, sizes)
    r = ex.outcome_ranks(["apogee", "mass"])
    assert same(r["apogee"], ref_ranks(vals[:, [4, 0]])[:, 0])
    c = ex.outcome_rank_correlation(["mass", "apogee"], groups=True)
    assert c["rho"].shape == (3, 2, 2) and same(c["count"], be.outcome_group_rank_correlation(planes[:1] + planes[4:5])[:, 0])
    s = ex.outcome_sensitivity(["mass", "wind", "thrust"], ["apogee", "xmin"])
    R = be.outcome_rank_correlation([planes[k] for k in (0, 1, 2, 4, 5)])[1:].reshape(5, 5)
    assert same(s["rho"], R[3:, :3])
    assert same(s["prcc"][0], partial_rank_correlation(R[np.ix_([0, 1, 2, 3], [0, 1, 2, 3])]))
    assert same(s["prcc"][1], partial_rank_correlation(R[np.ix_([0, 1, 2, 4], [0, 1, 2, 4])]))


def _adversarial(M, seed):
    """[M, 8] planes: continuous, 4 distinct values, all equal, 1 ulp apart (two adjacent values, with the range
    stretched to +-1e300: every refinement level), Cauchy with one 1e300 outlier, signed zeros with subnormals,
    uniform over one binade, and rounded normals with non-finite values."""
    rng = np.random.default_rng(seed)
    v = np.empty((M, 8))
    v[:, 0] = rng.normal(0, 1, M)
    v[:, 1] = rng.integers(0, 4, M).astype(np.float64)
    v[:, 2] = 3.25
    v[:, 3] = np.where(rng.random(M) < 0.5, 1.0, np.nextafter(1.0, 2.0))
    if M >= 4:
        v[rng.permutation(M)[:2], 3] = [-1e300, 1e300]
    v[:, 4] = rng.standard_cauchy(M)
    if M:
        v[rng.integers(0, M), 4] = 1e300
    z = rng.integers(0, 4, M)
    v[:, 5] = np.choose(z, [0.0, -0.0, 5e-324, -1e-310])
    v[:, 6] = rng.uniform(1.0, 2.0, M)
    v[:, 7] = np.round(rng.normal(0, 3, M))
    v[rng.random(M) < 0.03, 7] = np.nan
    v[rng.random(M) < 0.01, 7] = np.inf
    v[rng.random(M) < 0.01, 7] = -np.inf
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_route_edges_and_adversarial_planes(math):
    need_gpu()
    sizes = [0, 1, 2, 256, 257, 8192, 8193, (1 << 20) + 5]
    M = sum(sizes)
    values = _adversarial(M, seed=1)
    ex = _only_values(values, math, groups=sizes)
    planes = list(range(values.shape[1]))
    assert same(ex.outcome_group_ranks(planes), ref_ranks(values, sizes))
    assert 1.0 <= ex.rank_reads() <= READ_BOUND
    assert same(ex.outcome_group_ranks(planes), ref_ranks(values, sizes))  # two calls, the same bits
    for j in planes:  # each plane alone: every world whose value is finite
        assert same(ex.outcome_group_ranks([j]), ref_ranks(values[:, [j]], sizes)), j
        assert ex.rank_reads() <= READ_BOUND, j
    _check_rho(ex, values, [0, 1, 2, 4, 6], math, sizes)
    # ungrouped over the 2^20 + 5 worlds alone: the bound on every plane, 3 reads on a uniform one, 7 on 1-ulp ties
    big = values[-sizes[-1]:]
    one = _only_values(big, math)
    reads = []
    for j in planes:
        assert same(one.outcome_ranks([j]), ref_ranks(big[:, [j]])), j
        reads.append(one.rank_reads())
    assert max(reads) <= READ_BOUND and reads[6] <= 3.0 and reads[3] == READ_BOUND, reads
    assert reads[2] == 2.0, reads  # one value: the count and the scatter
    assert same(one.outcome_ranks(planes), ref_ranks(big))
    _check_rho(one, big, [0, 3, 4, 6, 7], math)


@pytest.mark.gpu
def test_several_scratch_slices():
    """25 planes x 64 groups of 8193 worlds: more large tasks than one 256 MiB slice of the scratch holds."""
    need_gpu()
    sizes = [8193] * 64
    rng = np.random.default_rng(9)
    values = rng.normal(0, 1, (sum(sizes), 25))
    values[:, 7] = np.round(values[:, 7] * 3)
    values[rng.random(values.shape) < 0.0005] = np.nan
    ex = _only_values(values, "fast", groups=sizes)
    order = list(range(25))[::-1]
    assert same(ex.outcome_group_ranks(order), ref_ranks(values[:, ::-1], sizes))
    _check_rho(ex, values, order, "fast", sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_group_records_equal_a_handle_over_the_group(math):
    need_gpu()
    sizes = [0, 300, 57, 8643, 9000, 1]
    values = _adversarial(sum(sizes), seed=4)
    planes = [0, 1, 3, 5, 7]
    ex = _only_values(values, math, groups=sizes)
    ranks = ex.outcome_group_ranks(planes)
    rec = ex.outcome_group_rank_correlation(planes)
    assert same(ex.outcome_group_rank_correlation(planes), rec)
    o = 0
    for g, n in enumerate(sizes):
        if n:
            alone = _only_values(values[o:o + n], math)
            assert same(ranks[o:o + n], alone.outcome_ranks(planes)), g
            assert same(rec[g], alone.outcome_rank_correlation(planes)), g
        else:
            assert rec[g, 0] == 0 and np.all(np.isnan(rec[g, 1:]))
        o += n


@pytest.mark.gpu
@pytest.mark.parametrize("math", MODES)
def test_no_side_effects_on_the_outcomes(math):
    need_gpu()
    ex, _, _ = campaign(200, math, "resident", groups=[120, 80])
    be = ex.backend
    P = be.n_outcomes
    vals = be.outcome_values()
    cov = be.outcome_covariance(list(range(P)))
    gcov = be.outcome_group_covariance(list(range(P)))
    be.outcome_group_ranks(list(range(P)))
    be.outcome_rank_correlation(list(range(P))[::-1])
    be.outcome_group_rank_correlation([3, 22, 0])
    assert same(be.outcome_values(), vals)
    assert same(be.outcome_covariance(list(range(P))), cov)
    assert same(be.outcome_group_covariance(list(range(P))), gcov)


def _refused(call, code, match):
    with pytest.raises(_lib.B200Error, match=match) as e:
        call()
    assert e.value.code == code


@pytest.mark.gpu
def test_abi_refusals_destinations_and_a_caller_stream():
    need_gpu()
    import torch

    M = 9000
    values = _adversarial(M, seed=8)[:, [0, 1, 7]]
    ex = el.B200Exec(1, M, 0.01, None, [], "rk4", "exact")
    INV = _lib.ERR_INVALID_ARGUMENT
    _refused(lambda: ex.outcome_ranks([0]), INV, "no outcomes: call b200_sixdof_set_outcomes first")
    ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, np.ascontiguousarray(values[:, j])) for j in range(3)])
    L, h = ex._L, ex._h
    out = np.empty(M * 4)
    u32p = ctypes.POINTER(ctypes.c_uint32)

    def call(name, planes, n_p, nbytes):
        fn = getattr(L, f"b200_sixdof_outcome_{name}")
        arr = None if planes is None else (ctypes.c_uint32 * max(len(planes), 1))(*planes)
        return lambda: _lib.check(fn(h, ctypes.cast(arr, u32p) if arr is not None else None, n_p,
                                     ctypes.c_void_p(out.ctypes.data), nbytes))

    for name, least, nb in (("ranks", 1, M * 8), ("rank_correlation", 2, 5 * 8)):
        what = "ranks are" if name == "ranks" else "rank correlation is"
        _refused(call(name, None, 2, nb), INV, "null rank planes")
        _refused(call(name, [0], 0, nb), INV, f"0 rank planes: {least} to 3")
        _refused(call(name, [0, 1, 2, 0], 4, nb), INV, f"4 rank planes: {least} to 3")
        _refused(call(name, [3, 0], 2, nb), INV, "rank plane 0 is 3: the outcome has 3 planes")
        _refused(call(name, [1, 1], 2, nb), INV, "rank plane 1 listed twice")
        _refused(call(f"group_{name}", [0, 1], 2, nb), INV, "grouped outcome rank")
    _refused(call("rank_correlation", [0], 1, 2 * 8), INV, "1 rank planes: 2 to 3")
    _refused(call("ranks", [0], 1, M * 8 - 8), _lib.ERR_VALUE_SIZE_MISMATCH, f"outcome ranks are {M * 8} bytes, got")
    _refused(call("rank_correlation", [0, 1], 2, 48), _lib.ERR_VALUE_SIZE_MISMATCH,
             "outcome rank correlation is 40 bytes, got 48")
    call("ranks", [2], 1, M * 8)()
    assert same(out[:M], ref_ranks(values[:, [2]])[:, 0])
    assert L.b200_sixdof_rank_reads(None) == 0.0
    # a summary that drops what an outcome names: refused, naming the outcome
    ex2 = el.B200Exec(1, 50, 0.01, None, [], "rk4", "exact")
    ex2.summary_begin(True, [(0, 6, False, 0.0)])
    ex2.set_outcomes([(_lib.OUTCOME_THRESHOLD, 0, 0), (_lib.OUTCOME_THRESHOLD, 0, 0)])
    ex2.summary_begin(True)
    _refused(lambda: ex2.outcome_rank_correlation([0, 1]), INV, "outcome 0: threshold 0, the summary in force has 0")
    # host and device destinations, and a caller-owned stream: the same tables
    sizes = [100, 8900]
    ex.set_world_groups(sizes)
    for name, shape in (("group_ranks", (M, 2)), ("group_rank_correlation", (2, 5))):
        want = getattr(ex, f"outcome_{name}")([2, 0])
        dev = torch.empty(want.size, dtype=torch.float64, device="cuda")
        ex._reduce(name, "outcome", ex._selection([2, 0]), shape, dev.data_ptr())
        torch.cuda.synchronize()
        assert same(dev.cpu().numpy().reshape(shape), want)
        s = torch.cuda.Stream()
        ex.set_stream(s.cuda_stream)
        with torch.cuda.stream(s):
            dev2 = torch.full((want.size,), 5.0, dtype=torch.float64, device="cuda")
            ex._reduce(name, "outcome", ex._selection([2, 0]), shape, dev2.data_ptr())
            back = dev2.cpu()  # ordered after the entry on the caller's stream
        assert same(back.numpy().reshape(shape), want)
        ex.set_stream(None)
    assert same(ex.outcome_group_ranks([2, 0]), ref_ranks(values[:, [2, 0]], sizes))
    # launches of one large group: the mask, the count .. finish sequence of one slice, the row layout
    ex.set_world_groups([M])
    n0 = ex.timings()["kernel_launches"]
    ex.outcome_group_ranks([0])
    assert ex.timings()["kernel_launches"] - n0 == 1 + 15 + 1
