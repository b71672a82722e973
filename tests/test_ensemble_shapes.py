"""The ensemble reductions (statistics, covariance, quantiles) at every boundary of their launch geometry and at the top
of the f64 range, against an exact reference.

Reference.  The mean, m2 = sum (x - mean)^2 and the co-moments M_ab are exact rationals (integer sums of the values
scaled by 2^1074, a fractions.Fraction per result), rounded once to f64; a result beyond DBL_MAX keeps its exact value
in long double, so a finite answer there is measured against the true spread.  math.fsum cannot be the reference here:
it raises OverflowError past DBL_MAX, and the squared deviations of the top-range planes overflow before it sees them.
Quantiles keep the bit-exact ref_quantiles of test_ensemble_quantiles.

Contract, for every group of every shape and every catalogue plane (n = count, s = max|x| over the group's values):
  R1  count, min and max are exact; a quantile equals ref_quantiles bit for bit.
  R2  a finite mean, m2 or M_ab keeps the bounds of test_ensemble_stats / test_ensemble_covariance: mean within
      1e-13 s, std = sqrt(m2 / n) within 1e-8 std + 32 eps s, C = M / n within 1e-8 sig_a sig_b + 32 eps (s_a sig_b +
      sig_a s_b).  No exception: a finite value outside its bound is a failure.
  R3  a mean, m2 or M_ab of a group with n > 0 may be non-finite only where the data reaches the top of the range:
      s > 2^990, or the exact m2 (for covariance M_aa or M_bb) > 2^990.
  R4  where every |x| <= 2^1000 and the exact m2 (M_aa) exceeds DBL_MAX, the result is +inf: never 0, NaN or finite.

Shapes.  stats_shape, cov_chunks / cov_geo / slice_shape, the quantile route thresholds, pass_shape and the quantile
slice_shape are restated below (kNumSMs = 132).  The cases are each boundary and its neighbours, and every case asserts
the launch count its restated shape predicts, so the sweep is known to have run the geometry it names.  The data goes
in through the state entries (set_state, then state_stats / state_covariance / state_quantiles), which write it bit for
bit and reach the same kernels as the ring."""

import math
import warnings
from fractions import Fraction

import numpy as np
import pytest

import elodin_b200 as el
from tests.ensemble_util import need_gpu, split
from tests.test_ensemble_covariance import ref_table as fsum_cov_table
from tests.test_ensemble_quantiles import _degenerate, ref_quantiles
from tests.test_ensemble_stats import ref_table as fsum_stats_table

EPS = np.finfo(np.float64).eps
DBL_MAX = np.finfo(np.float64).max
LD = np.longdouble
TOP = 2.0 ** 990    # R3: the data reaches the top of the range above this
EDGE = 2.0 ** 1000  # R4: every |x| at most this
MODES = ("exact", "fast")
LEVELS16 = (0.0, 1e-3, 0.01, 0.05, 0.1, 0.25, 1 / 3, 0.5, 0.5 + 1e-9, 2 / 3, 0.75, 0.9, 0.95, 0.99, 0.999, 1.0)


# --------------------------------------------------------------------------- the launch geometry, restated

NUM_SMS = 132


def cdiv(a, b):
    return -(-a // b)


def stats_shape(M, E):
    """stats_kernels.cu stats_shape -> (J, Wc, C): world lanes per entity, worlds per chunk, chunks."""
    J = 256 // E if E <= 256 else 1
    per = max(cdiv(M, 64 * J), 8)  # kMaxChunks = 64, kMinPerThread = 8
    Wc = per * J
    return J, Wc, cdiv(M, Wc)


def stats_launches(M, E):
    return 1 if stats_shape(M, E)[2] == 1 else 2


def cov_chunks(M, E):
    """cov_kernels.cu cov_chunks -> (Wc, C)."""
    C = max(1, cdiv(4 * NUM_SMS, cdiv(E, 32)))  # kChunkTasks chunk tasks over entity tiles of kEntTile
    C = min(C, max(1, cdiv(M, 64)))              # kMinWorlds
    Wc = cdiv(M, C)
    return Wc, cdiv(M, Wc)


def cov_et(p):
    """cov_kernels.cu cov_geo: entities per block before the min with n_entities."""
    nb = (p + 3) // 4
    T = nb * (nb + 1) // 2
    et = 32
    while et > 1 and et * T > 512:
        et >>= 1
    return et


def cov_launches(M, E, p, samples=1):
    """Chunk launch (+ merge launch when C > 1) per slice of cov_kernels.cu slice_shape."""
    C = cov_chunks(M, E)[1]
    per = C * (1 + p + p * p) * 8 if C > 1 else 0
    ns = max(1, ((256 << 20) // per if per else 2 ** 64) // E)
    return cdiv(samples, ns) * (2 if C > 1 else 1)


# quantile_kernels.cu: kWarpMax, kSmallMax, and kSliceGroups from kGroupBytes = sizeof(QGroup) (72 bytes of counts and
# ranges + 32 QSlot of 48 bytes) + kBins u32 + kGroupCap u64
WARP_MAX, SMALL_MAX = 256, 8192
SLICE_GROUPS = ((256 << 20) - 256) // (72 + 32 * 48 + (1 << 14) * 4 + 16384 * 8)


def quantile_slices(E, planes=25):
    """quantile_kernels.cu slice_shape: slices of whole planes, or entity ranges of one plane."""
    if E <= SLICE_GROUPS:
        return cdiv(planes, max(1, SLICE_GROUPS // E))
    return planes * cdiv(E, SLICE_GROUPS)


def quantile_launches(M, E, planes=25):
    return 1 if M <= SMALL_MAX else 18 * quantile_slices(E, planes)


def pass_shape(M, E, planes):
    """quantile_kernels.cu pass_shape -> (Et, J, T, C)."""
    Et = min(E, 256)
    J = 256 // E if E <= 256 else 1
    T = cdiv(E, Et)
    want = max(1, 4 * NUM_SMS // max(1, planes * T))
    per = max(cdiv(M, want * J), 16)
    return Et, J, T, cdiv(M, per * J)


# --------------------------------------------------------------------------- exact reference


def _fixed(v):
    """Finite f64 [k] -> (three signed limbs of 18 bits [3][k] int64, shift [k]) with
    v = sum_i limb_i 2^(18 i + shift - 1074) exactly."""
    m, e = np.frexp(v)
    mi = np.abs(m * 2.0 ** 53).astype(np.int64)  # |mantissa| < 2^53, exact
    s = e.astype(np.int64) + (1074 - 53)
    low = np.minimum(s, 0)
    mi = mi >> -low  # subnormals: the bits shifted out are zeros
    s = s - low
    sg = np.where(v < 0, -1, 1).astype(np.int64)
    mask = (1 << 18) - 1
    return [sg * (mi & mask), sg * ((mi >> 18) & mask), sg * (mi >> 36)], s


def _group_sums(g, s, parts, G):
    """sum over entries k of parts[j][k] 2^(18 j + s[k]) per group g[k], as Python ints [G].  Entries of one group and
    shift are summed in int64 first (|part| < 2^38, so at most 2^25 entries per key stay exact)."""
    out = [0] * G
    if g.size == 0:
        return out
    key = g.astype(np.int64) * 8192 + s
    order = np.argsort(key, kind="stable")
    k = key[order]
    starts = np.flatnonzero(np.r_[True, k[1:] != k[:-1]])
    sums = [np.add.reduceat(p[order], starts).tolist() for p in parts]
    for i, kk in enumerate(k[starts].tolist()):
        gi, si = divmod(kk, 8192)
        out[gi] += sum(c[i] << (18 * j + si) for j, c in enumerate(sums) if c[i])
    return out


def _sums(X, ok):
    """X [M, G, p], ok [M, G] -> n [G], S[a] [G] = sum x_a 2^1074 and Q[a, b] [G] = sum x_a x_b 2^2148 (a <= b) over
    the rows where ok, as Python ints."""
    M, G, p = X.shape
    r, g = np.nonzero(ok)
    limbs, shifts = zip(*[_fixed(X[r, g, a]) for a in range(p)])
    S = [_group_sums(g, shifts[a], limbs[a], G) for a in range(p)]
    Q = {}
    for a in range(p):
        for b in range(a, p):
            P = [sum(limbs[a][i] * limbs[b][j - i] for i in range(3) if 0 <= j - i < 3) for j in range(5)]
            Q[a, b] = _group_sums(g, shifts[a] + shifts[b], P, G)
    return ok.sum(0), S, Q


def _ld(f):
    """A Fraction in long double, whose range holds every result here (about 2^-2200 to 2^2050 n)."""
    if f == 0:
        return LD(0.0)
    n, d = abs(f.numerator), f.denominator
    k = n.bit_length() - d.bit_length() - 64
    v = np.ldexp(LD((n >> k) // d if k >= 0 else (n << -k) // d), k)
    return -v if f < 0 else v


def _round(f):
    """A Fraction rounded once to f64 (Fraction -> float is correctly rounded); beyond DBL_MAX its long double value."""
    try:
        return LD(float(f))
    except OverflowError:
        return _ld(f)


def exact_stats(x):
    """x [M, G] -> the exact reference per group: n, mean, m2 (long double, see _round), sd = the exact sqrt(m2 / n)
    unrounded (the spread the bounds scale with: m2 of subnormal data underflows in f64, its spread does not), mn, mx,
    s = max|x| (f64)."""
    x = np.asarray(x, dtype=np.float64)
    ok = np.isfinite(x)
    n, S, Q = _sums(x[..., None], ok)
    G = x.shape[1]
    mean, m2, var = (np.full(G, LD(np.nan)) for _ in range(3))
    for g in range(G):
        k = int(n[g])
        if k:
            mean[g] = _round(Fraction(S[0][g], k << 1074))
            f = Fraction(k * Q[0, 0][g] - S[0][g] ** 2, k << 2148)
            m2[g], var[g] = _round(f), _ld(f / k)
    xf = np.where(ok, x, np.nan)
    if x.shape[0] == 0:
        mn = mx = s = np.full(G, np.nan)
    else:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            mn, mx, s = np.nanmin(xf, 0), np.nanmax(xf, 0), np.nanmax(np.abs(xf), 0)
    return dict(n=n.astype(np.float64), mean=mean, m2=m2, sd=np.sqrt(var), mn=mn, mx=mx, s=np.nan_to_num(s))


def exact_cov(X):
    """X [M, G, p] -> the exact record per group over the complete rows: n, mean [G, p], M [G, p, p] (long double, see
    _round), sd [G, p] = the exact sqrt(M_aa / n) unrounded and s [G, p] = max|x_a| over those rows."""
    X = np.asarray(X, dtype=np.float64)
    M_, G, p = X.shape
    ok = np.isfinite(X).all(-1)
    n, S, Q = _sums(X, ok)
    mean, var, Mm = np.full((G, p), LD(np.nan)), np.full((G, p), LD(np.nan)), np.full((G, p, p), LD(np.nan))
    for g in range(G):
        k = int(n[g])
        if not k:
            continue
        for a in range(p):
            mean[g, a] = _round(Fraction(S[a][g], k << 1074))
            for b in range(a, p):
                f = Fraction(k * Q[a, b][g] - S[a][g] * S[b][g], k << 2148)
                Mm[g, a, b] = Mm[g, b, a] = _round(f)
                if a == b:
                    var[g, a] = _ld(f / k)
    s = np.max(np.where(ok[..., None], np.abs(X), 0.0), axis=0, initial=0.0)
    return dict(n=n.astype(np.float64), mean=mean, M=Mm, sd=np.sqrt(var), s=s)


# --------------------------------------------------------------------------- the contract


def _report(bad, what, mask):
    if np.any(mask):
        bad.append(f"{what}: {int(np.sum(mask))} groups, first {np.flatnonzero(mask.ravel())[0]}")


def stats_violations(got, ref):
    """got [G, 5] against exact_stats: the rules the table breaks (empty if none)."""
    bad = []
    n = ref["n"]
    if not np.array_equal(got[:, 0], n):
        return [f"R1 count: {np.flatnonzero(got[:, 0] != n)[:5]}"]
    empty = n == 0
    _report(bad, "R1 a group without finite values is not NaN", empty & ~np.all(np.isnan(got[:, 1:]), axis=1))
    full = ~empty
    _report(bad, "R1 min", full & (got[:, 3] != ref["mn"]))
    _report(bad, "R1 max", full & (got[:, 4] != ref["mx"]))
    s = ref["s"].astype(LD)
    top = (s > TOP) | (ref["m2"] > TOP)
    with np.errstate(all="ignore"):
        mean = got[:, 1].astype(LD)
        fin = np.isfinite(mean)
        _report(bad, "R2 mean", full & fin & ~(np.abs(mean - ref["mean"]) <= LD(1e-13) * s))
        _report(bad, "R3 mean", full & ~fin & ~top)
        m2 = got[:, 2].astype(LD)
        fin = np.isfinite(m2)
        nl = n.astype(LD)
        sg, sr = np.sqrt(m2 / nl), np.sqrt(ref["m2"] / nl)
        _report(bad, "R2 std", full & fin & ~(np.abs(sg - sr) <= LD(1e-8) * ref["sd"] + LD(32 * EPS) * s))
        _report(bad, "R3 m2", full & ~fin & ~top)
        _report(bad, "R4 m2", full & (s <= EDGE) & (ref["m2"] > DBL_MAX) & ~(m2 == np.inf))
    return bad


def cov_violations(got, ref):
    """got [G, 1 + p + p*p] against exact_cov: the rules the table breaks (empty if none)."""
    bad = []
    p = ref["s"].shape[-1]
    n = ref["n"]
    if not np.array_equal(got[:, 0], n):
        return [f"R1 count: {np.flatnonzero(got[:, 0] != n)[:5]}"]
    empty = n == 0
    _report(bad, "R1 a group without complete worlds is not NaN", empty & ~np.all(np.isnan(got[:, 1:]), axis=1))
    Mg = got[:, 1 + p:].reshape(-1, p, p)
    _report(bad, "R1 M[b][a] has other bits than M[a][b]",
            np.any(Mg.view(np.int64) != np.swapaxes(Mg, 1, 2).view(np.int64), axis=(1, 2)))
    full = ~empty
    s = ref["s"].astype(LD)
    diag = np.diagonal(ref["M"], axis1=1, axis2=2)
    top_a = (s > TOP) | (diag > TOP)
    with np.errstate(all="ignore"):
        mean = got[:, 1:1 + p].astype(LD)
        fin = np.isfinite(mean)
        _report(bad, "R2 mean", full[:, None] & fin & ~(np.abs(mean - ref["mean"]) <= LD(1e-13) * s))
        _report(bad, "R3 mean", full[:, None] & ~fin & ~top_a)
        nl = n.astype(LD)[:, None, None]
        Cg, Cr = Mg.astype(LD) / nl, ref["M"] / nl
        sig = ref["sd"]
        bound = LD(1e-8) * sig[:, :, None] * sig[:, None, :] + \
            LD(32 * EPS) * (s[:, :, None] * sig[:, None, :] + sig[:, :, None] * s[:, None, :])
        fin = np.isfinite(Cg)
        f3 = full[:, None, None]
        _report(bad, "R2 M", f3 & fin & ~(np.abs(Cg - Cr) <= bound))
        _report(bad, "R3 M", f3 & ~fin & ~(top_a[:, :, None] | top_a[:, None, :]))
        gd = np.diagonal(Mg, axis1=1, axis2=2)
        _report(bad, "R4 M_aa", full[:, None] & (s <= EDGE) & (diag > DBL_MAX) & ~(gd == np.inf))
    return bad


def assert_clear_of_the_edge(m2):
    """The catalogue keeps every exact m2 (M_aa) a factor 2 away from DBL_MAX, so rounding cannot decide R4."""
    m2 = np.asarray(m2)
    assert not np.any((m2 > DBL_MAX / 2) & (m2 < LD(DBL_MAX) * 2)), "a group's exact m2 is too close to DBL_MAX"


# --------------------------------------------------------------------------- data


def diverging(M):
    """A plane that diverged in all worlds but one: m2 = 6.2e306, but (sum of 8 deviations)^2 overflows."""
    x = np.full(M, 2.5e153)
    x[0] = 0.0
    return x


def alternating(M, J):
    """+-1e155, the sign flipping every J worlds (so every thread of stride J sees both): m2 = M 1e310 > DBL_MAX."""
    return np.where((np.arange(M) // J) % 2 == 0, 1e155, -1e155)


def catalogue(M, E, J, wc, seed=0):
    """[M, E, 25] planes, the data of every shape.  J: the flip period of the alternating plane; wc: the chunk length
    the non-finite run of plane 6 spans twice, so that a chunk between two others has no finite world."""
    rng = np.random.default_rng(seed)
    sh = (M, E)
    x = np.empty((M, E, 25))
    x[..., 0] = rng.normal(3.0, 2.0, sh)                                      # normal
    x[..., 1] = 6.4e6 + rng.normal(0.0, 6.4, sh)                              # |mean| / sigma = 1e6
    x[..., 2] = 1.25                                                          # all equal
    x[..., 3] = rng.choice([1.0, 2.0, 3.0], sh)                               # heavy ties
    x[..., 4] = rng.choice([0.0, -0.0, 5e-324, -5e-324, 2.2e-308], sh)        # signed zeros and subnormals
    x[: 2, :, 4] = [[2.2e-308], [-2.2e-308]][: M]
    x[..., 5] = rng.normal(0.0, 1.0, sh)                                      # NaN and +-inf worlds
    bad = rng.random(sh) < 0.1
    x[..., 5][bad] = rng.choice([np.nan, np.inf, -np.inf], int(bad.sum()))
    x[..., 6] = rng.normal(-2.0, 0.5, sh)                                     # a run of non-finite worlds
    x[wc // 2: wc // 2 + 2 * wc, :, 6] = np.nan
    x[..., 7] = diverging(M)[:, None]                                         # the two overflow planes
    x[..., 8] = alternating(M, J)[:, None]
    big = rng.random(sh) < 0.5                                                # 1e150 and 1e300 modes: m2 beyond DBL_MAX
    x[..., 9] = np.where(big, 1e300, 1e150) * rng.choice([-1.0, 1.0], sh) * (1.0 + 0.5 * rng.random(sh))
    x[: 2, :, 9] = [[1.2e300], [-1e150]][: M]
    x[..., 10] = rng.choice([-1e150, 1e150], sh) * (1.0 + 0.1 * rng.normal(size=sh))  # bimodal, finite m2
    x[..., 11] = rng.choice([DBL_MAX, -DBL_MAX], sh)                          # +-DBL_MAX
    x[: 2, :, 11] = [[DBL_MAX], [-DBL_MAX]][: M]
    x[..., 12] = 0.5 * x[..., 0] + rng.normal(0.0, 0.1, sh)                   # correlated with 0
    x[..., 13] = -3.1e6 + 0.9 * (x[..., 1] - 6.4e6) + rng.normal(0.0, 2.8, sh)  # with 1, at 1e6 sigma
    x[..., 14] = 1e-3 * rng.exponential(1.0, sh)
    x[..., 15] = 2.5e153                                                      # diverged but the last world
    x[-1, :, 15] = -1e153
    x[..., 16] = alternating(M, 1)[:, None] * 0.3                             # +-3e154 flipping every world
    x[..., 17] = 1e100 * rng.normal(size=sh)
    x[..., 18] = rng.uniform(-1.0, 1.0, sh)
    x[..., 19] = rng.normal(0.0, 1e-5, sh)
    x[..., 20] = -0.0
    x[..., 21] = np.where(rng.random(sh) < 1e-3, -3.0, 2.0)
    x[..., 22] = 7.0e5 + rng.exponential(1.0, sh)
    x[..., 23] = rng.normal(0.0, 1.0, sh)
    x[..., 24] = 1e3 + 1e-3 * rng.normal(size=sh)
    return x


def state_call(x, call):
    """Upload x [M, E, 25] as the state planes of a fresh handle in each math mode and run call(ex) there; returns
    (result, launches of the call, quantile_reads()), the same in both modes."""
    M, E, _ = x.shape
    ine = np.broadcast_to(np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 1.0]), (M, E, 7))
    out = []
    for mode in MODES:
        with el.B200Exec(E, M, 0.01, None, [], "rk4", mode) as ex:
            ex.set_state(x[..., :7], x[..., 7:13], ine, accel=x[..., 13:19], force=x[..., 19:25])
            n0 = ex.timings()["kernel_launches"]
            got = call(ex)
            out.append((got, ex.timings()["kernel_launches"] - n0, ex.quantile_reads()))
    (a, la, ra), (b, lb, rb) = out
    assert a.tobytes() == b.tobytes() and la == lb and ra == rb, "the math mode changed a reduction"
    return a, la, ra


# --------------------------------------------------------------------------- CPU: the reference


def test_exact_reference_equals_fsum_on_ordinary_data():
    rng = np.random.default_rng(0)
    x = np.stack([rng.normal(3.0, 2.0, 5000), 6.4e6 + rng.normal(0.0, 6.4, 5000), rng.choice([1.0, 2.0], 5000),
                  1e-3 * rng.exponential(1.0, 5000), rng.normal(0.0, 1e100, 5000)], 1)
    x[::97, 0] = np.nan
    ref, fs = exact_stats(x), fsum_stats_table(x)
    assert np.array_equal(ref["n"], fs[:, 0]) and np.array_equal(ref["mn"], fs[:, 3])
    assert np.all(np.abs(ref["mean"] - fs[:, 1].astype(LD)) <= LD(EPS) * np.abs(fs[:, 1]))  # fsum rounds twice
    assert np.all(np.abs(ref["m2"] - fs[:, 2].astype(LD)) <= LD(1e-13) * fs[:, 2])
    X = x[:, None, :]
    cr, cf = exact_cov(X), fsum_cov_table(X, range(5))
    assert cr["n"][0] == cf[0, 0]
    assert np.all(np.abs(cr["mean"][0] - cf[0, 1:6].astype(LD)) <= LD(EPS) * np.abs(cf[0, 1:6]))
    Mf = cf[0, 6:].reshape(5, 5).astype(LD)
    sig = np.sqrt(np.diagonal(Mf))
    assert np.all(np.abs(cr["M"][0] - Mf) <= LD(1e-13) * sig[:, None] * sig[None, :])


def test_exact_reference_closed_forms():
    for a in (3.0, 1e-160, 5e-324, 1e150, 1e154, 1e300, DBL_MAX):
        r = exact_stats(np.array([[-a], [a]]))
        assert r["mean"][0] == 0.0
        want = _round(2 * Fraction(a) ** 2)
        assert r["m2"][0] == want and (want > DBL_MAX) == (a >= 1e154)
    for M in (2, 9, 65539):
        v = 2.5e153
        r = exact_stats(diverging(M)[:, None])
        assert r["m2"][0] == _round(Fraction(v) ** 2 * (M - 1) / M)
        assert r["mean"][0] == _round(Fraction(v) * (M - 1) / M)
    a, b = 3e154, -7.0
    c = exact_cov(np.array([[[-a, -b]], [[a, b]]]))
    assert c["M"][0, 0, 1] == c["M"][0, 1, 0] == _round(2 * Fraction(a) * Fraction(b))
    assert c["M"][0, 0, 0] == _round(2 * Fraction(a) ** 2) > DBL_MAX and c["M"][0, 1, 1] == 98.0
    assert exact_cov(np.array([[[np.nan, 1.0]]]))["n"][0] == 0


# --------------------------------------------------------------------------- CPU: the old arithmetic fails the contract


def _empty_groups(k):
    return dict(n=np.zeros(k), mean=np.zeros(k), m2=np.zeros(k))


def _merge(a, b):
    """stats_merge / cov_merge (one plane), vectorised: a := a (+) b."""
    with np.errstate(all="ignore"):
        n = a["n"] + b["n"]
        d = b["mean"] - a["mean"]
        mean = a["mean"] + d * b["n"] / n
        m2 = a["m2"] + b["m2"] + d * d * a["n"] * b["n"] / n
    r = dict(n=n, mean=mean, m2=m2)
    return {k: np.where(b["n"] == 0, a[k], np.where(a["n"] == 0, b[k], r[k])) for k in r}


def _shifted(lanes, fixed):
    """Shifted::add over the columns of lanes [L, k] (NaN: no value), then Shifted::group / the diagonal of the
    covariance chunk record; the sum of squares without the kernel's fma (rounding only, not overflow, differs)."""
    L = lanes.shape[0]
    n, K, s1, s2 = np.zeros(L), np.zeros(L), np.zeros(L), np.zeros(L)
    with np.errstate(all="ignore"):
        for v in lanes.T:
            ok = np.abs(v) <= DBL_MAX
            K = np.where(ok & (n == 0), v, K)
            y = np.where(ok, v - K, 0.0)
            s1, s2, n = s1 + y, s2 + y * y, n + ok
        mean = K + s1 / n
        if fixed:
            m2 = np.where(s2 > DBL_MAX, np.inf, np.fmax(s2 - s1 * (s1 / n), 0.0))
        else:
            m2 = np.fmax(s2 - s1 * s1 / n, 0.0)
    return dict(n=n, mean=np.where(n > 0, mean, 0.0), m2=np.where(n > 0, m2, 0.0))


def restated_stats(x, fixed):
    """stats_kernels.cu on one group of one entity, x [M]: a lane per j < J takes worlds w0 + j, w0 + j + J, ... of
    its chunk, the J lanes merge in the binary tree, the chunks left to right -> (n, mean, m2)."""
    M = x.size
    J, Wc, C = stats_shape(M, 1)
    acc = _empty_groups(1)
    for c in range(C):
        chunk = np.full(Wc, np.nan)
        part = x[c * Wc: (c + 1) * Wc]
        chunk[: part.size] = part
        g = _shifted(chunk.reshape(Wc // J, J).T, fixed)
        s = 1
        while s < J:
            j = np.arange(0, J - s, 2 * s)
            m = _merge({k: v[j] for k, v in g.items()}, {k: v[j + s] for k, v in g.items()})
            for k in g:
                g[k][j] = m[k]
            s *= 2
        acc = _merge(acc, {k: v[:1] for k, v in g.items()})
    return np.array([[acc["n"][0], acc["mean"][0], acc["m2"][0], np.min(x), np.max(x)]])


def restated_cov_diagonal(x, fixed):
    """cov_kernels.cu at p = 1 on one group x [M]: the chunk records (shift = the chunk's first world, one thread walks
    the chunk in order), folded left to right with cov_merge -> the record (n, mean, M)."""
    M = x.size
    Wc, C = cov_chunks(M, 1)
    chunks = np.full(C * Wc, np.nan)
    chunks[:M] = x
    recs = _shifted(chunks.reshape(C, Wc), fixed)
    acc = _empty_groups(1)
    for c in range(C):
        acc = _merge(acc, {k: v[c:c + 1] for k, v in recs.items()})
    return np.array([[acc["n"][0], acc["mean"][0], acc["m2"][0]]])


def test_contract_rejects_the_old_chunk_arithmetic():
    """At (65539, 1), a shape the suite already ran, one world at 0 and 65538 at 2.5e153 (m2 = 6.2e306); and +-1e155
    alternating in the order a thread reads them (m2 > DBL_MAX), at 65536 worlds for the statistics (eight values a
    lane) and 65472 for the covariance (chunks of 124 worlds), where every chunk's mean is 0 and no merge overflows.
    The old s2 - s1 * s1 / n gives a finite spread 8x too small on the first and 0 on the second; s2 - s1 * (s1 / n)
    with +inf for an overflowed s2 keeps the contract on both."""
    M = 65539
    assert stats_shape(65536, 1)[:2] == (256, 2048) and cov_chunks(65472, 1) == (124, 528)
    cases = [("stats", diverging(M)), ("stats", alternating(65536, 256)),
             ("cov", diverging(M)), ("cov", alternating(65472, 1))]
    for kernel, x in cases:
        want = exact_stats(x[:, None])
        if kernel == "stats":
            old, new = restated_stats(x, False), restated_stats(x, True)
            check = lambda t: stats_violations(t, want)
        else:
            ref = exact_cov(x[:, None, None])
            old, new = restated_cov_diagonal(x, False), restated_cov_diagonal(x, True)
            check = lambda t: cov_violations(t, ref)
        assert any(v.startswith(("R2", "R4")) for v in check(old)), (kernel, old)
        assert check(new) == [], (kernel, new, check(new))
    # the issue's numbers: the old lanes lose a factor 8 of m2 on the first plane, all of it on the second
    old = restated_stats(diverging(M), False)[0, 2]
    assert 7e305 < old < 9e305 and restated_stats(alternating(65536, 256), False)[0, 2] == 0.0


def _part_tables(x, parts, stats):
    """Exact per-part tables rounded to f64 (a part's m2 beyond DBL_MAX is +inf), empty parts as count 0 + NaN."""
    out = []
    for idx in parts:
        if stats:
            r = exact_stats(x[idx])
            t = np.stack([r["n"], r["mean"].astype(np.float64), r["m2"].astype(np.float64), r["mn"], r["mx"]], -1)
            t[r["n"] == 0, 1:] = np.nan
        else:
            r = exact_cov(x[idx])
            p = x.shape[-1]
            t = np.concatenate([r["n"][:, None], r["mean"].astype(np.float64),
                                r["M"].astype(np.float64).reshape(-1, p * p)], -1)
            t[r["n"] == 0, 1:] = np.nan
        out.append(t)
    return out


@pytest.mark.parametrize("seed", range(3))
def test_host_merges_keep_the_contract_at_the_range_edge(seed):
    """b200_stats_merge and b200_covariance_merge share stats_merge and cov_merge with the kernels."""
    rng = np.random.default_rng(seed)
    M = int(rng.integers(2000, 20000))
    x = catalogue(M, 1, 64, 100, seed)[:, 0, :]                           # [M, 25]
    parts = split(rng, M, int(rng.integers(2, 9)))
    parts.insert(1, parts[0][:0])                                         # an empty part between two others
    with np.errstate(over="ignore"):
        got = el.merge_stats(_part_tables(x, parts, True))
    ref = exact_stats(x)
    assert stats_violations(got, ref) == []
    assert got[8, 2] == np.inf and got[9, 2] == np.inf                      # R4 planes
    sel = [0, 7, 8, 9, 10, 13, 15, 16]
    X = x[:, None, sel]
    with np.errstate(over="ignore"):
        gotc = el.merge_covariance(_part_tables(X, parts, False))
    assert cov_violations(gotc, exact_cov(X)) == []


# --------------------------------------------------------------------------- CPU: the sweep reaches what it aims at


STATS_CASES = ([(37, E) for E in (1, 2, 3, 128, 129, 255, 256, 257, 513)]
               + [(M, 1) for M in (2047, 2048, 2049, 65539, 126977, 129024, 131072, 131073, 147455)]
               + [(680, 3), (681, 3), (512, 257), (513, 257)])

COV_P = (1, 4, 5, 8, 9, 20, 21, 24, 25)
_PERM = tuple(np.random.default_rng(1).permutation(25).tolist())


def _selection(p, i):
    return tuple(_PERM[(5 * i + k) % 25] for k in range(p))


COV_CASES = [(65, E, _selection(p, i)) for i, (p, E) in enumerate(
    (p, E) for p in COV_P for E in (1, cov_et(p) - 1, cov_et(p), cov_et(p) + 1, 2 * cov_et(p) + 1))]
COV_CASES += [(64, cov_et(p), _selection(p, 3 * i + 1)) for i, p in enumerate(COV_P)]
COV_CASES += [(65, 129, (0, 7, 8, 23)),                                   # 5 entity tiles
              (65539, 1, (7, 8, 16)),                                     # the overflow planes at a shape the suite ran
              (33792, 1, (6, 7, 8, 16, 9)),                               # C = kChunkTasks, empty chunks
              (6784, 129, (6, 0, 12, 1, 13, 7, 16, 10, 4))]               # C = 106, not a multiple of kMergeBatch

QUANTILE_ROUTE_WORLDS = (256, 257, 4097, 8192, 8193)
QUANTILE_RADIX_ENTITIES = (2, 60, 257)


def test_sweep_reaches_every_boundary():
    st = {(M, E): stats_shape(M, E) for M, E in STATS_CASES}
    Cs = {C for J, Wc, C in st.values()}
    assert {1, 2, 63, 64} <= Cs
    assert any(C == 64 and M % Wc and E == 1 for (M, E), (J, Wc, C) in st.items())  # a short last chunk at C = 64
    assert any(Wc // J > 8 for J, Wc, C in st.values())                            # per > kMinPerThread
    assert any(C == 64 and E > 256 for (M, E), (J, Wc, C) in st.items())           # two tiles at 64 chunks
    assert st[(37, 129)][0] == 1 and 256 % 3 == 1                                   # J = 1; an idle lane at E = 3
    ps = {len(sel) for M, E, sel in COV_CASES}
    assert set(COV_P) <= ps and cov_et(20) == 32 and cov_et(21) == 16
    for p in COV_P:
        Es = {E for M, E, sel in COV_CASES if len(sel) == p}
        et = cov_et(p)
        assert {1, et - 1, et, et + 1, 2 * et + 1} <= Es
    cc = {(M, E): cov_chunks(M, E)[1] for M, E, sel in COV_CASES}
    assert cc[(64, 32)] == 1 and cc[(65, 32)] == 2 and 528 in cc.values()
    assert any(C % 8 and C > 8 for C in cc.values())
    assert 6 in COV_CASES[-1][2] and 6 in COV_CASES[-2][2]                          # the run: chunks without worlds
    assert [quantile_launches(M, 3) for M in QUANTILE_ROUTE_WORLDS] == [1, 1, 1, 1, 18]
    assert [M <= WARP_MAX for M in QUANTILE_ROUTE_WORLDS] == [True, False, False, False, False]
    assert [quantile_launches(8193, E) for E in QUANTILE_RADIX_ENTITIES] == [18, 36, 90]
    assert pass_shape(8193, 257, 5)[2] == 2                                         # a second tile of one entity
    assert SLICE_GROUPS == 1354 and quantile_launches(8193, SLICE_GROUPS + 1) == 18 * 50


def test_catalogue_keeps_clear_of_the_edge():
    for M, E in ((37, 3), (2049, 1)):
        x = catalogue(M, E, stats_shape(M, E)[0], stats_shape(M, E)[1])
        ref = exact_stats(x.reshape(M, -1))
        assert_clear_of_the_edge(ref["m2"])
        R4 = set(np.flatnonzero(((ref["s"] <= EDGE) & (ref["m2"] > DBL_MAX)).reshape(E, 25)[0]))
        # the planes that must read +inf (the alternating plane 8 flips every J = 85 worlds: not within 37)
        assert R4 == ({9, 16} if M < stats_shape(M, E)[0] else {8, 9, 16})


# --------------------------------------------------------------------------- GPU: statistics


@pytest.mark.gpu
@pytest.mark.parametrize("shape", STATS_CASES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_state_stats_sweep(shape):
    need_gpu()
    M, E = shape
    J, Wc, C = stats_shape(M, E)
    x = catalogue(M, E, J, Wc)
    got, launches, _ = state_call(x, lambda ex: ex.state_stats())
    assert launches == stats_launches(M, E), (launches, C)
    ref = exact_stats(x.reshape(M, -1))
    assert_clear_of_the_edge(ref["m2"])
    assert stats_violations(got.reshape(-1, 5), ref) == []


# --------------------------------------------------------------------------- GPU: covariance


@pytest.mark.gpu
@pytest.mark.parametrize("case", COV_CASES, ids=lambda c: f"{c[0]}x{c[1]}-p{len(c[2])}")
def test_state_covariance_sweep(case):
    need_gpu()
    M, E, sel = case
    Wc, C = cov_chunks(M, E)
    x = catalogue(M, E, 1, Wc, seed=len(sel))
    got, launches, _ = state_call(x, lambda ex: ex.state_covariance(sel))
    assert launches == cov_launches(M, E, len(sel)), (launches, C)
    X = x[..., list(sel)]
    ref = exact_cov(X)
    assert_clear_of_the_edge(np.diagonal(ref["M"], axis1=1, axis2=2))
    assert cov_violations(got, ref) == []
    if 6 in sel and C > 2:                                                # a chunk without a complete world
        ok = np.isfinite(X).all(-1)[:, 0]
        assert any(not ok[c * Wc:(c + 1) * Wc].any() for c in range(1, C - 1))


# --------------------------------------------------------------------------- GPU: quantiles


@pytest.mark.gpu
@pytest.mark.parametrize("M", QUANTILE_ROUTE_WORLDS)
def test_state_quantile_routes(M):
    need_gpu()
    E = 3
    x = catalogue(M, E, stats_shape(M, E)[0], 100)
    got, launches, _ = state_call(x, lambda ex: ex.state_quantiles(LEVELS16))
    assert launches == quantile_launches(M, E)
    assert got.tobytes() == ref_quantiles(x, LEVELS16).tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("E", QUANTILE_RADIX_ENTITIES)
def test_state_quantile_radix_degenerate_entities(E):
    """Entities > 1 keep the histograms in global memory and pass_shape tiles them (two tiles at 257)."""
    need_gpu()
    M = 8193
    x = _degenerate(M * E, seed=E).reshape(M, E, 25)
    got, launches, reads = state_call(x, lambda ex: ex.state_quantiles(LEVELS16))
    assert launches == quantile_launches(M, E)
    assert 1 <= reads <= 8
    assert got.tobytes() == ref_quantiles(x, LEVELS16).tobytes()


def _planes(col):
    """col [M, E] -> [M, E, 25]: every plane the same data, so that the reference sorts it once."""
    return np.broadcast_to(col[..., None], col.shape + (25,))


@pytest.mark.gpu
def test_state_quantiles_in_entity_range_slices():
    """kSliceGroups + 1 entities: each plane runs as two entity ranges, the second of one entity."""
    need_gpu()
    M, E = 8193, SLICE_GROUPS + 1
    rng = np.random.default_rng(8)
    col = np.round(rng.normal(0.0, 1.0, (M, E)) * 64) / 64
    col[rng.random((M, E)) < 0.05] = np.nan
    got, launches, _ = state_call(_planes(col), lambda ex: ex.state_quantiles(LEVELS16))
    assert launches == quantile_launches(M, E) == 18 * 25 * 2
    want = ref_quantiles(col, LEVELS16)                                   # [E, n_q]
    for k in range(25):
        assert got[:, k].tobytes() == want.tobytes(), k


def deep_refinement():
    """32 clusters of 8200 worlds on two adjacent doubles (different exponents: pass 1 puts each in its own bin), one
    world at each of +-DBL_MAX (the first range spans the whole key space), and 16 levels whose ranks i, i + 1 are the
    last of cluster 2k and the first of cluster 2k + 1.  Every cluster holds one rank, so 32 ranges refine at 9 bits a
    pass after pass 1's 14: 14 + 5 * 9 = 59 < 64 bits, and the last histogram pass is needed -> (column, levels)."""
    size = 8200
    lo = 1.5 * np.ldexp(1.0, np.arange(32) * 10 - 150)
    vals = np.concatenate([np.repeat(np.stack([lo, np.nextafter(lo, np.inf)], 1).ravel(), size // 2),
                           [DBL_MAX, -DBL_MAX]])
    n = vals.size
    ranks = [(2 * k + 1) * size for k in range(16)]                       # the last rank of cluster 2k (rank 0: -DBL_MAX)
    q = tuple((r + 0.5) / (n - 1) for r in ranks)
    assert [math.floor(float(n - 1) * v) for v in q] == ranks
    return np.random.default_rng(2).permutation(vals), q


def compaction_cap():
    """4 clusters of 7000 keys in one pass-1 bin each, a level in each: two compacted ranges fill 14000 of kGroupCap's
    16384 keys, so the other two are refined by pass 2 and compacted by pass 3 -> (column, levels)."""
    rng = np.random.default_rng(4)
    vals = np.concatenate([1.5 * np.ldexp(1.0, 20 * c) * (1.0 + rng.random(7000) / 8) for c in range(4)]
                          + [[DBL_MAX, -DBL_MAX]])
    n = vals.size
    q = tuple((1 + 7000 * c + 3500.25) / (n - 1) for c in range(4))
    return rng.permutation(vals), q


@pytest.mark.gpu
def test_state_quantiles_need_every_histogram_pass():
    need_gpu()
    col, q = deep_refinement()
    got, launches, reads = state_call(_planes(col[:, None]), lambda ex: ex.state_quantiles(q))
    assert launches == 18 and reads == 8
    assert got.tobytes() == ref_quantiles(_planes(col[:, None]), q).tobytes()


@pytest.mark.gpu
def test_state_quantiles_refine_past_the_compaction_cap():
    need_gpu()
    col, q = compaction_cap()
    got, launches, reads = state_call(_planes(col[:, None]), lambda ex: ex.state_quantiles(q))
    assert launches == 18 and reads == 4                                  # count, histogram, compact + refine, compact
    assert got.tobytes() == ref_quantiles(_planes(col[:, None]), q).tobytes()
