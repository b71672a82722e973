"""The time-axis kernels of ensemble mode (the run-summary fold, the channel pass and the outcome pass) at every boundary
of their launch geometry, every condition slot and the edges of the f64 range, against the numpy references of
test_run_summary, test_run_scores and test_ensemble_channels.

Geometry.  launch_summary_fold (grid (ceil(n_bodies / 256), n_planes), n_planes the union summary_params builds),
launch_summary_clear, launch_channels (bx, by, and the samples each block row walks) and body_table_download (chunks
of floor(2^28 / per_body) bodies through the staging buffer, one launch for a device destination) are restated below
(kNumSMs = 132).  The sweep takes each boundary and its neighbours: 1, 255, 256, 257 and 2^16 + 3 bodies with entity
counts that do not divide 256, 1 to 9 rows per fold (every n_rows % 4 after a full unrolled iteration), rows of 25,
26 and 33 planes, 8 thresholds and 8 dwells on one (entity, plane), every spec combination that picks an
instantiation, a 65,537-row fold in which the channel pass loops over its samples, and downloads that end in a
one-body chunk.  Every case asserts the launch count its restated geometry predicts.  The fold takes no math mode,
so the sweep runs in one mode; the Exec case runs in both.

Arithmetic.  The catalogue puts hand-made row sequences through the state route (set_state, then summary_add_state,
then one tick so that the next row gets a new label): signed zeros, ties, subnormals, +-DBL_MAX, NaN payloads, +-inf,
leading non-finite rows, K = -DBL_MAX then +DBL_MAX, S1 overflowing to +inf and then to NaN, sums whose
S2 - S1 (S1 / n) rounds below 0, and offset data.  For every (world, entity, plane), with n the finite rows, K the
first of them, y_i = x_i - K exactly, S1 = sum y_i, s = max |x_i|, mu and m2 the exact rational mean and
sum (x_i - mu)^2, u = 2^-53 and gamma_k = k u / (1 - k u):
  R1  extrema, threshold events, dwells and the moment count equal the numpy fold exactly; mean and m2 equal
      ref_moments bit for bit (the payload of a NaN the arithmetic makes is not part of the contract).
  R2  a finite mean is within gamma_{n+2} sum |y_i| / n + u |mu| + 2^-1074 of mu, a finite m2 within
      gamma_{2n+8} (sum y_i^2 + S1^2 / n) + (n + 2) 2^-1074 of m2.
  R3  a non-finite mean or m2 with n > 0 appears only where s > 2^990 or m2 > 2^990.
  R4  where every |x_i| <= 2^1000 and m2 > DBL_MAX, the table's m2 is +inf and its mean is finite and keeps R2.
The bounds of R2 follow from the standard model fl(a op b) = (a op b)(1 + d) + e, |d| <= u, with e = 0 for sums and
|e| <= 2^-1075 for products and quotients (subnormal results).  The computed y_i carries one rounding and S1 n - 1 more,
so |S1^ - S1| <= gamma_n sum |y_i|; K + S1^ / n adds two roundings, hence the mean's bound.  S2 carries gamma_{n+2}
sum y_i^2; S1^ (S1^ / n) is within gamma_{n+3} (S1^2 / n + sum y_i^2) + gamma_n^2 sum y_i^2 of S1^2 / n (by
2 |S1| sum |y_i| / n <= S1^2 / n + sum y_i^2); the last subtraction adds u sum y_i^2; the clamp at 0 only moves m2
towards the exact value, which is >= 0.  The bounds grow with n: a 65k-row sequential sum is not held to the fixed
1e-13 s of the world-axis reductions.  The outcome pass then turns these summaries into 25 outcome planes of every
kind and field, which equal a numpy restatement of the downloaded tables bit for bit.

Sensitivity.  fold_model restates the fold over a sequence of folds; with one fault at a time it must fail a catalogue
or geometry case, so each reference and bound above is known to catch it."""

import math
from fractions import Fraction

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200.executor import WORLD_POS
from tests.ensemble_util import ROCKET, handle, need_gpu, rocket_world, sampled_state
from tests.test_ensemble_channels import CHANNELS, check_values, records, ref_channels
from tests.test_ensemble_histograms import state_handle
from tests.test_run_scores import bits, ref_dwell, ref_moments
from tests.test_run_summary import ref_tables, ref_threshold

DBL_MAX = np.finfo(np.float64).max
INF = np.inf
U = Fraction(1, 2 ** 53)
TINY = Fraction(1, 2 ** 1074)
TOP = 2.0 ** 990    # R3
EDGE = 2.0 ** 1000  # R4
MODES = ("exact", "fast")

# --------------------------------------------------------------------------- the launch geometry, restated

NUM_SMS = 132
THREADS = 256
STAGING = 256 << 20


def cdiv(a, b):
    return -(-a // b)


def fold_planes(R, extrema, thresholds=(), moments=(), dwells=()):
    """sixdof_abi.cu summary_params -> (planes, mom_slot): the planes a fold reads, in plane order, and the moment slot
    of each (None = kNoMoment)."""
    planes, slots = [], []
    for p in range(R):
        used = extrema or any(t[1] == p for t in thresholds) or any(d[1] == p for d in dwells)
        slot = list(moments).index(p) if p in moments else None
        if used or slot is not None:
            planes.append(p)
            slots.append(slot)
    return planes, slots


def fold_grid(n_bodies, planes):
    """summary_kernels.cu launch_summary_fold: the grid, (0, 0) when nothing is launched."""
    if n_bodies == 0 or not planes:
        return 0, 0
    return cdiv(n_bodies, THREADS), len(planes)


def fold_scores(moments, dwells):
    """The kScores = true instantiation: moments or dwells in the spec."""
    return bool(moments) or bool(dwells)


def clear_launches(extrema, n_thr, moments, dwells):
    """launch_summary_clear: one launch for extrema / thresholds, one for moments / dwells."""
    return int(bool(extrema) or n_thr > 0) + int(bool(moments) or bool(dwells))


def channel_shape(n_bodies, n_samples):
    """channel_kernels.cu launch_channels -> (bx, by, samples per block row at most)."""
    bx = cdiv(n_bodies, THREADS)
    by = min(n_samples, max(1, min(65535, 64 * NUM_SMS * 8 // bx)))
    return bx, by, cdiv(n_samples, by)


def download_chunks(n_bodies, per_body, direct):
    """sixdof_abi.cu body_table_download -> (chunks = launches, bodies in the last chunk)."""
    chunk = n_bodies if direct else max(1, min(n_bodies, STAGING // per_body))
    n = cdiv(n_bodies, chunk)
    return n, n_bodies - (n - 1) * chunk


def fold_launches(n_rows, n_c, planes):
    """One summary_add_*: the channel refresh where the fold reads a channel plane, then the fold."""
    if n_rows == 0 or not planes:
        return 0
    return int(n_c > 0 and max(planes) >= 25) + 1


# --------------------------------------------------------------------------- the sweep

COMBOS = ("all", "extrema", "thresholds", "moments", "dwells", "moments_all")


def cond_plane(n_c):
    return {0: 24, 1: 25, 8: 32}[n_c]


def combo_spec(combo, R, conds, moments):
    """(extrema, thresholds, moments, dwells) of a combination."""
    return {"all": (True, conds, moments, conds), "extrema": (True, [], [], []), "thresholds": (False, conds, [], []),
            "moments": (False, [], moments, []), "dwells": (False, [], [], conds),
            "moments_all": (False, [], list(range(R))[::-1], [])}[combo]


def case_moments(R):
    """Moments on planes 24, 25 and 32 where the row has them, out of plane order."""
    return [p for p in (32, 6, 24, 25, 0) if p < R]


# (n_worlds, n_entities, n_channels, every, ticks before the reset, rows in the ring fold, combination)
SWEEP = [
    (1, 1, 0, 1, 0, 1, "all"),
    (85, 3, 1, 1, 0, 2, "thresholds"),
    (256, 1, 8, 3, 4, 3, "all"),
    (257, 1, 0, 1, 0, 4, "moments"),
    (37, 7, 1, 3, 2, 5, "dwells"),
    (1, 300, 8, 1, 0, 6, "moments_all"),
    (2, 300, 0, 3, 1, 8, "extrema"),
    (65539, 1, 8, 1, 0, 9, "all"),
    (128, 2, 1, 1, 0, 7, "all"),
    (255, 1, 8, 3, 5, 9, "moments_all"),
]
LONG = (1, 1, 8, 1, 0, 65537, "all")
CHUNKED = [((1 << 28) // 1000 + 1, 0, "extrema"), ((1 << 28) // 792 + 1, 8, "moments_all")]


def case_id(c):
    M, E, n_c, every, pre, n, combo = c
    return f"{M}x{E}-c{n_c}-e{every}p{pre}-r{n}-{combo}"


def test_sweep_reaches_every_boundary():
    bodies = {M * E for M, E, *_ in SWEEP}
    assert {1, 255, 256, 257, (1 << 16) + 3} <= bodies
    assert {3, 7, 300} <= {E for _, E, *_ in SWEEP if 256 % E}
    grids = {fold_grid(M * E, [0])[0] for M, E, *_ in SWEEP}
    assert {1, 2, 257} <= grids                                     # one block, one straddling block, many
    rows = {c[5] for c in SWEEP}
    assert {1, 2, 3, 4, 5, 8, 9} <= rows
    assert {n % 4 for n in rows if n >= 4} == {0, 1, 2, 3}            # every tail after a full unrolled iteration
    assert any(every == 3 and pre % every for _, _, _, every, pre, *_ in SWEEP)
    assert {0, 1, 8} == {c[2] for c in SWEEP}
    assert {24, 25, 32} == {cond_plane(c[2]) for c in SWEEP}
    assert set(COMBOS) == {c[6] for c in SWEEP}
    # every instantiation and every early-out of the kernel: extrema only, thresholds only (kScores = false, ext null),
    # moments only, dwells only (kScores = true, ext null), all four, and moments on every plane of a 33-plane row
    insts = set()
    for M, E, n_c, _, _, _, combo in SWEEP:
        R = 25 + n_c
        conds = [(E - 1, cond_plane(n_c), True, 0.0)] * 8
        ext, thr, mom, dw = combo_spec(combo, R, conds, case_moments(R))
        planes, slots = fold_planes(R, ext, thr, mom, dw)
        insts.add((ext, bool(thr), fold_scores(mom, dw)))
        if combo == "moments_all":
            assert planes == list(range(R)) and sorted(slots) == list(range(R))
            if R == 33:
                assert fold_grid(M * E, planes)[1] == 33
        assert clear_launches(ext, len(thr), mom, dw) == 1 + int(combo == "all")
    assert {(True, False, False), (False, True, False), (False, False, True), (True, True, True)} <= insts
    # the long fold: one body, by = 65535 < 65537 samples, so block row 0 takes a second sample inside the grid
    M, E, n_c, every, _, n, _ = LONG
    assert n >= 65537 and channel_shape(M * E, n) == (1, 65535, 2)
    assert all(channel_shape(M * E, c[5] + 1)[2] == 1 for c in SWEEP)  # the sweep alone never loops
    assert 65537 * 25 * 128 * 8 + 65537 * 8 * 128 * 8 < 2.3e9     # the ring and its channel planes, in bytes
    # chunked downloads end in a one-body chunk on the host route, one launch on the device route
    for nb, n_c, combo in CHUNKED:
        per = 5 * 25 * 8 if combo == "extrema" else 3 * (25 + n_c) * 8
        assert download_chunks(nb, per, False) == (2, 1) and download_chunks(nb, per, True) == (1, nb)
        assert download_chunks(nb - 1, per, False) == (1, nb - 1)
    assert download_chunks(268436, 1000, False) == (2, 1) and download_chunks(338934, 792, False) == (2, 1)


# --------------------------------------------------------------------------- the fold, restated with faults

FAULTS = ("le_minmax", "ge_condition", "nan_below", "k_reset", "nonfinite_counted", "no_clamp", "k_zero",
          "last_tick_min", "skip_tail", "tick_off")


@np.errstate(over="ignore", invalid="ignore", divide="ignore")
def fold_model(folds, thresholds, dwells, fault=None):
    """folds = [(rows [r, M, E, P], tick0, tick_step), ...] folded in order -> (extrema [M, E, P, 5], threshold ticks
    [M, T], moments [M, E, P, 3], dwells [M, D, 3]): summary_fold_kernel written out row by row, with `fault`."""
    shape = folds[0][0].shape[1:]
    M = shape[0]
    mn, mx = np.full(shape, np.nan), np.full(shape, np.nan)
    mn_t, mx_t, nf_t = (np.full(shape, -1.0) for _ in range(3))
    best = np.full((M, len(thresholds)), -1.0)
    n, K, S1, S2 = (np.zeros(shape) for _ in range(4))
    dw = np.zeros((M, len(dwells), 3))
    dw[..., 1:] = -1.0

    def hit(x, above, value):
        if fault == "ge_condition":
            f = x >= value if above else x <= value
        else:
            f = x > value if above else x < value
        if fault == "nan_below" and not above:
            f = f | np.isnan(x)
        return f

    for rows, tick0, step in folds:
        kset = np.zeros(shape, bool) if fault == "k_reset" else n > 0
        cnt = np.zeros((M, len(dwells)))
        first, last = np.full((M, len(dwells)), -1.0), np.full((M, len(dwells)), -1.0)
        todo = len(rows) // 4 * 4 if fault == "skip_tail" else len(rows)
        for r in range(todo):
            x = rows[r]
            t = float(tick0 + (r + (fault == "tick_off")) * step)
            fin = np.isfinite(x)
            newk = fin & ~kset
            K = np.where(newk, 0.0 if fault == "k_zero" else x, K)
            kset = kset | fin
            y = x - K
            S1 = np.where(fin, S1 + y, S1)
            S2 = np.where(fin, S2 + y * y, S2)
            n = n + (1.0 if fault == "nonfinite_counted" else fin)
            if fault == "le_minmax":
                lo, hi = fin & ((mn_t < 0) | (x <= mn)), fin & ((mx_t < 0) | (x >= mx))
            else:
                lo = fin & ((mn_t < 0) | (x < mn) | ((x == mn) & (t < mn_t)))
                hi = fin & ((mx_t < 0) | (x > mx) | ((x == mx) & (t < mx_t)))
            mn, mn_t = np.where(lo, x, mn), np.where(lo, t, mn_t)
            mx, mx_t = np.where(hi, x, mx), np.where(hi, t, mx_t)
            nf_t = np.where(~fin & ((nf_t < 0) | (t < nf_t)), t, nf_t)
            for i, (e, p, above, value) in enumerate(thresholds):
                f = hit(x[:, e, p], above, value)
                best[:, i] = np.where(f & ((best[:, i] < 0) | (t < best[:, i])), t, best[:, i])
            for i, (e, p, above, value) in enumerate(dwells):
                f = hit(x[:, e, p], above, value)
                first[:, i] = np.where(f & (cnt[:, i] == 0), t, first[:, i])
                last[:, i] = np.where(f, t, last[:, i])
                cnt[:, i] += f
        c = cnt > 0
        of, ol = dw[..., 1], dw[..., 2]
        dw[..., 0] += cnt
        dw[..., 1] = np.where(c & ((of < 0) | (first < of)), first, of)
        merged_last = np.where(ol < 0, last, np.minimum(last, ol)) if fault == "last_tick_min" else np.maximum(last, ol)
        dw[..., 2] = np.where(c, merged_last, ol)
    mean = K + S1 / n
    d = S2 - S1 * (S1 / n)
    m2 = np.where(S2 > DBL_MAX, np.inf, d if fault == "no_clamp" else np.where(d < 0.0, 0.0, d))
    none = n == 0.0
    mom = np.stack([n, np.where(none, np.nan, mean), np.where(none, np.nan, m2)], -1)
    return np.stack([mn, mx, mn_t, mx_t, nf_t], -1), best, mom, dw


def canon(a):
    """f64 bits with every NaN the same NaN: R1 does not cover the payload of a NaN the arithmetic makes."""
    a = np.array(a, dtype=np.float64)
    a[np.isnan(a)] = np.nan
    return a.view(np.uint64)


def ref_thresholds(rows, ticks, thresholds):
    """[M, T, 26] from ref_threshold, for conditions on any plane of the row (the record keeps the 25 raw planes)."""
    out = np.empty((rows.shape[1], len(thresholds), 26))
    for i, (e, p, above, value) in enumerate(thresholds):
        tick, planes = ref_threshold(rows[:, :, e, :], ticks, p, above, value)
        out[:, i, 0] = tick
        out[:, i, 1:] = planes[:, :25]
    return out


def ref_dwells(rows, ticks, dwells):
    out = np.empty((rows.shape[1], len(dwells), 3))
    for i, (e, p, above, value) in enumerate(dwells):
        out[:, i] = np.stack(ref_dwell(rows[:, :, e, p], ticks, above, value), -1)
    return out


def r1_failures(got, rows, ticks, thresholds, dwells):
    """The parts of (extrema, threshold ticks, moments, dwells) that differ from the references (R1)."""
    ext, thr, mom, dw = got
    bad = []
    want_ext = ref_tables(rows, ticks, [])[0]
    if not np.array_equal(canon(ext), canon(want_ext)):
        bad.append("extrema")
    if thresholds and not np.array_equal(thr, ref_thresholds(rows, ticks, thresholds)[..., 0]):
        bad.append("thresholds")
    n, mean, m2 = ref_moments(rows)
    if not np.array_equal(canon(mom), canon(np.stack([n, mean, m2], -1))):
        bad.append("moments")
    if dwells and not np.array_equal(dw, ref_dwells(rows, ticks, dwells)):
        bad.append("dwells")
    return bad


def gamma(k):
    return k * U / (1 - k * U)


def exact_moments(seq):
    """The exact rationals of one (world, entity, plane) sequence: (n, mu, m2, sum |y|, sum y^2, S1, s)."""
    fin = [Fraction(float(v)) for v in seq if math.isfinite(v)]
    if not fin:
        return None
    n = len(fin)
    mu = sum(fin) / n
    K = fin[0]
    ys = [v - K for v in fin]
    S1 = sum(ys)
    return n, mu, sum((v - mu) ** 2 for v in fin), sum(abs(y) for y in ys), sum(y * y for y in ys), S1, max(abs(v) for v in fin)


def contract_failures(rows, mom):
    """R2-R4 over every sequence of rows [R, ...] and its table record mom [..., 3]; a list of (index, rule)."""
    bad = []
    flat_rows = rows.reshape(rows.shape[0], -1)
    flat = mom.reshape(-1, 3)
    for j in range(flat.shape[0]):
        ex = exact_moments(flat_rows[:, j])
        if ex is None:
            continue
        n, mu, m2, sy, sy2, S1, s = ex
        _, mean, got_m2 = flat[j]
        if math.isfinite(mean) and abs(Fraction(mean) - mu) > gamma(n + 2) * sy / n + U * abs(mu) + TINY:
            bad.append((j, "R2 mean"))
        if math.isfinite(got_m2) and abs(Fraction(got_m2) - m2) > gamma(2 * n + 8) * (sy2 + S1 * S1 / n) + (n + 2) * TINY:
            bad.append((j, "R2 m2"))
        if not (math.isfinite(mean) and math.isfinite(got_m2)) and not (s > TOP or m2 > TOP):
            bad.append((j, "R3"))
        if s <= EDGE and m2 > Fraction(DBL_MAX) and not (got_m2 == np.inf and math.isfinite(mean)):
            bad.append((j, "R4"))
    return bad


# --------------------------------------------------------------------------- the catalogue

NAN_PAYLOADS = (0x7FF8000000000123, 0xFFF8000000000456, 0x7FF4000000000001, 0x7FFFFFFFFFFFFFFF)
CAT_L, CAT_M, CAT_E = 24, 16, 2


def _payload_nan(rng):
    return np.array([NAN_PAYLOADS[rng.integers(len(NAN_PAYLOADS))]], dtype=np.uint64).view(np.float64)[0]


def catalogue_sequence(kind, rng, L):
    """One row sequence of L values of a catalogue kind."""
    if kind == "zeros_pm":
        return np.array([0.0, -0.0] * (L // 2))
    if kind == "zeros_mp":
        return np.array([-0.0, 0.0] * (L // 2))
    if kind == "ties":
        return rng.choice([1.5, -2.0, 3.0], L)
    if kind == "subnormal":
        return rng.integers(-(1 << 20), 1 << 20, L) * 5e-324
    if kind == "dblmax":
        return rng.choice([DBL_MAX, -DBL_MAX, 1.0, -1.0], L)
    if kind == "nan_payload":
        x = rng.normal(0.0, 4.0, L)
        for r in rng.choice(L, L // 3, replace=False):
            x[r] = _payload_nan(rng)
        return x
    if kind == "inf":
        x = rng.normal(0.0, 4.0, L)
        x[rng.choice(L, L // 3, replace=False)] = rng.choice([INF, -INF], L // 3)
        return x
    if kind == "leading_nonfinite":
        x = rng.normal(10.0, 1.0, L)
        x[:5] = [np.nan, INF, _payload_nan(rng), -INF, np.nan]
        return x
    if kind == "y_overflow":                        # K = -DBL_MAX, then y = DBL_MAX - K overflows
        return np.concatenate([[-DBL_MAX, DBL_MAX], rng.choice([DBL_MAX, -DBL_MAX, 0.0], L - 2)])
    if kind == "s1_nan":                            # S1 overflows to +inf, then y = -DBL_MAX - K is -inf: NaN
        return np.concatenate([[EDGE, DBL_MAX, DBL_MAX, -DBL_MAX], rng.choice([DBL_MAX, -DBL_MAX, 1.0], L - 4)])
    if kind == "clamp":                             # squares underflow to 0, S1 (S1 / n) does not: d < 0
        return np.concatenate([[0.0], np.full(L - 1, 1.5e-162)])
    if kind == "offset":
        return 1e6 + rng.uniform(-1e-3, 1e-3, L)
    if kind == "big_const":                         # m2 = 0, mean * mean overflows in the rms
        return np.full(L, 1e300 * rng.choice([1.0, -1.0]))
    if kind == "edge":                              # R4: the exact m2 is beyond DBL_MAX
        return np.array([EDGE, -EDGE] * (L // 2)) * rng.choice([1.0, 0.75], L)
    return rng.normal(0.0, 1.0, L) * 10.0 ** rng.integers(-5, 6)


KINDS = ("zeros_pm", "zeros_mp", "ties", "subnormal", "dblmax", "nan_payload", "inf", "leading_nonfinite",
         "y_overflow", "s1_nan", "clamp", "offset", "big_const", "edge", "normal")


def catalogue(M=CAT_M, E=CAT_E, L=CAT_L, seed=0):
    """rows [L, M, E, 25] and the kind of each (world, entity, plane): kind (e * 25 + p + w) mod len(KINDS), so a
    condition on one (entity, plane) meets every kind over the worlds."""
    rng = np.random.default_rng(seed)
    x = np.empty((L, M, E, 25))
    kinds = np.empty((M, E, 25), dtype=object)
    for w in range(M):
        for e in range(E):
            for p in range(25):
                k = KINDS[(e * 25 + p + w) % len(KINDS)]
                kinds[w, e, p] = k
                x[:, w, e, p] = catalogue_sequence(k, rng, L)
    return x, kinds


def catalogue_conditions(E=CAT_E):
    """8 conditions, strict at +-0, at a tie value and at +-inf / +-DBL_MAX."""
    last = E - 1
    return [(last, 3, False, 0.0), (last, 3, True, -0.0), (last, 7, True, 1.5), (last, 7, False, 1.5),
            (0, 5, True, -INF), (0, 5, False, INF), (0, 11, True, DBL_MAX), (0, 11, False, -DBL_MAX)]


def catalogue_folds(x):
    """The state route: one fold per row, row r at tick r (tick_step 0)."""
    return [(x[r:r + 1], r, 0) for r in range(len(x))]


def test_catalogue_reaches_every_edge():
    x, kinds = catalogue()
    with np.errstate(over="ignore", invalid="ignore"):
        n, mean, m2 = ref_moments(x)
        K = np.where(np.isfinite(x[0]), x[0], 0.0)
        S1 = np.sum(x - K, 0)
    assert set(kinds.ravel()) == set(KINDS)
    v = x.view(np.uint64)
    assert {int(b) for b in v[np.isnan(x)]} >= set(NAN_PAYLOADS) - {0x7FF8000000000000}
    assert np.any((x == 0) & np.signbit(x)) and np.any((x == 0) & ~np.signbit(x))
    assert np.any((x != 0) & (np.abs(x) < np.finfo(np.float64).tiny))
    assert np.any(x == DBL_MAX) and np.any(x == -DBL_MAX) and np.any(x == INF) and np.any(x == -INF)
    # S1 -> +inf, then NaN; m2 = +inf where S2 overflows; the clamp
    s1 = kinds == "s1_nan"
    assert np.all(np.isnan(mean[s1])) and np.all(m2[s1] == np.inf)
    assert np.any(np.isinf(S1[kinds == "y_overflow"]))
    cl = kinds == "clamp"
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        S1c = np.sum(x[1:] - x[0], 0)
        S2c = np.sum((x[1:] - x[0]) ** 2, 0)
    assert np.all(S2c[cl] == 0.0) and np.all(S1c[cl] * (S1c[cl] / n[cl]) > 0.0) and np.all(m2[cl] == 0.0)
    assert np.all(m2[kinds == "edge"] == np.inf) and np.all(np.isfinite(mean[kinds == "edge"]))
    assert np.all(n[kinds == "leading_nonfinite"] == CAT_L - 5)
    # the clean restatement is the references, and keeps R2-R4
    conds = catalogue_conditions()
    got = fold_model(catalogue_folds(x), conds, conds)
    assert r1_failures(got, x, np.arange(CAT_L), conds, conds) == []
    assert contract_failures(x, got[2]) == []


# --------------------------------------------------------------------------- sensitivity

def synthetic_geometry(case, seed):
    """A sweep case's fold structure over random rows with ties: row 0 from the state at tick pre, then the ring's
    n_rows rows at pre + (k + 1) every in one fold."""
    M, E, n_c, every, pre, n_rows, _ = case
    M = min(M, 5)
    rng = np.random.default_rng(seed)
    rows = rng.integers(-3, 4, (n_rows + 1, M, E, 25)).astype(np.float64)
    folds = [(rows[:1], pre, 0), (rows[1:], pre + every, every)]
    ticks = np.array([pre] + [pre + (k + 1) * every for k in range(n_rows)])
    conds = [(E - 1, 24, True, 0.5), (E - 1, 24, False, -0.5), (0, 6, True, 2.5), (0, 6, False, 0.0)]
    return rows, ticks, folds, conds


@pytest.mark.parametrize("fault", FAULTS)
def test_each_fault_fails_a_case(fault):
    x, kinds = catalogue()
    conds = catalogue_conditions()
    caught = []
    got = fold_model(catalogue_folds(x), conds, conds, fault)
    caught += r1_failures(got, x, np.arange(CAT_L), conds, conds)
    caught += [r for _, r in contract_failures(x, got[2])]
    for k, case in enumerate(SWEEP):
        rows, ticks, folds, gconds = synthetic_geometry(case, k)
        caught += r1_failures(fold_model(folds, gconds, gconds, fault), rows, ticks, gconds, gconds)
    assert caught, f"{fault} passes every case"
    if fault == "k_zero":  # unshifted sums: R2 fails on the offset data itself
        off = kinds == "offset"
        got = fold_model(catalogue_folds(x), [], [], fault)
        assert any(r.startswith("R2") for _, r in contract_failures(x[:, off], got[2][off]))


def test_clean_restatement_passes_the_geometry_cases():
    for k, case in enumerate(SWEEP):
        rows, ticks, folds, conds = synthetic_geometry(case, k)
        assert r1_failures(fold_model(folds, conds, conds), rows, ticks, conds, conds) == [], case_id(case)


# --------------------------------------------------------------------------- GPU helpers


def rows_now(ex, n_c):
    """The state as the fold reads it: [M, E, 25 + n_c]."""
    x = sampled_state(ex)
    return np.concatenate([x, ex.state_channels()], -1) if n_c else x


def ring_rows(ex, n_c):
    x = ex.trajectory()
    if n_c:
        ch = ex.trajectory_channels()
        want, angle = ref_channels(x, CHANNELS[:n_c])
        check_values(ch, want, angle)
        x = np.concatenate([x, ch], -1)
    return x


def launches(ex, call):
    n0 = ex.timings()["kernel_launches"]
    got = call()
    return got, ex.timings()["kernel_launches"] - n0


def tail_bound(x, start):
    """(above, bound) that first fires at a row >= start of world 0's sequence x [R], or None."""
    head, tail = x[:start], x[start:]
    if len(head) and len(tail):
        if np.any(tail > head.max()):
            return True, float(head.max())
        if np.any(tail < head.min()):
            return False, float(head.min())
    return None


def case_conditions(rows, E, p, n_rows):
    """8 conditions on (E - 1, p): one firing in the ring fold's unroll tail where the data allows, one at the median of
    row 0, and bounds at +-0 and +-inf, above and below."""
    x = rows[:, :, E - 1, p]
    tail = tail_bound(x[:, 0], 1 + n_rows // 4 * 4)                   # row 0 is the state's own fold
    med = float(np.median(x[0]))
    conds = [(E - 1, p, True, med), (E - 1, p, False, med), (E - 1, p, False, 0.0), (E - 1, p, True, -0.0),
             (E - 1, p, True, INF), (E - 1, p, False, -INF), (E - 1, p, True, -INF), (E - 1, p, False, INF)]
    if tail is not None:
        conds[0] = (E - 1, p) + tail
    return conds, tail is not None


def check_tables(ex, rows, ticks, spec, R):
    """Every table the spec keeps against the references of rows [S, M, E, R], bit for bit."""
    ext, thr, mom, dw = spec
    if ext:
        want = ref_tables(rows, ticks, [])[0]
        assert ex.extrema().tobytes() == want.tobytes()
    if thr:
        assert np.array_equal(canon(ex.thresholds()), canon(ref_thresholds(rows, ticks, thr)))
        # the copied planes keep their bits, NaN payloads included
        assert ex.thresholds().tobytes() == ref_thresholds(rows, ticks, thr).tobytes()
    if mom:
        n, mean, m2 = ref_moments(rows[..., mom])
        assert np.array_equal(canon(ex.moments()), canon(np.stack([n, mean, m2], -1)))
    if dw:
        assert np.array_equal(ex.dwells(), ref_dwells(rows, ticks, dw))
    if thr and dw and thr == dw:
        assert np.array_equal(ex.dwells()[..., 1], ex.thresholds()[..., 0])


def begin(ex, spec):
    ext, thr, mom, dw = spec
    return launches(ex, lambda: ex.summary_begin(ext, thr, mom, dw))[1]


# --------------------------------------------------------------------------- GPU: the geometry sweep


@pytest.mark.gpu
@pytest.mark.parametrize("case", SWEEP, ids=case_id)
def test_geometry_sweep(case):
    """Ring and state routes at one boundary: the tables of one fold, of single-row folds and of refolds equal the
    numpy fold of the rows the handle recorded, with the launches the restated geometry predicts."""
    need_gpu()
    M, E, n_c, every, pre, n_rows, combo = case
    R = 25 + n_c
    mode = "exact"

    def make(capacity):
        ex, st = handle(ROCKET, M, E, mode, every=every, capacity=capacity, state=state)
        if n_c:
            ex.set_channels(records(CHANNELS[:n_c]))
        ex.step(pre)
        ex.trajectory_reset()
        return ex

    state = None
    probe, state = handle(ROCKET, M, E, mode, every=every, capacity=n_rows)
    with probe:
        if n_c:
            probe.set_channels(records(CHANNELS[:n_c]))
        probe.step(pre)
        probe.trajectory_reset()
        prows = np.concatenate([rows_now(probe, n_c)[None]])
        probe.step(n_rows * every)
        prows = np.concatenate([prows, ring_rows(probe, n_c)])
    p = cond_plane(n_c)
    conds, fires_in_tail = case_conditions(prows, E, p, n_rows)
    spec = combo_spec(combo, R, conds, case_moments(R))
    planes, _ = fold_planes(R, *spec)
    ticks = np.array([pre] + [pre + (k + 1) * every for k in range(n_rows)])

    big, one = make(n_rows), make(1)
    with big, one:
        for ex in (big, one):
            assert begin(ex, spec) == clear_launches(spec[0], len(spec[1]), spec[2], spec[3])
            row0 = rows_now(ex, n_c)
            assert launches(ex, ex.summary_add_state)[1] == fold_launches(1, n_c, planes)
        big.step(n_rows * every)
        ring = ring_rows(big, n_c)
        assert launches(big, big.summary_add_trajectory)[1] == fold_launches(n_rows, n_c, planes)
        rows = np.concatenate([row0[None], ring])
        assert rows.tobytes() == prows.tobytes()                        # the probe's rows: the bounds fit the data
        check_tables(big, rows, ticks, spec, R)
        if fires_in_tail and spec[1]:
            t = big.thresholds()[0, 0, 0]
            assert t >= ticks[1 + n_rows // 4 * 4]                      # fired in the unroll tail of the ring fold
        for k in range(n_rows):                                         # the same rows as single-row folds
            one.trajectory_reset()
            one.step(every)
            assert launches(one, one.summary_add_trajectory)[1] == fold_launches(1, n_c, planes)
        assert one.tick == big.tick
        for name in ("extrema", "thresholds", "moments", "dwells"):
            if spec[("extrema", "thresholds", "moments", "dwells").index(name)]:
                assert getattr(one, name)().tobytes() == getattr(big, name)().tobytes(), name
        # regrouping: the ring once, the ring twice, the ring and then its last row again from the state
        begin(big, spec)
        big.summary_add_trajectory()
        once = {k: getattr(big, k)() for k, on in zip(("extrema", "thresholds", "moments", "dwells"), spec) if on}
        check_tables(big, ring, ticks[1:], spec, R)
        big.summary_add_trajectory()
        for k in ("extrema", "thresholds"):
            if k in once:
                assert getattr(big, k)().tobytes() == once[k].tobytes(), k
        if "moments" in once:
            twice = big.moments()
            assert np.array_equal(twice[..., 0], 2 * once["moments"][..., 0])
            n, mean, m2 = ref_moments(np.concatenate([ring, ring])[..., spec[2]])
            assert np.array_equal(canon(twice), canon(np.stack([n, mean, m2], -1)))
        if "dwells" in once:
            d2 = big.dwells()
            assert np.array_equal(d2[..., 0], 2 * once["dwells"][..., 0])
            assert np.array_equal(d2[..., 1:], once["dwells"][..., 1:])
        begin(big, spec)
        big.summary_add_trajectory()
        big.summary_add_state()                                         # the last row, a second time
        check_tables(big, np.concatenate([ring, ring[-1:]]), np.concatenate([ticks[1:], ticks[-1:]]), spec, R)
        for ex in (big, one):
            assert _lib.lib().b200_sixdof_status(ex._h) == 0


@pytest.mark.gpu
def test_long_fold_loops_the_channel_pass():
    """65,537 rows of one body in one fold: the channel pass runs its in-grid sample loop (bx = 1, by = 65535), the
    fold walks 16,384 unrolled iterations and a one-row tail, and every table equals numpy."""
    need_gpu()
    M, E, n_c, every, _, n_rows, _ = LONG
    R = 25 + n_c
    assert channel_shape(M * E, n_rows)[2] == 2
    ex, _ = handle(ROCKET, M, E, "exact", every=every, capacity=n_rows)
    with ex:
        ex.set_channels(records(CHANNELS[:n_c]))
        ex.step(n_rows)
        ring = ring_rows(ex, n_c)                                       # the channels checked against ref_channels
        assert ring.shape == (n_rows, 1, 1, R)
        conds, tail = case_conditions(np.concatenate([ring[:1], ring]), E, 32, n_rows)
        spec = (True, conds, list(range(R)), conds)
        planes, _ = fold_planes(R, *spec)
        assert fold_grid(M * E, planes) == (1, 33)
        assert begin(ex, spec) == 2
        assert launches(ex, ex.summary_add_trajectory)[1] == 2         # the channel refresh, then the fold
        ticks = np.arange(1, n_rows + 1)
        check_tables(ex, ring, ticks, spec, R)
        if tail:
            assert ex.thresholds()[0, 0, 0] == n_rows                   # the last row: the tail of the unroll
        assert ex.moments()[0, 0, 0, 0] == n_rows
        assert _lib.lib().b200_sixdof_status(ex._h) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("chunked", CHUNKED, ids=lambda c: f"{c[0]}-{c[2]}")
def test_chunked_downloads(chunked):
    """A table whose host download ends in a one-body chunk: the host and device-destination downloads have the same
    bits as numpy, with one launch per chunk."""
    import torch

    need_gpu()
    M, n_c, combo = chunked
    R = 25 + n_c
    ex, _ = handle(ROCKET, M, 1, "exact", capacity=2)
    with ex:
        if n_c:
            ex.set_channels(records(CHANNELS[:n_c]))
        spec = combo_spec(combo, R, [], [])
        ex.summary_begin(*spec)
        row0 = rows_now(ex, n_c)
        ex.summary_add_state()
        ex.step(2)
        rows = np.concatenate([row0[None], ring_rows(ex, n_c)])
        ex.summary_add_trajectory()
        name = "extrema" if combo == "extrema" else "moments"
        per = 5 * R * 8 if combo == "extrema" else 3 * R * 8
        host, n_host = launches(ex, getattr(ex, name))
        assert (n_host, 1) == download_chunks(M, per, False)
        fn = getattr(_lib.lib(), f"b200_sixdof_{name}_download")
        dev = torch.empty(host.shape, dtype=torch.float64, device="cuda")
        _, n_dev = launches(ex, lambda: _lib.check(fn(ex._h, dev.data_ptr(), host.nbytes)))
        assert n_dev == download_chunks(M, per, True)[0] == 1
        assert dev.cpu().numpy().tobytes() == host.tobytes()
        assert _lib.lib().b200_sixdof_status(ex._h) == 0
    ticks = np.array([0, 1, 2])
    if combo == "extrema":
        assert host.tobytes() == ref_tables(rows, ticks, [])[0].tobytes()
    else:
        n, mean, m2 = ref_moments(rows[..., spec[2]])
        assert np.array_equal(bits(host), bits(np.stack([n, mean, m2], -1)))
        assert host[-1, 0, 0, 0] == 3                                   # the last body, alone in its chunk


# --------------------------------------------------------------------------- GPU: the arithmetic catalogue


def catalogue_outcomes(M, E, kinds):
    """25 outcomes of every kind and field, and the restatement of each: f(ext, thr, mom, dw, state, values) -> [M]."""
    def tick(v):
        v = np.array(v, dtype=np.float64)
        v[v == -1.0] = np.nan
        return v

    def moment(f, slot, e):
        def g(ext, thr, mom, dw, st, val):
            n, mean, m2 = mom[:, e, slot, 0], mom[:, e, slot, 1], mom[:, e, slot, 2]
            with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
                return (n, mean, np.sqrt(m2 / n), np.sqrt(mean * mean + m2 / n))[f]
        return g

    last = E - 1
    slot_a, slot_b = 32, 4          # moments on every plane in plane order: slot = plane
    outs, want = [], []
    for f in range(5):              # EXTREMA of channel plane 32
        outs.append((_lib.OUTCOME_EXTREMA, f, 32, last))
        want.append(lambda ext, thr, mom, dw, st, val, f=f: ext[:, last, 32, f] if f < 2 else tick(ext[:, last, 32, f]))
    for f in (0, 1):
        outs.append((_lib.OUTCOME_EXTREMA, f, 24, 0))
        want.append(lambda ext, thr, mom, dw, st, val, f=f: ext[:, 0, 24, f])
    for i, f in ((0, 0), (2, 0), (0, 1 + 3), (5, 1 + 0), (6, 1 + 24)):   # THRESHOLD tick and planes
        outs.append((_lib.OUTCOME_THRESHOLD, f, i))
        want.append(lambda ext, thr, mom, dw, st, val, i=i, f=f: tick(thr[:, i, 0]) if f == 0 else thr[:, i, f])
    for slot, e in ((slot_a, last), (slot_b, 0)):             # MOMENT count, mean, std, rms
        for f in range(4):
            outs.append((_lib.OUTCOME_MOMENT, f, slot, e))
            want.append(moment(f, slot, e))
    for f in range(3):                                         # DWELL fields
        outs.append((_lib.OUTCOME_DWELL, f, 1))
        want.append(lambda ext, thr, mom, dw, st, val, f=f: dw[:, 1, 0] if f == 0 else tick(dw[:, 1, f]))
    outs.append((_lib.OUTCOME_COLUMN, 4, 0, last, "world_pos"))  # COLUMN: the device state now
    want.append(lambda ext, thr, mom, dw, st, val: st[:, last, 4])
    values = np.linspace(-1.0, 1.0, M)
    values[1] = _payload_nan(np.random.default_rng(0))
    outs.append((_lib.OUTCOME_VALUES, 0, 0, 0, 0, values))
    want.append(lambda ext, thr, mom, dw, st, val: val)
    assert len(outs) == _lib.MAX_OUTCOMES
    return outs, want, values


@pytest.mark.gpu
def test_catalogue_keeps_the_contract():
    """R1-R4 over the catalogue on the state route, every channel plane included, then 25 outcomes over its
    summaries against numpy on the downloaded tables."""
    need_gpu()
    x, kinds = catalogue()
    L, M, E, _ = x.shape
    n_c = 8
    R = 25 + n_c
    conds = catalogue_conditions(E)
    spec = (True, conds, list(range(R)), conds)
    planes, _ = fold_planes(R, *spec)
    rows = []
    with state_handle(x[0], "exact") as h:
        h.set_channels(records(CHANNELS))
        assert begin(h, spec) == 2
        for r in range(L):
            h.set_state(x[r, ..., :7], x[r, ..., 7:13], None, accel=x[r, ..., 13:19], force=x[r, ..., 19:25])
            now = rows_now(h, n_c)
            assert now[..., :25].tobytes() == x[r].tobytes()            # the row went up bit for bit
            want, angle = ref_channels(x[r], CHANNELS)
            check_values(now[..., 25:], want, angle)
            rows.append(now)
            assert launches(h, h.summary_add_state)[1] == fold_launches(1, n_c, planes)
            h.step(1)
        rows = np.stack(rows)
        ticks = np.arange(L)
        check_tables(h, rows, ticks, spec, R)
        ext, thr, mom, dw = h.extrema(), h.thresholds(), h.moments(), h.dwells()
        assert np.array_equal(mom[..., 0], np.sum(np.isfinite(rows), 0))
        assert contract_failures(rows, mom) == []
        edge = kinds == "edge"
        assert np.all(mom[..., :25, 2][edge] == np.inf) and np.all(np.isfinite(mom[..., :25, 1][edge]))
        assert np.all(mom[..., :25, 2][kinds == "clamp"] == 0.0)
        # the outcome pass over these summaries
        outs, want, values = catalogue_outcomes(M, E, kinds)
        h.set_outcomes(outs)
        got, n = launches(h, h.outcome_values)
        assert n == 2 and got.shape == (M, len(outs))                   # the outcome pass, then the [M][P] transpose
        st = h.download(WORLD_POS)
        for k, f in enumerate(want):
            assert np.array_equal(canon(got[:, k]), canon(f(ext, thr, mom, dw, st, values))), (k, outs[k][:4])
        assert got[:, -1].tobytes() == values.tobytes()                 # a copied value keeps its payload
        mean, std, rms = got[:, 17], got[:, 18], got[:, 19]            # slot 4 of entity 0: every kind over the worlds
        assert np.any(np.isinf(rms) & np.isfinite(mean) & np.isfinite(std))  # mean * mean past the range
        assert np.any(np.isinf(std) & np.isfinite(mean))                # m2 = +inf
        assert _lib.lib().b200_sixdof_status(h._h) == 0


# --------------------------------------------------------------------------- GPU: an Exec at the maxima

EXEC_CHANNELS = [el.Norm("speed", "world_vel", (3, 4, 5)), el.Norm("range", "world_pos", (4, 5), center=(1.5, -2.0)),
                 el.Norm("alt", "world_pos", (4, 5, 6), minus=0.75), el.Norm("acc", "world_accel", (5, 3, 4)),
                 el.Norm("dz", "world_pos", (6,), center=(-3.0,)), el.AxisAngle("pitch", (-1.0, 0.0, 0.0), (0.0, 0.0, 1.0)),
                 el.AxisAngle("aoa", (0.3, -2.0, 0.5), ("world_vel", (3, 4, 5))),
                 el.AxisAngle("spin", (0.0, 0.0, 2.0), ("world_vel", (0, 1, 2)))]
ENTITIES = ("rocket", "ball")


def _exec_rows(ref, mode):
    """[R, M, 2, 33]: a default-mode run's history, widened by EXEC_CHANNELS computed by the channel pass."""
    from tests.ensemble_util import SAMPLED

    rows = np.stack([np.concatenate([ref.history_worlds(f"{e}.{c}") for c in SAMPLED], -1) for e in ENTITIES], 2)
    with state_handle(rows[0], mode) as h:
        h.set_channels([c._record() for c in EXEC_CHANNELS])
        ch = []
        for x in rows:
            h.set_state(x[..., :7], x[..., 7:13], None, accel=x[..., 13:19], force=x[..., 19:25])
            ch.append(h.state_channels())
    return np.concatenate([rows, np.stack(ch)], -1)


@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", MODES)
def test_exec_at_the_maxima(math_mode):
    """8 channels, 8 thresholds, 8 dwells, moments on every plane of world_vel and every channel and 25 outcomes, on
    the resident and host-callback routes, against the references over a default-mode Exec's rows."""
    need_gpu()
    O = el.Outcome
    M, ticks = 64, 23
    w, sys_, params = rocket_world(M)
    kw = dict(simulation_rate=120.0, telemetry_rate=24.0, math=math_mode, n_worlds=M, world_params=params)
    ref = w.build(sys_, **kw)
    ref.run(ticks)
    rows = _exec_rows(ref, math_mode)                                   # [6, M, 2, 33]
    row_ticks = np.asarray(ref.history("globals.tick")["globals.tick"], dtype=np.int64)
    mid = float(np.median(rows[3, :, 0, 26]))                           # range: world-dependent first ticks
    up = rows[4, 0, 0, 26] > rows[0, 0, 0, 26]
    conds = [el.Threshold("rocket.channels", 1, above=mid) if up else el.Threshold("rocket.channels", 1, below=mid),
             el.Threshold("rocket.channels", 5, below=1.0),
             el.Threshold("rocket.channels", 0, above=5.0), el.Threshold("rocket.world_pos", 6, below=2.0),
             el.Threshold("ball.world_pos", 6, below=0.0), el.Threshold("ball.channels", 4, above=0.0),
             el.Threshold("rocket.world_vel", 5, above=-0.0), el.Threshold("rocket.channels", 2, above=1e9)]
    spec = [(ENTITIES.index(t.pair.split(".")[0]), t.plane, t.above, t.value) for t in conds]
    moments = ["world_vel", "channels"]
    planes = list(range(7, 13)) + list(range(25, 33))
    gain = np.linspace(0.5, 1.5, M)
    outs = ([O(f"x_{f}", "rocket.channels", 7, f) for f in ("min", "max", "min_tick", "max_tick", "first_nonfinite_tick")]
            + [O.threshold(f"t{i}", i, "tick") for i in range(4)]
            + [O.threshold("tp", 0, "world_pos", 4), O.threshold("tf", 3, "force", 5)]
            + [O(f"s_{f}", "rocket.channels", 0, f) for f in ("count", "mean", "std", "rms")]
            + [O(f"v_{f}", "ball.world_vel", 5, f) for f in ("count", "mean", "std", "rms")]
            + [O.dwell(f"d_{f}", 0, f) for f in ("rows", "first_tick", "last_tick")]
            + [O("mass", "rocket.inertia", 6), O("zfin", "rocket.world_pos", 6), O.values("gain", gain)])
    assert len(outs) == _lib.MAX_OUTCOMES

    want_ext = ref_tables(rows, row_ticks, [])[0]
    want_thr = ref_thresholds(rows, row_ticks, spec)
    n, mean, m2 = ref_moments(rows[..., planes])
    want_mom = np.stack([n, mean, m2], -1)
    want_dw = ref_dwells(rows, row_ticks, spec)
    assert len(set(want_thr[:, 0, 0])) >= 2 and np.all(want_thr[:, 7, 0] == -1)

    def tick(v):
        v = np.array(v, dtype=np.float64)
        v[v == -1.0] = np.nan
        return v

    with np.errstate(invalid="ignore", divide="ignore"):
        mo = lambda e, k: (n[:, e, k], mean[:, e, k], np.sqrt(m2[:, e, k] / n[:, e, k]),
                           np.sqrt(mean[:, e, k] ** 2 + m2[:, e, k] / n[:, e, k]))
        expect = ([want_ext[:, 0, 32, f] if f < 2 else tick(want_ext[:, 0, 32, f]) for f in range(5)]
                  + [tick(want_thr[:, i, 0]) for i in range(4)] + [want_thr[:, 0, 1 + 4], want_thr[:, 3, 1 + 24]]
                  + list(mo(0, 6)) + list(mo(1, 5))
                  + [want_dw[:, 0, 0], tick(want_dw[:, 0, 1]), tick(want_dw[:, 0, 2])]
                  + [params["inertia"][:, 0, 6], None, gain])
    for route in ("resident", "host"):
        s = (sys_ | el.host_system(lambda ctx: None)) if route == "host" else sys_
        ex = w.build(s, ensemble=True, channels=EXEC_CHANNELS, extrema=True, thresholds=conds, moments=moments,
                     dwells=conds, outcomes=outs, **kw)
        ex.run(ticks)
        b = ex.backend
        assert b.extrema().tobytes() == want_ext.tobytes(), route
        assert np.array_equal(canon(b.thresholds()), canon(want_thr)), route
        assert np.array_equal(canon(b.moments()), canon(want_mom)), route
        assert np.array_equal(b.dwells(), want_dw), route
        assert np.array_equal(b.dwells()[..., 1], b.thresholds()[..., 0]), route
        v = ex.outcome_values()
        expect[-2] = b.download(WORLD_POS)[:, 0, 6]
        for o, e in zip(outs, expect):
            assert np.array_equal(canon(v[o.name]), canon(e)), f"{route} {o.name}"
        assert ex.tick == ticks
        b.close()
