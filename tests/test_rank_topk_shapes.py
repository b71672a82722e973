"""The rank pass (rank_kernels.cu, behind outcome_[group_]ranks, _rank_correlation and Exec.outcome_sensitivity) and the
worst-worlds select (topk_kernels.cu, behind outcome_[group_]top_worlds) at every level, bucket, range and slice edge of
their plans, against scipy.stats.rankdata and the numpy order of test_outcome_top_worlds.

Restatement.  rank_plan writes the MSD bucket pass out level by level in numpy over one task's keys: the count and plan
0 (shift = 1 + level_shift(kmax - kmin)), then per level kBins = 2^14 equal-width bins per range, each bin resolved as
a tie run (count 1, or one key wide at shift 0), a bucket (at most kCap = 8192 worlds) or a range of the next level, at
most R = max(1, n / 8193) ranges a level (the size of rg0 / rg1).  Its midranks, built from the pieces (a run's
base + (count + 1) / 2, a bucket's base + the in-bucket midrank), must equal scipy, which checks the restatement itself.
topk_plan writes the TState machine out: plan 0 (kk = min(k, n); a task of at most kCap finite worlds is gathered
whole), phase-0 histograms of the value key with shift bit_len(hi - lo) - 14, the move to the bin holding rank kk - 1,
the switch to world indices [0, n - 1] once the range holds one key (phase 1), and the gather; its record must equal
ref_top.  rank_geometry and topk_geometry restate the routes (quantile_order), the slices of the scratch (256 MiB;
sizeof(TRow) = 32 and sizeof(TState) = 80 give 176,240 bytes per top-worlds task and 1523 tasks a slice), the world
chunks (kNumSMs = 132) and the launch counts.  test_constants_match_the_sources_and_the_shared_header reads every
constant and struct the restatement uses from the sources (each kernel file with order_stats.cuh, which holds the route
split and chunk_of), so an edit to a kernel that leaves it behind fails without a GPU.

Catalogue.  The planes are built from keys (key_value, the inverse of order_key), so that a case sits on the bin edge
it names rather than hoping random data finds it: a bin of kCap and of kCap + 1 worlds at levels 1, 2 and 4, R ranges
at one level, buckets of 2 .. 8192 worlds at each power-of-two edge of the finish sort, a run of kCap + 1 zeros reached
at shift 0 over the 64-bit key span of +-DBL_MAX, every read count of the rank pass (1 .. 7) and of the select (1 .. 8),
the phase-1 switch after 0 .. 5 phase-0 levels, rank kk - 1 at either end of its bin, a below area of 1023, a gathered
range of kCap, -0 and +0 split by a bin edge, and the geometry edges (route order, chunk multiples and their
neighbours, a rank slice filled to within 8 bytes of the cap and the same plus one world, a boundary between one
group's planes, a rank task that needs more than the cap alone, 1522 top-worlds tasks in one slice and 1524 in a full
slice and one more, and a correlation call whose rank scratch sits behind a 1.3 MB covariance table).  A call has at
most 1024 groups and 25 planes and 1523 is prime, so no call has exactly 1523 tasks.
test_sweep_reaches_every_boundary asserts each edge is reached.
Nine reads of the select need two index levels, so a group of more than 2^27 worlds (a 1 GiB plane, tens of GB of
handle state), and ten need three (more than 2^28): the catalogue stops at eight.

Contract, for every GPU case.  R1: the ranks equal ref_ranks bit for bit, the records ref_top bit for bit and world
for world, and a correlation keeps _check_rho.  R2: rank_reads() and top_worlds_reads() times the tasks equal the
restated sums exactly.  R3: the kernel_launches delta equals the restated count.  R4: the outcome planes keep their
bits.  The kernels take no math mode: the sweep runs in exact, one case of each in fast.

Sensitivity.  Each of FAULTS, injected into the restatements one at a time, must fail a catalogue case or miss an
edge, so the catalogue tells each of them apart from the kernels' plan."""

import os
import re

import numpy as np
import pytest
import scipy.stats

from tests.ensemble_util import need_gpu
from tests.test_outcome_rank_correlation import _check_rho, _only_values, ref_ranks, same
from tests.test_outcome_top_worlds import ref_top

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "elodin_b200", "csrc")

# --------------------------------------------------------------------------- the constants, restated

KCAP = 8192
KBINS = 1 << 14
KBINBITS = 14
RANK_LEVELS = 5
TOPK_LEVELS = 8
SMALL_MAX = 8192
WARP_MAX = 256
PASS_THREADS = 256
SCRATCH_CAP = 256 << 20
HEADER = 256
NUM_SMS = 132
KBELOW = 1024
RANK_TROW, RANK_TSTATE, RANK_RANGE = 40, 56, 16
TOPK_TROW, TOPK_TSTATE = 32, 80
TOPK_TASK_BYTES = TOPK_TROW + TOPK_TSTATE + KBINS * 4 + (KBELOW + KCAP) * 12
SLICE_TASKS = (SCRATCH_CAP - 256) // TOPK_TASK_BYTES
RANK_SEQUENCE = 5 + 2 * RANK_LEVELS  # init, count, plan 0, 5 x (pass, plan), scatter, finish
TOPK_SEQUENCE = 5 + 2 * TOPK_LEVELS  # init, count, plan 0, 8 x (pass, plan), gather, finish
MASK64 = (1 << 64) - 1
U64 = np.uint64

FAULTS = ("bucket_below_cap", "no_run_at_shift0", "midrank_half", "ranges_one_fewer", "no_phase1", "no_hi_clamp",
          "late_bin", "empty_slice", "unrounded_chunk")


def cdiv(a, b):
    return -(-a // b)


def align8(x):
    return cdiv(x, 8) * 8


def order_key(x):
    """The IEEE totalOrder key of every value (as the kernels' order_key)."""
    u = np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)
    return np.where(u >> U64(63), ~u, u | U64(1 << 63))


def key_value(k):
    """The value of every key: the inverse of order_key."""
    k = np.asarray(k, dtype=np.uint64)
    return np.ascontiguousarray(np.where(k >> U64(63), k & U64((1 << 63) - 1), ~k)).view(np.float64)


def rank_key(x):
    """rank_kernels.cu rank_key: -0 is +0."""
    x = np.asarray(x, dtype=np.float64)
    return order_key(np.where(x == 0.0, 0.0, x))


def level_shift(span):
    return max(int(span).bit_length() - KBINBITS, 0)


def ranges_of(n, fault=None):
    R = max(1, n // (KCAP + 1))
    return R - 1 if fault == "ranges_one_fewer" and R > 1 else R


def rank_task_bytes(n):
    R = ranges_of(n)
    return (align8(RANK_TSTATE) + 2 * R * RANK_RANGE + 2 * R * KBINS * 4 + n * 16 + align8(n * 4)
            + align8((n // 2 + 1) * 4) + align8(n * 4))


def chunk_of(n, T, fault=None):
    want = max(1, 8 * NUM_SMS // max(1, T))
    per = max(cdiv(n, want), 16 * PASS_THREADS)
    return per if fault == "unrounded_chunk" else cdiv(per, PASS_THREADS) * PASS_THREADS


def quantile_order(sizes):
    route = [0 if n <= WARP_MAX else 1 if n <= SMALL_MAX else 2 for n in sizes]
    return [g for r in range(3) for g in range(len(sizes)) if route[g] == r]


# --------------------------------------------------------------------------- the rank pass, restated


def _bucket_midranks(keys, base):
    """base + the midrank within its bucket of every world (the finish kernel's bitonic sort and midrank_at)."""
    o = np.lexsort((keys, base))
    sb, sk = base[o], keys[o]
    m = sk.size
    new = np.ones(m, bool)
    new[1:] = (sk[1:] != sk[:-1]) | (sb[1:] != sb[:-1])
    starts = np.flatnonzero(new)
    run = np.cumsum(new) - 1
    s, e = starts[run], np.append(starts[1:], m)[run]
    bnew = np.ones(m, bool)
    bnew[1:] = sb[1:] != sb[:-1]
    bs = np.flatnonzero(bnew)[np.cumsum(bnew) - 1]
    out = np.empty(m)
    out[o] = sb + ((s - bs) + (e - bs) + 1) * 0.5
    return out


def rank_plan(keys, n_group, fault=None):
    """rank_kernels.cu on the rank keys of one task's complete worlds (n_group worlds in its group) -> (plan, midranks).
    plan: reads, ranges per level, R, and per resolved bin (level, count, kind 0 run / 1 bucket / 2 range, shift); per
    world the base of its piece and whether that piece is a run; errors (what the kernel would do out of bounds)."""
    keys = np.asarray(keys, dtype=np.uint64)
    n = keys.size
    P = dict(reads=1, ranges=[0] * (RANK_LEVELS + 2), R=ranges_of(n_group, fault), bins=[], errors=[],
             span=0, piece=np.zeros(n, np.int64), is_run=np.zeros(n, bool))
    ranks = np.full(n, np.nan)
    if n == 0:
        return P, ranks
    P["reads"] += 1  # the scatter
    kmin, kmax = int(keys.min()), int(keys.max())
    P["span"] = kmax - kmin
    shift0 = 0 if kmin == kmax else 1 + level_shift(kmax - kmin)
    # the bins of the level being resolved, and each live world's bin
    w = np.arange(n)
    wbin = np.zeros(n, np.int64)
    count = np.array([n], np.int64)
    base = np.array([0], np.int64)
    lo = np.array([kmin], np.uint64)
    shift = np.array([shift0], np.int64)
    nxt = np.array([shift0 - 1 if shift0 else 0], np.int64)
    level = 0
    while True:
        run = (count == 1) | ((shift == 0) & (fault != "no_run_at_shift0"))
        bucket = ~run & ((count < KCAP) if fault == "bucket_below_cap" else (count <= KCAP))
        rng = ~run & ~bucket
        kind = np.where(run, 0, np.where(bucket, 1, 2))
        P["bins"].append((level, count, kind, shift))
        wr, wb = run[wbin], bucket[wbin]
        c = count[wbin[wr]]
        ranks[w[wr]] = base[wbin[wr]] + (c / 2.0 if fault == "midrank_half" else (c + 1) / 2.0)
        P["piece"][w[wr | wb]] = base[wbin[wr | wb]]
        P["is_run"][w[wr]] = True
        if wb.any():
            ranks[w[wb]] = _bucket_midranks(keys[w[wb]], base[wbin[wb]])
        nr = int(rng.sum())
        if nr == 0:
            break
        level += 1
        if level > RANK_LEVELS:
            P["errors"].append(f"ranges at level {level}, past the {RANK_LEVELS} passes")
            break
        P["ranges"][level] = nr
        if nr > P["R"]:
            P["errors"].append(f"{nr} ranges at level {level}: rg and hist hold {P['R']}")
        P["reads"] += 1
        rid_of = np.full(count.size, -1)
        rid_of[rng] = np.arange(nr)
        live = rid_of[wbin] >= 0
        w, rid = w[live], rid_of[wbin[live]]
        rlo, rsh, rbase = lo[rng], nxt[rng], base[rng]
        b = ((keys[w] - rlo[rid]) >> rsh[rid].astype(np.uint64)).astype(np.int64)
        if b.size and b.max() >= KBINS:
            P["errors"].append(f"bin {b.max()} at level {level}")
            b = np.minimum(b, KBINS - 1)
        uniq, wbin, count = np.unique(rid * KBINS + b, return_inverse=True, return_counts=True)
        ur, ub = uniq // KBINS, uniq % KBINS
        cum = np.cumsum(count) - count
        base = rbase[ur] + cum - cum[np.searchsorted(ur, ur)]
        lo = rlo[ur] + (ub.astype(np.uint64) << rsh[ur].astype(np.uint64))
        shift = rsh[ur]
        nxt = np.maximum(shift - KBINBITS, 0)
    return P, ranks


# --------------------------------------------------------------------------- the worst-worlds select, restated

DONE, REFINE, GATHER = 0, 1, 2


def topk_plan(values, k, largest, fault=None, offset=0):
    """topk_kernels.cu on one task's plane `values` [n] (worlds offset + i) -> plan: reads, the final (state, phase,
    levels, below, count, ilo, ihi), the hits (level, phase, rank within the hit bin, its count), the phase-0 levels
    before the phase-1 switch, whether -0 and +0 fell in different bins of one histogram, the record and errors."""
    x = np.ascontiguousarray(values, dtype=np.float64)
    n = x.size
    fin = np.isfinite(x)
    w = np.flatnonzero(fin).astype(np.int64)
    s = order_key(x[fin])
    if largest:
        s = ~s
    nf = w.size
    kk = min(k, nf)
    zk = order_key(np.array([-0.0, 0.0]))
    if largest:
        zk = ~zk
    zk = [int(z) for z in zk]
    P = dict(reads=1, errors=[], hits=[], phase1_after=None, zero_split=False, n=n, nf=nf, kk=kk, k=k)
    rec = np.full(1 + 2 * k, np.nan)
    rec[0] = nf
    rec[1 + k:] = -1.0
    P["record"] = rec
    st = dict(state=DONE, phase=0, levels=0, below=0, count=nf, ilo=0, ihi=0xFFFFFFFF, lo=0, hi=MASK64, shift=0)
    P["final"] = st
    if nf == 0:
        return P
    r = kk - 1
    if nf > KCAP:
        st["lo"], st["hi"] = int(s.min()), int(s.max())

    def next_pass():
        if st["count"] <= KCAP:
            st["state"] = GATHER
            return
        st["state"] = REFINE
        if not st["phase"] and st["lo"] == st["hi"] and fault != "no_phase1":
            st["phase"], st["ilo"], st["ihi"] = 1, 0, n - 1
            P["phase1_after"] = st["levels"]
        span = st["ihi"] - st["ilo"] if st["phase"] else st["hi"] - st["lo"]
        st["shift"] = max(int(span).bit_length() - KBINBITS, 0)

    next_pass()
    P["reads"] += 1
    for level in range(1, TOPK_LEVELS + 1):
        if st["state"] != REFINE:
            break
        sh, lo, hi = st["shift"], st["lo"], st["hi"]
        if not st["phase"]:
            inr = (s >= U64(lo)) & (s <= U64(hi))
            bins = ((s[inr] - U64(lo)) >> U64(sh)).astype(np.int64)
            z = [((zv - lo) >> sh) for zv in zk if lo <= zv <= hi and np.any(s[inr] == U64(zv))]
            if len(z) == 2 and z[0] != z[1]:
                P["zero_split"] = True
        else:
            inr = (s == U64(lo)) & (w >= st["ilo"]) & (w <= st["ihi"])
            bins = (w[inr] - st["ilo"]) >> sh
        if bins.size and bins.max() >= KBINS:
            P["errors"].append(f"bin {bins.max()} at level {level}")
            bins = np.minimum(bins, KBINS - 1)
        hist = np.bincount(bins, minlength=KBINS)
        cum = np.cumsum(hist)
        b = int(np.searchsorted(cum, r, side="right"))
        if fault == "late_bin":
            b = min(b + 1, KBINS - 1)
        hb, hc = int(cum[b] - hist[b]), int(hist[b])
        P["hits"].append((level, st["phase"], r - hb, hc))
        span = (1 << sh) - 1 if sh else 0
        if not st["phase"]:
            st["lo"] = (lo + (b << sh)) & MASK64
            if fault != "no_hi_clamp":
                st["hi"] = min(hi, (st["lo"] + span) & MASK64)
        else:
            ilo = st["ilo"] + (b << sh)
            st["ihi"] = min(st["ihi"], ilo + span)
            st["ilo"] = ilo
        r -= hb
        st["below"] += hb
        st["count"] = hc
        st["levels"] = level
        next_pass()
        P["reads"] += 1
    if st["state"] == REFINE:
        P["errors"].append(f"still refining after {TOPK_LEVELS} passes")
        return P
    lo, hi, ilo, ihi = U64(st["lo"]), U64(st["hi"]), st["ilo"], st["ihi"]
    before = (s < lo) | ((s == lo) & (w < ilo))
    inside = ~before & ((s < hi) | ((s == hi) & (w <= ihi)))
    if before.sum() != st["below"] or st["below"] > KBELOW:
        P["errors"].append(f"below area of {before.sum()} worlds, plan {st['below']}")
    if inside.sum() != st["count"] or st["count"] > KCAP:
        P["errors"].append(f"range area of {inside.sum()} worlds, plan {st['count']}")
    take = kk - st["below"]
    if take < 0 or take > inside.sum():
        P["errors"].append(f"{take} worlds taken from a range of {inside.sum()}")
        return P
    ob = np.lexsort((w[before], s[before]))
    oi = np.lexsort((w[inside], s[inside]))[:take]
    sk = np.concatenate([s[before][ob], s[inside][oi]])
    sw = np.concatenate([w[before][ob], w[inside][oi]])
    rec[1:1 + kk] = key_value(~sk if largest else sk)
    rec[1 + k:1 + k + kk] = sw + offset
    return P


# --------------------------------------------------------------------------- the geometry, restated


def rank_slices(task_n, fault=None):
    """slices_of over the large tasks' group sizes -> [(t0, T, bytes)]; a slice of no task (what the host loop would
    repeat forever without its at-least-one rule) ends the list."""
    out, t = [], 0
    while t < len(task_n):
        t0, T, b = t, 0, HEADER
        while t < len(task_n):
            add = RANK_TROW + rank_task_bytes(task_n[t])
            if (T > 0 or fault == "empty_slice") and b + add > SCRATCH_CAP:
                break
            b, T, t = b + add, T + 1, t + 1
        out.append((t0, T, b))
        if T == 0:
            break
    return out


def rank_geometry(sizes, n_p, corr=False, fault=None):
    """The routes, slices, chunks and launches of one rank call over groups `sizes` and n_p planes."""
    order = quantile_order(sizes)
    warp = sum(n <= WARP_MAX for n in sizes)
    block = sum(n <= SMALL_MAX for n in sizes)
    task_n = [sizes[order[block + t // n_p]] for t in range((len(sizes) - block) * n_p)]
    slices = rank_slices(task_n, fault) if task_n else []
    chunks = [[(task_n[t0 + i], chunk_of(task_n[t0 + i], T, fault)) for i in range(T)] for t0, T, _ in slices]
    launches = 0
    if sum(sizes):
        launches = 1 + (warp > 0) + (block > warp) + RANK_SEQUENCE * len(slices) + (0 if corr else 1)
    return dict(order=order, warp=warp, block=block, task_n=task_n, slices=slices,
                chunks=[[(n, wc, cdiv(n, wc)) for n, wc in c] for c in chunks], launches=launches,
                scratch=max([b for _, _, b in slices], default=0))


def topk_geometry(sizes, n_p, fault=None):
    order = quantile_order(sizes)
    warp = sum(n <= WARP_MAX for n in sizes)
    block = sum(n <= SMALL_MAX for n in sizes)
    n_tasks = (len(sizes) - block) * n_p
    slices = [(t0, min(SLICE_TASKS, n_tasks - t0)) for t0 in range(0, n_tasks, SLICE_TASKS)]
    task_n = [sizes[order[block + t // n_p]] for t in range(n_tasks)]
    chunks = [[(task_n[t0 + i], chunk_of(task_n[t0 + i], T, fault)) for i in range(T)] for t0, T in slices]
    return dict(order=order, warp=warp, block=block, slices=slices,
                chunks=[[(n, wc, cdiv(n, wc)) for n, wc in c] for c in chunks],
                launches=(warp > 0) + (block > warp) + TOPK_SEQUENCE * len(slices),
                scratch=256 + min(SLICE_TASKS, n_tasks) * TOPK_TASK_BYTES if n_tasks else 0)


# --------------------------------------------------------------------------- the catalogue

KEY_ONE = int(order_key(np.array([1.0]))[0])
KEY_LOW = int(order_key(np.array([-np.finfo(np.float64).max]))[0])   # -DBL_MAX
KEY_HIGH = int(order_key(np.array([np.finfo(np.float64).max]))[0])   # +DBL_MAX


def u64(*parts):
    return np.concatenate([np.asarray(p, dtype=np.uint64).ravel() for p in parts])


def from_keys(offsets, base=0):
    """The values whose keys are base + offsets (all finite)."""
    v = key_value(U64(base) + u64(offsets))
    assert np.all(np.isfinite(v))
    return v


def _fill(rng, n, lo, hi, avoid=()):
    """n offsets uniform in [lo, hi] outside the half-open offset intervals `avoid`."""
    out = np.empty(0, np.uint64)
    while out.size < n:
        c = rng.integers(lo, hi, 2 * n, endpoint=True, dtype=np.uint64)
        for a, b in avoid:
            c = c[(c < a) | (c >= b)]
        out = np.concatenate([out, c])
    return out[:n]


def _shuffled(rng, offsets):
    o = np.asarray(offsets)
    return o[rng.permutation(o.size)]


def _level_cap_plane(rng, a, l1_shift, layout):
    """Offsets of a task whose bin at one level holds `a` worlds; layout (level-1 bin, cluster offset in it, partner
    offsets in it) with 2000 fillers in other level-1 bins and the span's two ends."""
    D = (1 << (l1_shift + KBINBITS)) - 1
    b1, at, partners = layout
    start = b1 << l1_shift
    cluster = start + at + np.arange(a)
    fill = _fill(rng, 2000, 1, D - 1, [(start, start + (1 << l1_shift))])
    return _shuffled(rng, u64([0, D], cluster, start + np.asarray(partners, np.int64), fill))


def rank_catalogue():
    """[(name, values [M, p], sizes or None, planes, reads per task in task order or None)]."""
    rng = np.random.default_rng(20)
    nan, inf = np.nan, np.inf
    cases = []
    # complete counts in groups of 9000: 0 (the count alone), 1 (a run of one), kCap (a bucket at plan 0), kCap + 1
    v = rng.normal(0, 1, (9000, 4))
    for g, c in enumerate((0, 1, KCAP, KCAP + 1)):
        v[c:, g] = [nan, inf, -inf][g % 3] if c < 9000 else 0
    cases.append(("complete_counts", v.T.reshape(-1, 1).copy(), [9000] * 4, [0], [1, 2, 2, 3]))
    # one value: a run of 20000 at plan 0
    cases.append(("constant", np.full((20000, 1), 3.25), None, [0], [2]))
    # a level-1 bin of kCap (a bucket) and of kCap + 1 (level-2 ranges of 64 keys): shift 20
    planes = [_level_cap_plane(rng, a, 20, (5, 0, [])) for a in (KCAP, KCAP + 1)]
    planes[0] = u64(planes[0], [3 << 20])  # one more filler, in another bin: both planes of one size
    cases.append(("level1_cap", np.stack([from_keys(p, KEY_ONE) for p in planes], 1), None, [0, 1], [3, 4]))
    # a level-2 bin of kCap and of kCap + 1 beside 100 worlds of another level-2 bin: shifts 30, 16, 2
    planes = [_level_cap_plane(rng, a, 30, (7, 3 << 16, (9 << 16) + np.arange(100 + KCAP + 1 - a))) for a in
              (KCAP, KCAP + 1)]
    cases.append(("level2_cap", np.stack([from_keys(p, KEY_ONE) for p in planes], 1), None, [0, 1], [4, 5]))
    # a level-4 bin of kCap and of kCap + 1 (256 keys, ties) over the 64-bit span of +-DBL_MAX: shifts 50 .. 0
    D = KEY_HIGH - KEY_LOW
    c0 = (KEY_ONE - KEY_LOW) >> 22 << 22
    planes = []
    for a in (KCAP, KCAP + 1):
        cl = U64(c0 + 5 * 256) + (np.arange(a) % 256).astype(U64)
        fill = _fill(rng, 2000 + KCAP + 1 - a, 1, D - 1, [(c0 >> 50 << 50, (c0 >> 50) + 1 << 50)])
        planes.append(_shuffled(rng, u64([0, D, c0 + 9 * 256], cl, fill)))
    cases.append(("level4_cap", np.stack([from_keys(p, KEY_LOW) for p in planes], 1), None, [0, 1], [6, 7]))
    # R = 8 ranges at level 2: n = 8 (kCap + 1) worlds in 8 clusters of kCap + 1 keys, one per level-1 bin (shift 20)
    R = 8
    cl = np.concatenate([(2000 * c << 20) + np.arange(KCAP + 1) for c in range(R)])
    cases.append(("r_ranges", from_keys(_shuffled(rng, cl), KEY_ONE)[:, None], None, [0], [4]))
    # buckets at the power-of-two edges of the finish sort, each in its own level-1 bin (shift 20), ties in half
    parts = [[0, (1 << 34) - 1]]
    for i, a in enumerate((2, 3, 256, 257, 4096, 4097, 8191, 8192)):
        parts.append((1000 * (i + 1) << 20) + (np.arange(a) // 2 if i % 2 else np.arange(a)))
    parts.append(_fill(rng, 500, 1, (1 << 34) - 2, [(1000 << 20, 9000 << 20)]))
    cases.append(("bucket_sizes", from_keys(_shuffled(rng, u64(*parts)), KEY_ONE)[:, None], None, [0], [3]))
    # zeros: plane 0 a run of kCap + 1 signed zeros reached at shift 0 beside subnormals over +-DBL_MAX; plane 1 signed
    # zeros and subnormals in one bucket; plane 2 NaN and +-inf, which drop their worlds from every plane
    M = 12000
    z = np.empty((M, 3))
    sub = np.array([5e-324, -5e-324, 1e-310, -1e-310, 2.5e-320, -7e-315])
    z[:, 0] = rng.normal(0, 1, M)
    z[:KCAP + 1, 0] = np.where(np.arange(KCAP + 1) % 2, 0.0, -0.0)
    z[KCAP + 1:KCAP + 61, 0] = np.resize(sub, 60)
    z[KCAP + 61:KCAP + 63, 0] = [-np.finfo(np.float64).max, np.finfo(np.float64).max]
    z[:, 1] = rng.normal(0, 1, M)
    z[:, 1][rng.permutation(M)[:400]] = np.resize(np.concatenate([[0.0, -0.0], sub]), 400)
    z[:, 2] = rng.uniform(-1, 1, M)
    bad = KCAP + 63 + rng.permutation(M - KCAP - 63)[:300]
    z[bad[:100], 2], z[bad[100:200], 2], z[bad[200:], 2] = nan, inf, -inf
    perm = rng.permutation(M)
    cases.append(("zeros", z[perm], None, [0, 1, 2], [7, 3, 3]))
    return cases


def _tk_block_plane(rng, n, L, where):
    """One plane of n worlds: a block of kCap + 1 worlds at 1.0, one world above and one below it with a key span of
    b bits (L phase-0 levels to one key), the rest NaN; the block at the start, the end or spread."""
    b = {1: 14, 2: 28, 3: 42, 4: 56, 5: 64}[L]
    if L == 5:
        lo, hi = KEY_LOW, KEY_HIGH
    else:
        lo, hi = KEY_ONE - (1 << (b - 2)), KEY_ONE + (1 << (b - 2))
    assert (hi - lo).bit_length() == b
    x = np.full(n, np.nan)
    if where == "start":
        x[:KCAP + 1], x[KCAP + 1:KCAP + 3] = 1.0, from_keys([lo, hi])
    elif where == "end":
        x[n - KCAP - 1:], x[:2] = 1.0, from_keys([lo, hi])
    else:
        idx = rng.permutation(n)[:KCAP + 3]
        x[idx[2:]], x[idx[:2]] = 1.0, from_keys([lo, hi])
    return x


def topk_catalogue():
    """[(name, values [M, p], sizes or None, planes)]."""
    rng = np.random.default_rng(21)
    nan, inf = np.nan, np.inf
    cases = []
    # finite counts of large groups: none (1 read), kCap and 1000 and 1024 (gathered whole), kCap + 1
    v = rng.normal(0, 1, (9000, 5))
    for g, c in enumerate((0, KCAP, KCAP + 1, 1000, 1024)):
        v[rng.permutation(9000)[:9000 - c], g] = np.resize([nan, inf, -inf], 9000 - c)
    cases.append(("finite_counts", v.T.reshape(-1, 1).copy(), [9000] * 5, [0]))
    # the phase-1 switch after 1 .. 5 phase-0 levels; the block from world 0 (plane 0) and to world n - 1 (plane 1)
    n = 9000
    planes = [_tk_block_plane(rng, n, L, w) for L, w in ((1, "start"), (2, "end"), (3, None), (4, None), (5, None))]
    cases.append(("phase1_levels", np.stack(planes, 1), None, [0, 1, 2, 3, 4]))
    # phase 1 over 2^18 worlds (bins of 16 indices): the block on the even worlds, NaN between them, 1023 worlds above
    # and 1023 below it
    n = 1 << 18
    x = np.full(n, np.nan)
    x[0::2] = 2.5
    odd = n // 2 + 1 + 2 * rng.permutation(n // 4 - 1)[:2046]  # odd worlds of the second half
    x[odd[:1023]] = rng.uniform(3.0, 1e6, 1023)
    x[odd[1023:]] = rng.uniform(-1e6, 2.0, 1023)
    cases.append(("phase1_wide", x[:, None], None, [0]))
    # one value over 40000 worlds: phase 1 from plan 0
    cases.append(("phase1_at_plan0", np.full((40000, 1), -2.0), None, [0]))
    # plane 0: 1024 worlds at the top of one bin (rank 1023 its last); plane 1: a top bin of exactly kCap worlds;
    # plane 2: -0 and +0 split by the bin edge at 2^62 over the span +-nextafter(2, 0)
    M = 10024
    p0 = np.concatenate([from_keys(np.arange(1024), KEY_ONE + (2000 << 30)), rng.uniform(-1.0, 1.0, M - 1024)])
    p1 = np.concatenate([from_keys(np.arange(KCAP), KEY_ONE + (3000 << 30)), rng.uniform(-1.0, 1.0, M - KCAP)])
    x2 = np.nextafter(2.0, 0.0)
    p2 = np.concatenate([[-x2, x2], rng.uniform(-2.0, -0.5, 500), np.resize([-0.0, 0.0], 60),
                         rng.uniform(0.5, 2.0, M - 562)])
    cases.append(("bin_edges", np.stack([rng.permutation(p) for p in (p0, p1, p2)], 1), None, [0, 1, 2]))
    return cases


def top_ks(values, sizes, planes):
    """k in {1, 2, 1023, 1024} and every task's finite count +-1 within [1, 1024]."""
    ks = {1, 2, 1023, 1024}
    o = 0
    for n in sizes or [values.shape[0]]:
        for j in planes:
            c = int(np.isfinite(values[o:o + n, j]).sum())
            ks |= {c + d for d in (-1, 0, 1) if 1 <= c + d <= 1024}
        o += n
    return sorted(ks)


# --------------------------------------------------------------------------- the geometry catalogue


def _slice_at_cap():
    """(nA, nB): two groups of two planes whose first three tasks fill a slice to within 8 bytes of the cap."""
    add = lambda n: RANK_TROW + rank_task_bytes(n)  # noqa: E731
    for nA in range(2_200_000, 2_200_100):
        room = SCRATCH_CAP - HEADER - 2 * add(nA)
        lo, hi = 0, room // 16  # the most worlds whose task fits in `room` (add grows with n)
        while lo < hi:
            mid = (lo + hi + 1) // 2
            lo, hi = (mid, hi) if add(mid) <= room else (lo, mid - 1)
        if room - add(lo) < 8:
            break
    return nA, lo, room - add(lo)


NA, NB, CAP_GAP = _slice_at_cap()
MIXED = [9000, 3, 8192, 300, 8193, 0, (1 << 20) + 7]
ALONE = 6_720_000  # 1050 chunks of 6400 worlds: ceil(n / 1056) = 6364, rounded up to 6400
# (name, sizes, n_p, kind, expected: launches, slice task counts, (n, Wc, C) of named tasks)
GEOMETRY = [
    ("rank_mixed", MIXED, 2, "rank", dict(launches=1 + 1 + 1 + 15 + 1, slices=[6],
                                          chunks={(1 << 20) + 7: (6144, 171)})),
    ("rank_chunk_edges", [12287, 12288, 12289], 1, "rank", dict(launches=1 + 15 + 1, slices=[3],
                                                                 chunks={12287: (4096, 3), 12289: (4096, 4)})),
    ("rank_alone", [ALONE], 1, "rank", dict(launches=1 + 15 + 1, slices=[1], chunks={ALONE: (6400, 1050)})),
    ("rank_slice_at_cap", [NA, NB, 1], 2, "rank", dict(launches=1 + 1 + 2 * 15 + 1, slices=[3, 1])),
    ("rank_slice_past_cap", [NA, NB + 1, 0], 2, "rank", dict(launches=1 + 1 + 2 * 15 + 1, slices=[2, 2])),
    ("rank_corr_table", [3] * 1000 + [20000], 12, "corr", dict(launches=1 + 1 + 15, slices=[12])),
    ("topk_mixed", MIXED, 2, "topk", dict(launches=1 + 1 + 21, slices=[6])),
    ("topk_1522", [KCAP + 1] * 761, 2, "topk", dict(launches=21, slices=[1522])),
    ("topk_1524", [KCAP + 1] * 127, 12, "topk", dict(launches=2 * 21, slices=[1523, 1])),
]


def geometry_of(case, fault=None):
    name, sizes, n_p, kind, _ = case
    if kind == "topk":
        return topk_geometry(sizes, n_p, fault)
    return rank_geometry(sizes, n_p, corr=kind == "corr", fault=fault)


def geometry_values(case, seed):
    """Continuous planes with ties and a few non-finite values for a geometry case: [M, n_p]."""
    _, sizes, n_p, kind, _ = case
    rng = np.random.default_rng(seed)
    M = sum(sizes)
    v = rng.normal(0, 1, (M, n_p))
    v[:, -1] = np.round(v[:, -1] * 8)
    v[rng.random((M, n_p)) < 1e-4] = np.nan
    return v


# --------------------------------------------------------------------------- edges and failures


def _group_tasks(values, sizes, planes):
    """(group offset, n, selected values [n, p]) of every group."""
    o = 0
    for n in sizes or [values.shape[0]]:
        yield o, n, values[o:o + n][:, planes]
        o += n


def rank_report(case, fault=None):
    """(edges, failures, reads per task) of a rank catalogue case through the restatement."""
    name, values, sizes, planes, want_reads = case
    edges, fails, reads = set(), [], []
    for o, n, sel in _group_tasks(values, sizes, planes):
        ok = np.all(np.isfinite(sel), axis=1)
        if (~ok).any() and np.any(np.isfinite(sel[~ok]).sum(1) == len(planes) - 1):
            edges.add("incomplete in one plane")
        for j in range(len(planes)):
            if n <= SMALL_MAX:
                reads.append(1)
                continue
            edges.add(f"complete {ok.sum()}")
            keys = rank_key(sel[ok, j])
            P, r = rank_plan(keys, n, fault)
            reads.append(P["reads"])
            fails += [f"{name} plane {j}: {e}" for e in P["errors"]]
            if ok.any() and not same(r, scipy.stats.rankdata(sel[ok, j], method="average")):
                fails.append(f"{name} plane {j}: midranks differ from scipy")
            edges.add(f"reads {P['reads']}")
            edges |= {f"ranges at level {l}" for l, nr in enumerate(P["ranges"]) if nr}
            if P["R"] > 1 and max(P["ranges"]) == P["R"]:
                edges.add("R ranges at one level")
            if P["span"].bit_length() == 64:
                edges.add("64-bit key span")
            for level, count, kind, shift in P["bins"]:
                if np.any((count == KCAP) & (kind == 1)):
                    edges.add(f"bucket of kCap at level {level}")
                if np.any((count == KCAP + 1) & (kind == 2)):
                    edges.add(f"range of kCap + 1 at level {level}")
                edges |= {f"bucket of {c}" for c in count[kind == 1]}
                if np.any((count == 1) & (shift > 0)):
                    edges.add("run of 1 in a wide bin")
                if np.any((count == KCAP + 1) & (kind == 0) & (shift == 0) & (level > 0)):
                    edges.add("run of kCap + 1 at shift 0")
            x = sel[ok, j]
            zero, subn = x == 0, (x != 0) & (np.abs(x) < np.finfo(np.float64).tiny)
            for is_run, label in ((False, "bucket"), (True, "run")):
                on = P["is_run"] == is_run
                pz = set(P["piece"][on & zero])
                if is_run and any(len(set(np.signbit(x[on & zero & (P["piece"] == b)]))) == 2 for b in pz):
                    edges.add("signed zeros in a run")
                if not is_run and pz & set(P["piece"][on & subn]):
                    edges.add("zeros and subnormals in a bucket")
    if want_reads is not None and reads != want_reads:
        fails.append(f"{name}: reads {reads}, the case is built for {want_reads}")
    return edges, fails, reads


def topk_report(case, k, largest, fault=None):
    """(edges, failures, reads per task) of a top-worlds catalogue case at (k, largest)."""
    name, values, sizes, planes = case
    edges, fails, reads = set(), [], []
    for o, n, sel in _group_tasks(values, sizes, planes):
        for j in range(len(planes)):
            if n <= SMALL_MAX:
                reads.append(1)
                continue
            P = topk_plan(sel[:, j], k, largest, fault, o)
            reads.append(P["reads"])
            fails += [f"{name} plane {j} k {k} largest {largest}: {e}" for e in P["errors"]]
            if not same(P["record"], ref_top(sel[:, j], k, largest, o)):
                fails.append(f"{name} plane {j} k {k} largest {largest}: record differs from ref_top")
            f = P["final"]
            edges.add(f"reads {P['reads']}")
            nf = P["nf"]
            edges |= {f"finite {lab}" for lab, c in (("kCap", KCAP), ("kCap + 1", KCAP + 1), ("k - 1", k - 1),
                                                     ("k", k), ("k + 1", k + 1)) if nf == c}
            if P["phase1_after"] is not None:
                edges.add(f"phase 1 after {P['phase1_after']} levels")
                fin = np.isfinite(sel[:, j])
                block = np.flatnonzero(fin & (order_key(np.where(fin, sel[:, j], 0.0)) ^ U64(MASK64 if largest else 0)
                                              == U64(f["lo"])))
                if block.size and block[0] == 0:
                    edges.add("block from world 0")
                if block.size and block[-1] == n - 1:
                    edges.add("block to world n - 1")
                if f["phase"] and np.any(~fin[f["ilo"]:f["ihi"] + 1]):
                    edges.add("non-finite worlds inside the index range")
            for level, phase, rb, hc in P["hits"]:
                if hc > 1 and rb == 0:
                    edges.add("rank kk - 1 first in its bin")
                if hc > 1 and rb == hc - 1:
                    edges.add("rank kk - 1 last in its bin")
            if P["kk"] == 1024 and f["below"] == 1023:
                edges.add("below area of 1023")
            if f["levels"] and f["count"] == KCAP and f["state"] == GATHER:
                edges.add("gathered range of kCap")
            if P["zero_split"]:
                edges.add("-0 and +0 split by a bin edge")
    return edges, fails, reads


def geometry_report(case, fault=None):
    name, sizes, n_p, kind, want = case
    G = geometry_of(case, fault)
    edges, fails = set(), []
    if G["order"] != sorted(G["order"]):
        edges.add(f"{'topk' if kind == 'topk' else 'rank'} route order differs from table order")
    Ts = [s[1] for s in G["slices"]]
    if Ts != want["slices"]:
        fails.append(f"{name}: slices of {Ts} tasks, the case is built for {want['slices']}")
    if G["launches"] != want["launches"]:
        fails.append(f"{name}: {G['launches']} launches, the case is built for {want['launches']}")
    for c in G["chunks"]:
        for n, wc, C in c:
            if n in want.get("chunks", {}) and (wc, C) != want["chunks"][n]:
                fails.append(f"{name}: {n} worlds in {C} chunks of {wc}, the case is built for {want['chunks'][n]}")
            edges |= {f"chunk {lab}" for lab, r in (("multiple", 0), ("multiple + 1", 1), ("multiple - 1", wc - 1))
                      if n % wc == r}
            if wc % PASS_THREADS == 0 and cdiv(n, max(1, 8 * NUM_SMS // len(c))) % PASS_THREADS and n % wc == 0:
                edges.add("chunk multiple of a rounded-up Wc")
    if kind != "topk":
        for t0, T, b in G["slices"]:
            if T == 0:
                fails.append(f"{name}: a slice of no task at task {t0}")
            if T == 1 and b > SCRATCH_CAP:
                edges.add("rank task alone over the cap")
            if SCRATCH_CAP - 8 < b <= SCRATCH_CAP:
                edges.add("rank slice within 8 bytes of the cap")
            if t0 % n_p:
                edges.add("rank slice boundary between a group's planes")
        if kind == "corr" and G["task_n"] and len(sizes) * (1 + n_p + n_p * n_p) * 8 > 1 << 20:
            edges.add("rank scratch behind a large covariance table")
    else:
        edges |= {f"topk slice of {T} tasks" for _, T in G["slices"]}
    return edges, fails


RANK_EDGES = ({f"reads {r}" for r in range(1, 8)} | {f"ranges at level {l}" for l in range(1, 6)}
              | {f"bucket of kCap at level {l}" for l in (1, 2, 4)}
              | {f"range of kCap + 1 at level {l}" for l in (1, 2, 4)}
              | {f"bucket of {c}" for c in (2, 3, 256, 257, 4096, 4097, 8191, 8192)}
              | {f"complete {c}" for c in (0, 1, KCAP, KCAP + 1)}
              | {"R ranges at one level", "run of 1 in a wide bin", "run of kCap + 1 at shift 0", "64-bit key span",
                 "incomplete in one plane", "signed zeros in a run", "zeros and subnormals in a bucket"})
TOPK_EDGES = ({f"reads {r}" for r in range(1, 9)} | {f"phase 1 after {L} levels" for L in range(0, 6)}
              | {f"finite {lab}" for lab in ("kCap", "kCap + 1", "k - 1", "k", "k + 1")}
              | {"block from world 0", "block to world n - 1", "non-finite worlds inside the index range",
                 "rank kk - 1 first in its bin", "rank kk - 1 last in its bin", "below area of 1023",
                 "gathered range of kCap", "-0 and +0 split by a bin edge"})
GEOMETRY_EDGES = {"rank route order differs from table order", "topk route order differs from table order",
                  "chunk multiple", "chunk multiple + 1", "chunk multiple - 1", "chunk multiple of a rounded-up Wc",
                  "rank task alone over the cap", "rank slice within 8 bytes of the cap",
                  "rank slice boundary between a group's planes", "rank scratch behind a large covariance table",
                  "topk slice of 1522 tasks", "topk slice of 1523 tasks", "topk slice of 1 tasks"}


def catalogue_outcome(fault=None):
    """(edges reached, failures) of the whole catalogue through the restatements, with `fault`."""
    edges, fails = set(), []
    for case in rank_catalogue():
        e, f, _ = rank_report(case, fault)
        edges |= e
        fails += f
    for case in topk_catalogue():
        for k in top_ks(case[1], case[2], case[3]):
            for largest in (False, True):
                e, f, _ = topk_report(case, k, largest, fault)
                edges |= e
                fails += f
    for case in GEOMETRY:
        e, f = geometry_report(case, fault)
        edges |= e
        fails += f
    missing = (RANK_EDGES | TOPK_EDGES | GEOMETRY_EDGES) - edges
    return edges, fails + [f"edge not reached: {m}" for m in sorted(missing)]


_CLEAN = {}


def clean_outcome():
    if not _CLEAN:
        _CLEAN["v"] = catalogue_outcome()
    return _CLEAN["v"]


# --------------------------------------------------------------------------- CPU


def _constants(*paths):
    src = re.sub(r"//[^\n]*", "", "".join(open(p).read() for p in paths))
    out = {}
    for m in re.finditer(r"constexpr\s+[\w ]+?\s+(k\w+)\s*=\s*([^;]+);", src):
        expr = re.sub(r"\b(\d+)(ull|u)\b", r"\1", m.group(2))
        if re.fullmatch(r"[\d\s<>()+*-]+", expr):
            out[m.group(1)] = eval(expr)  # digits and integer operators only
    return src, out


def _struct_bytes(src, name, consts):
    body = re.search(r"struct " + name + r" \{(.*?)\};", src, re.S).group(1)
    size, wide = 0, False
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        m = re.fullmatch(r"(unsigned long long|uint64_t|uint32_t)\s+(.+)", decl, re.S)
        width = 4 if m.group(1) == "uint32_t" else 8
        wide |= width == 8
        for nm in m.group(2).split(","):
            a = re.search(r"\[(.+)\]", nm)
            size += width * (eval(re.sub(r"k\w+", lambda t: str(consts[t.group(0)]), a.group(1))) if a else 1)
    return align8(size) if wide else size


def test_constants_match_the_sources_and_the_shared_header():
    shared = os.path.join(CSRC, "order_stats.cuh")  # the route split, chunk_of and the order helpers of both files
    rsrc, rk = _constants(os.path.join(CSRC, "rank_kernels.cu"), shared)
    tsrc, tk = _constants(os.path.join(CSRC, "topk_kernels.cu"), shared)
    h = open(os.path.join(CSRC, "sixdof_internal.h")).read()
    assert int(re.search(r"constexpr unsigned kNumSMs = (\d+);", h).group(1)) == NUM_SMS
    common = dict(kCap=KCAP, kBins=KBINS, kBinBits=KBINBITS, kSmallMax=SMALL_MAX, kWarpMax=WARP_MAX,
                  kPassThreads=PASS_THREADS, kScratchCap=SCRATCH_CAP)
    for got in (rk, tk):
        for name, want in common.items():
            assert got[name] == want, name
    assert rk["kLevels"] == RANK_LEVELS and tk["kLevels"] == TOPK_LEVELS and rk["kHeader"] == HEADER
    assert re.search(r"kBelow = B200_MAX_TOP_WORLDS;", tsrc)
    assert _struct_bytes(rsrc, "TRow", rk) == RANK_TROW and _struct_bytes(rsrc, "TState", rk) == RANK_TSTATE
    assert _struct_bytes(rsrc, "Range", rk) == RANK_RANGE
    assert _struct_bytes(tsrc, "TRow", tk) == TOPK_TROW and _struct_bytes(tsrc, "TState", tk) == TOPK_TSTATE
    assert TOPK_TASK_BYTES == 176_240 and SLICE_TASKS == 1523  # DESIGN section 5: slices of at most 1523 tasks
    squash = lambda s: re.sub(r"\s+", "", s)  # noqa: E731
    assert squash("return align8(sizeof(TState)) + 2 * R * sizeof(Range) + 2 * R * kBins * 4ull + n * 16ull + "
                  "align8(n * 4ull) + align8((n / 2 + 1) * 4ull) + align8(n * 4ull);") in squash(rsrc)
    assert squash("kTaskBytes = sizeof(TRow) + (sizeof(TState) + 7) / 8 * 8 + kBins * 4ull + (kBelow + kCap) * 12ull;"
                  ) in squash(tsrc)
    assert squash("std::max<uint64_t>(1, n / (kCap + 1))") in squash(rsrc)
    assert squash("*launches += 5 + 2 * kLevels;") in squash(rsrc) and squash("*launches += 5 + 2 * kLevels;") in \
        squash(tsrc)
    for src in (rsrc, tsrc):
        assert squash("want = std::max<uint64_t>(1, 8ull * kNumSMs / std::max<uint64_t>(1, T));") in squash(src)
        assert squash("(per + threads - 1) / threads * threads") in squash(src)
    for name in ("rank_kernels.cu", "topk_kernels.cu"):
        src = open(os.path.join(CSRC, name)).read()
        assert '#include "order_stats.cuh"' in src, name
        calls = re.findall(r"\bchunk_of\(([^()]*)\)", src)  # every chunk in blocks of the file's kPassThreads
        assert calls and all(squash(c).endswith(",kPassThreads") for c in calls), name


def test_restatements_on_hand_cases():
    # the key inverse, over the edges of the f64 range
    x = np.array([0.0, -0.0, 5e-324, -5e-324, 1.0, -np.finfo(np.float64).max, np.finfo(np.float64).max])
    assert same(key_value(order_key(x)), x) and rank_key(np.array([-0.0]))[0] == rank_key(np.array([0.0]))[0]
    assert (KEY_HIGH - KEY_LOW).bit_length() == 64
    # one world, one value, nothing complete
    assert rank_plan(np.zeros(0, np.uint64), 9000)[0]["reads"] == 1
    P, r = rank_plan(rank_key(np.full(9000, 2.0)), 9000)
    assert P["reads"] == 2 and np.all(r == 4500.5)
    # 2^20 worlds uniform over one binade: one level, the midranks of scipy
    v = np.random.default_rng(1).uniform(1.0, 2.0, (1 << 20) + 7)
    P, r = rank_plan(rank_key(v), v.size)
    assert P["reads"] == 3 and P["ranges"][1] == 1 and same(r, scipy.stats.rankdata(v))
    # the select: gathered whole, one level, and no finite world
    for n, want in ((9000, 2), (20000, 3)):
        v = np.random.default_rng(n).normal(size=n)
        v[:n - KCAP if n < 10000 else 0] = np.nan
        for k, largest in ((1, True), (1024, False)):
            P = topk_plan(v, k, largest)
            assert P["reads"] == want and same(P["record"], ref_top(v, k, largest))
    assert topk_plan(np.full(9000, np.nan), 3, True)["reads"] == 1
    # the geometry of the feature tests' launch count: one large group of 9000 worlds, one plane
    assert rank_geometry([9000], 1)["launches"] == 1 + 15 + 1
    assert topk_geometry([8193] * 1524, 1)["slices"] == [(0, 1523), (1523, 1)]


def test_sweep_reaches_every_boundary():
    edges, fails = clean_outcome()
    assert fails == []
    assert CAP_GAP < 8, CAP_GAP
    for case in GEOMETRY:
        assert geometry_report(case)[1] == [], case[0]


@pytest.mark.parametrize("fault", FAULTS)
def test_each_fault_fails_a_case(fault):
    _, fails = catalogue_outcome(fault)
    assert fails, f"{fault} passes every case"


# --------------------------------------------------------------------------- GPU


def launches(ex, call):
    n0 = ex.timings()["kernel_launches"]
    got = call()
    return got, ex.timings()["kernel_launches"] - n0


def restated_rank_reads(values, sizes, planes):
    """The restated reads of every task of a rank call, summed; the plans must keep in bounds."""
    total = 0
    for o, n, sel in _group_tasks(values, sizes, planes):
        ok = np.all(np.isfinite(sel), axis=1)
        for j in range(len(planes)):
            if n <= SMALL_MAX:
                total += 1
                continue
            P, _ = rank_plan(rank_key(sel[ok, j]), n)
            assert P["errors"] == []
            total += P["reads"]
    return total


def restated_topk_reads(values, sizes, planes, k, largest):
    total = 0
    for o, n, sel in _group_tasks(values, sizes, planes):
        for j in range(len(planes)):
            if n <= SMALL_MAX:
                total += 1
                continue
            P = topk_plan(sel[:, j], k, largest, offset=o)
            assert P["errors"] == []
            total += P["reads"]
    return total


def check_reads(got, tasks, want):
    assert round(got * tasks) == want and got == want / tasks, (got * tasks, want)


def check_ranks(ex, values, sizes, planes, geo=None):
    """R1 - R3 of one ranks call."""
    grouped = sizes is not None
    call = (lambda: ex.outcome_group_ranks(planes)) if grouped else (lambda: ex.outcome_ranks(planes))
    got, n = launches(ex, call)
    assert same(got, ref_ranks(values[:, planes], sizes))
    geo = geo or rank_geometry(sizes or [values.shape[0]], len(planes))
    assert n == geo["launches"]
    tasks = len(sizes or [0]) * len(planes)
    check_reads(ex.rank_reads(), tasks, restated_rank_reads(values, sizes, planes))


def check_top(ex, values, sizes, planes, k, largest):
    grouped = sizes is not None
    if grouped:
        got, n = launches(ex, lambda: ex.outcome_group_top_worlds(planes, k, largest))
        o = 0
        for g, m in enumerate(sizes):
            for jj, j in enumerate(planes):
                assert same(got[g, jj], ref_top(values[o:o + m, j], k, largest, o)), (g, j, k, largest)
            o += m
    else:
        got, n = launches(ex, lambda: ex.outcome_top_worlds(planes, k, largest))
        for jj, j in enumerate(planes):
            assert same(got[jj], ref_top(values[:, j], k, largest)), (j, k, largest)
    assert n == topk_geometry(sizes or [values.shape[0]], len(planes))["launches"], (k, largest)
    tasks = len(sizes or [0]) * len(planes)
    check_reads(ex.top_worlds_reads(), tasks, restated_topk_reads(values, sizes, planes, k, largest))


def _case(cases, name):
    return next(c for c in cases if c[0] == name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c[0] for c in rank_catalogue()])
def test_rank_catalogue(name):
    need_gpu()
    _, values, sizes, planes, want = _case(rank_catalogue(), name)
    assert rank_report(_case(rank_catalogue(), name))[2] == want
    with _only_values(values, "exact", groups=sizes) as ex:
        check_ranks(ex, values, sizes, planes)
        for j in range(len(planes)):  # each plane alone: its own complete worlds
            check_ranks(ex, values, sizes, [planes[j]])
        assert same(ex.outcome_values(), values)  # R4


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c[0] for c in topk_catalogue()])
def test_topk_catalogue(name):
    need_gpu()
    _, values, sizes, planes = _case(topk_catalogue(), name)
    with _only_values(values, "exact", groups=sizes) as ex:
        for k in top_ks(values, sizes, planes):
            for largest in (False, True):
                check_top(ex, values, sizes, planes, k, largest)
        assert same(ex.outcome_values(), values)  # R4


@pytest.mark.gpu
def test_one_case_of_each_in_fast():
    need_gpu()
    _, values, sizes, planes, _ = _case(rank_catalogue(), "level4_cap")
    with _only_values(values, "fast", groups=sizes) as ex:
        check_ranks(ex, values, sizes, planes)
        assert same(ex.outcome_values(), values)
    _, values, sizes, planes = _case(topk_catalogue(), "phase1_levels")
    with _only_values(values, "fast", groups=sizes) as ex:
        for k, largest in ((2, True), (1024, False)):
            check_top(ex, values, sizes, planes, k, largest)
        assert same(ex.outcome_values(), values)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c[0] for c in GEOMETRY])
def test_geometry(name):
    need_gpu()
    case = next(c for c in GEOMETRY if c[0] == name)
    _, sizes, n_p, kind, want = case
    values = geometry_values(case, GEOMETRY.index(case))
    planes = list(range(n_p))[::-1]
    geo = geometry_of(case)
    with _only_values(values, "exact", groups=sizes) as ex:
        if kind == "rank":
            check_ranks(ex, values, sizes, planes, geo)
        elif kind == "corr":
            # the covariance of the rank planes launches what the covariance of the outcome planes does, then one
            # launch turns each record into rho
            _, n_cov = launches(ex, lambda: ex.outcome_group_covariance(planes))
            rec, n = launches(ex, lambda: ex.outcome_group_rank_correlation(planes))
            assert n == geo["launches"] + n_cov + 1
            check_reads(ex.rank_reads(), len(sizes) * n_p, restated_rank_reads(values, sizes, planes))
            assert same(_check_rho(ex, values, planes, "exact", sizes), rec)
        else:
            for k, largest in ((16, True), (1024, False)):
                check_top(ex, values, sizes, planes, k, largest)
        assert same(ex.outcome_values(), values)
