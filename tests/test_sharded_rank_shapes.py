"""The world-sharded rank pass (rank_kernels.cu sharded_rank_round, behind b200_sixdof_sharded_ranks_* and
sharding.gather_ranks) round by round, against a restatement of its protocol, at the level, window, slice and
rank-count edges of its plan.

Restatement.  sharded_plan writes the protocol out in numpy over the keys of every rank.  Per task (group, plane), the
global plan: plan 0 makes a task of at most kCap = 8192 complete worlds over the ranks one piece (a tie run of one
world, else a bucket) and gives a larger one the range {0, shift 50}; each level then has 2^14 bins per range, a bin of
one world or at shift 0 a tie run, of at most kCap worlds a bucket, else a range at the next shift (max(shift - 14, 0)).
Ranges and buckets are numbered in the order the plans resolve them; a bucket's key offset kb is the running total of
bucket worlds.  The midranks built from the pieces must equal scipy, which checks the restatement itself.  Per rank,
its complete worlds and worlds of each group; the slices are cut from the most any rank holds (task_bytes_of,
kScratchCap, kMaxSliceTasks), so alike on every rank.  The exchanges, in order: the sizes (G n_ranks 8 bytes), per
slice one histogram exchange per level with ranges (64 KiB per range), then per window of W places the offsets
((s1 - s0) n_ranks 4 bytes) and the keys ((min(s1 + 8192, keys) - s0) 8 bytes), each cut into rounds of at most
32 MiB; a final 0.  W = max(1, min(4,186,111, 2^23 / n_ranks - 1)).  The reads: per task, one per level with ranges
and the scatter.  The launches of a rank: the mask and sizes if it holds worlds, per slice init and plan 0, a plan
per histogram exchange, the pass and the scatter where it holds worlds of the slice's groups, four per window.
test_constants_match_the_sources reads every constant, struct and formula the restatement uses from rank_kernels.cu
and order_stats.cuh, so an edit that leaves it behind fails without a GPU.

Driver.  drive() runs the real handles in lockstep and sums their partials; every other rank is virtual: a rank with no
worlds, whose partial is all zeros (its size slots, histograms, offsets and keys), which the header allows.  So one
handle runs any rank count.  A virtual rank may claim complete worlds in its size slots, for the group-size refusal
only: no fabricated histogram, offsets or keys word ever reaches the kernels.

Catalogue.  The planes are built from keys, so that each case sits on the edge it names: plan 0 at 1, 2, 8192 and 8193
complete worlds, a bin of 8192 and of 8193 worlds summed over three ranks at each of the shifts 50, 36, 22 and 8, a run
of 8193 signed zeros split over the ranks down to shift 0 (6 reads), R ranges at one level, a histogram exchange of
exactly 512 ranges (one round of 32 MiB) and of 525 (two rounds), windows under both terms of W's min, a bucket on
place W - 1 and on place W, a window where no bucket starts, a last window of one place, the sizes exchange in one
round and in two (4096 and 4097 ranks, 1024 groups), 2^22 and 2^22 + 1 ranks (the clamp), 2^23 - 1 ranks (an offsets
round 4 bytes below the cap), several slices, a slice filled to within 8 bytes of kScratchCap and the same with one
world more, a slice of one-world tasks (no exchange) between slices that exchange, a task alone over the cap, a rank
with none of a slice's groups, the rank holding the most not rank 0, and a call with no complete world.
test_sweep_reaches_every_boundary asserts the catalogue reaches each edge.

Contract, for every GPU case.  R1: every real rank's ranks equal ref_ranks bit for bit, as one handle's rows do.  R2:
every rank's round sizes equal the restated sequence.  R3: rank_reads() G p equals the restated reads.  R4: the
kernel_launches of each real rank over the rounds equal the restated count.  R5: the outcome planes keep their bits.
The rank kernels take no math mode: the sweep runs in exact, one case in fast.

Sensitivity.  Each of FAULTS, injected into the restatement one at a time, must fail a catalogue case or miss an
edge."""

import hashlib
import os
import re

import numpy as np
import pytest
import scipy.stats

from elodin_b200 import _lib
from tests.ensemble_util import need_gpu
from tests.test_outcome_rank_correlation import _only_values, ref_ranks, same
from tests.test_rank_topk_shapes import (CSRC, HEADER, KBINBITS, KBINS, KCAP, PASS_THREADS, RANK_LEVELS, RANK_RANGE,
                                         SCRATCH_CAP, U64, _bucket_midranks, _constants, _struct_bytes, align8,
                                         key_value, rank_key, u64)

ROUND_CAP = 32 << 20
MAX_SLICE_TASKS = 65535
SROW, TASK_STATE, PIECE = 48, 64, 32
TASK_FIXED = SROW + TASK_STATE + 24     # a task's row, state and three offsets (two pools, keys)
MAX_WORLDS = (0x80000000 // KBINS) * (KCAP + 1) - 1  # 1,073,872,895: what a world state can index
MAX_RANKS = (ROUND_CAP // 4) - 1        # 2^23 - 1: one window place's offsets below the cap
LEVEL0_SHIFT = 64 - KBINBITS

FAULTS = ("plan0_from_kmin", "r_from_rank", "bucket_below_cap", "no_run_at_shift0", "w_without_minus_1",
          "w_without_max", "keys_without_tail", "rounds_cap_minus_4", "slices_from_rank", "pass_on_empty_rank",
          "reads_with_mask", "sizes_of_4_bytes")


# --------------------------------------------------------------------------- the protocol, restated


def task_plan(keys, fault=None, R=None, owner=None):
    """The global plan of one task over the rank keys of its complete worlds on every rank (owner: each world's
    rank) -> (plan, midranks).  plan: ranges per level, buckets [(count, level)] in kb order, the resolved bins
    [(level, shift, counts, kinds)] (kind 0 run, 1 bucket, 2 range), the bins of kCap and kCap + 1 worlds [(count,
    kind, shift, the most worlds of the bin one rank holds)], errors."""
    keys = np.asarray(keys, dtype=np.uint64)
    N = keys.size
    owner = np.zeros(N, np.int64) if owner is None else owner
    P = dict(ranges=[0] * (RANK_LEVELS + 2), buckets=[], bins=[], errors=[], runs_at_0=[], cap_bins=[])
    ranks = np.full(N, np.nan)
    R = max(1, N // (KCAP + 1)) if R is None else R
    if N <= KCAP:
        if N == 1:
            ranks[:] = 1.0
        elif N > 1:
            P["buckets"].append((N, 0))
            ranks[:] = _bucket_midranks(keys, np.zeros(N))
        return P, ranks
    w = np.arange(N)
    if fault == "plan0_from_kmin":  # the unsharded plan 0: the range from kmin, as wide as kmax - kmin
        kmin = int(keys.min())
        span = int(keys.max()) - kmin
        if span == 0:
            ranks[:] = (N + 1) / 2.0
            return P, ranks
        rlo, rsh = np.array([kmin], np.uint64), np.array([max(span.bit_length() - KBINBITS, 0)])
    else:
        rlo, rsh = np.array([0], np.uint64), np.array([LEVEL0_SHIFT])
    rbase = np.array([0], np.int64)
    rid = np.zeros(N, np.int64)
    level = 1
    while True:
        nr = rlo.size
        P["ranges"][level] = nr
        if nr > R:
            P["errors"].append(f"{nr} ranges at level {level}: the area holds {R}")
        b = ((keys[w] - rlo[rid]) >> rsh[rid].astype(np.uint64)).astype(np.int64)
        if b.size and b.max() >= KBINS:
            P["errors"].append(f"bin {b.max()} at level {level}")
            b = np.minimum(b, KBINS - 1)
        uniq, wbin, count = np.unique(rid * KBINS + b, return_inverse=True, return_counts=True)
        ur, ub = uniq // KBINS, uniq % KBINS
        cum = np.cumsum(count) - count
        base = rbase[ur] + cum - cum[np.searchsorted(ur, ur)]
        shift = rsh[ur]
        run = (count == 1) | ((shift == 0) & (fault != "no_run_at_shift0"))
        bucket = ~run & ((count < KCAP) if fault == "bucket_below_cap" else (count <= KCAP))
        rng = ~run & ~bucket
        P["bins"].append((level, int(rsh[0]) if nr else 0, count, np.where(run, 0, np.where(bucket, 1, 2)), shift))
        P["runs_at_0"] += list(count[run & (shift == 0)])
        for i in np.flatnonzero((count == KCAP) | (count == KCAP + 1)):
            most = int(np.unique(owner[w[wbin == i]], return_counts=True)[1].max())
            P["cap_bins"].append((int(count[i]), int(0 if run[i] else 1 if bucket[i] else 2), int(shift[i]), most))
        wr, wb = run[wbin], bucket[wbin]
        ranks[w[wr]] = base[wbin[wr]] + (count[wbin[wr]] + 1) / 2.0
        if wb.any():
            ranks[w[wb]] = _bucket_midranks(keys[w[wb]], base[wbin[wb]])
        P["buckets"] += [(int(c), level) for c in count[bucket]]
        if not rng.any():
            break
        if level == RANK_LEVELS:
            P["errors"].append(f"ranges past level {RANK_LEVELS}")
            break
        live = rng[wbin]
        rid_of = np.full(count.size, -1)
        rid_of[rng] = np.arange(int(rng.sum()))
        w, rid = w[live], rid_of[wbin[live]]
        rlo = rlo[ur[rng]] + (ub[rng].astype(np.uint64) << shift[rng].astype(np.uint64))
        rsh = np.maximum(shift[rng] - KBINBITS, 0)
        rbase = base[rng]
        level += 1
    return P, ranks


def shard_ranges(N):
    return max(1, N // (KCAP + 1)) if N > KCAP else 0


def task_bytes_of(N, lcn, n, R=None):
    R = shard_ranges(N) if R is None else R
    return TASK_FIXED + align8(2 * R * RANK_RANGE + lcn * PIECE + align8(n * 4) + align8(lcn * 4) + lcn * 8)


def cut_slices(tasks, bytes_of):
    """The first task of every slice, then the task count."""
    out, t = [], 0
    while t < len(tasks):
        out.append(t)
        b = HEADER + bytes_of(t)
        for t in range(t + 1, len(tasks) + 1):
            if t == len(tasks) or b + bytes_of(t) > SCRATCH_CAP or t - out[-1] == MAX_SLICE_TASKS:
                break
            b += bytes_of(t)
    return out + [len(tasks)]


def window_places(n_ranks, fault=None):
    per = ROUND_CAP // (4 * n_ranks)
    m = min((ROUND_CAP - KCAP * 8) // 8, per)
    if fault == "w_without_minus_1":
        return max(1, m)
    if fault == "w_without_max":
        return (m - 1) % (1 << 64)
    return max(2, m) - 1


def rounds_of(nbytes, fault=None):
    cap = ROUND_CAP - 4 if fault == "rounds_cap_minus_4" else ROUND_CAP
    out = []
    while nbytes > 0:
        out.append(min(cap, nbytes))
        nbytes -= out[-1]
    return out


class Split:
    """n_ranks ranks; `real` {rank: (a, b)}: the global worlds [a, b) of each real rank (the others hold none);
    `claim` {rank: [(complete, worlds) per group]}: what a virtual rank's size slots claim."""

    def __init__(self, n_ranks, real, claim=None):
        self.n_ranks, self.real, self.claim = n_ranks, dict(real), claim or {}


def cut_groups(sizes, a, b):
    out, g0 = [], 0
    for s in sizes:
        out.append(max(0, min(g0 + s, b) - max(g0, a)))
        g0 += s
    return out


PLAN_FAULTS = ("plan0_from_kmin", "bucket_below_cap", "no_run_at_shift0")  # r_from_rank: through R
_PLANS = {}


def sharded_plan(values, sizes, planes, split, fault=None):
    """The protocol of one sharded call -> dict: rounds, reads, launches {real rank: n}, midranks [M, p], slices (task
    counts, bytes, whether each exchanges and which real ranks hold worlds of its groups), W, windows [(s0, s1)],
    histogram exchanges (bytes), the task plans and the edges' raw facts; errors.  The task plans are kept by the
    task's values and owners, so that the sweep's faults outside the plans reuse them."""
    M = values.shape[0]
    sizes_ = [M] if sizes is None else list(sizes)
    G, p, nR = len(sizes_), len(planes), split.n_ranks
    sel = values[:, planes]
    ok = np.all(np.isfinite(sel), axis=1)
    o = np.cumsum([0] + sizes_)
    owner = np.full(M, -1, np.int64)
    for r, (a, b) in split.real.items():
        owner[a:b] = r
    out = dict(errors=[], rounds=[], launches={}, ranks=np.full((M, p), np.nan), hist=[], windows=[], plans={})
    # the size slots: per rank and group, (complete, worlds)
    slots = {}
    for r, (a, b) in split.real.items():
        slots[r] = [(int(ok[max(a, o[g]):min(b, o[g + 1])].sum()) if min(b, o[g + 1]) > max(a, o[g]) else 0,
                     max(0, min(b, o[g + 1]) - max(a, o[g]))) for g in range(G)]
    slots.update(split.claim)
    n_global = [sum(s[g][0] for s in slots.values()) for g in range(G)]
    l_most = [max(s[g][0] for s in slots.values()) for g in range(G)]
    w_most = [max(s[g][1] for s in slots.values()) for g in range(G)]
    out["n_global"], out["l_most"], out["w_most"], out["slots"] = n_global, l_most, w_most, slots
    out["rounds"] += rounds_of(G * nR * (4 if fault == "sizes_of_4_bytes" else 8), fault)
    for r in split.real:
        out["launches"][r] = 2 if sum(w for _, w in slots[r]) else 0
    if max(n_global) > MAX_WORLDS:
        out["refused"] = True
        out["rounds"].append(0)
        return out
    tasks = [(g, j) for g in range(G) if n_global[g] for j in range(p)]
    out["tasks"] = tasks
    # the global plans, and their midranks against scipy
    plans = {}
    for g, j in tasks:
        w = np.arange(o[g], o[g + 1])[ok[o[g]:o[g + 1]]]
        R = max(1, n_global[g] // (KCAP + 1))
        if fault == "r_from_rank" and n_global[g] > KCAP:  # the ranges sized from each rank's own count
            R = min(max(1, s[g][0] // (KCAP + 1)) for s in slots.values() if s[g][0])
        x = np.ascontiguousarray(sel[w, j])
        key = (hashlib.blake2b(x.tobytes() + owner[w].tobytes()).digest(), fault if fault in PLAN_FAULTS else None, R)
        if key not in _PLANS:
            P, r = task_plan(rank_key(x), fault, R, owner[w])
            bad = w.size and not same(r, scipy.stats.rankdata(x, method="average"))
            _PLANS[key] = (P, r, P["errors"] + (["midranks differ from scipy"] if bad else []))
        P, r, errors = _PLANS[key]
        plans[(g, j)] = P
        out["errors"] += [f"task ({g}, {j}): {e}" for e in errors]
        out["ranks"][w, j] = r
    out["plans"] = plans
    out["reads"] = sum(1 + sum(1 for nr in P["ranges"] if nr) for P in plans.values())
    if fault == "reads_with_mask":
        out["reads"] += len(tasks)

    def bytes_of(t, r=None):
        g = tasks[t][0]
        if r is None:
            return task_bytes_of(n_global[g], l_most[g], w_most[g])
        return task_bytes_of(n_global[g], slots[r][g][0], slots[r][g][1])

    slices = cut_slices(tasks, bytes_of)
    if fault == "slices_from_rank":
        cuts = {tuple(cut_slices(tasks, lambda t, r=r: bytes_of(t, r))) for r in split.real}
        if len(cuts) > 1:
            out["errors"].append("the ranks cut different slices")
        slices = list(next(iter(cuts)))
    out["slices"] = [slices[k + 1] - slices[k] for k in range(len(slices) - 1)]
    out["slice_bytes"] = [HEADER + sum(bytes_of(t) for t in range(slices[k], slices[k + 1]))
                          for k in range(len(slices) - 1)]
    out["slice_exchanges"], out["slice_holds"], out["slice_one_world"] = [], [], []
    W = window_places(nR, fault)
    out["W"] = W
    if W == 0:
        out["errors"].append("a window of no place")
        return out
    out["bucket_starts"] = []
    for k in range(len(slices) - 1):
        ts = tasks[slices[k]:slices[k + 1]]
        holds = {r: any(slots[r][g][1] for g, _ in ts) for r in split.real}
        out["slice_holds"].append(holds)
        out["slice_one_world"].append(all(n_global[g] == 1 for g, _ in ts))
        n_rounds = len(out["rounds"])
        for level in range(1, RANK_LEVELS + 1):
            nr = sum(plans[t]["ranges"][level] for t in ts)
            if not nr:
                break
            out["hist"].append(nr * KBINS * 4)
            out["rounds"] += rounds_of(nr * KBINS * 4, fault)
            for r in split.real:
                out["launches"][r] += 1 + (holds[r] or fault == "pass_on_empty_rank")
        for r in split.real:
            out["launches"][r] += 2 + (holds[r] or fault == "pass_on_empty_rank")  # init, plan 0; the scatter
        starts, keys = [], 0
        for t in ts:
            kb = 0
            for c, _ in plans[t]["buckets"]:
                starts.append((keys + kb, c))
                kb += c
            keys += kb
        out["bucket_starts"].append(starts)
        s0 = 0
        while s0 < keys:
            s1 = min(s0 + W, keys)
            out["windows"].append((s0, s1, keys))
            out["rounds"] += rounds_of((s1 - s0) * nR * 4, fault)
            tail = s1 if fault == "keys_without_tail" else min(s1 + KCAP, keys)
            out["rounds"] += rounds_of((tail - s0) * 8, fault)
            for r in split.real:
                out["launches"][r] += 4
            s0 = s1
        out["slice_exchanges"].append(len(out["rounds"]) > n_rounds)
    out["rounds"].append(0)
    return out


def rle(rounds):
    out = []
    for n in rounds:
        if out and out[-1][0] == n:
            out[-1][1] += 1
        else:
            out.append([n, 1])
    return [tuple(x) for x in out]


# --------------------------------------------------------------------------- the catalogue

KEY_ONE = int(rank_key(np.array([1.0]))[0])
KEY_TINY = int(rank_key(np.array([1e-200]))[0])  # a level-1 bin of its own, far below 1.0's


def _cluster(a, level, partners):
    """Offsets of `a` worlds in one bin at `level` (shift 50 - 14 (level - 1)) of a level-(level - 1) bin, and
    `partners` worlds in the next bin of the same level-(level - 1) bin; a next level resolves the cluster into runs of
    one world (or, at shift 8, ties on 256 keys)."""
    s = LEVEL0_SHIFT - KBINBITS * (level - 1)
    start = (KEY_ONE >> (s + KBINBITS) << (s + KBINBITS)) + (5 << s)
    step = max(1, (1 << s) >> KBINBITS)
    off = np.arange(a) % 256 if s < KBINBITS else np.arange(a) * step
    return u64(U64(start) + off.astype(U64), U64(start + (1 << s)) + np.arange(partners, dtype=U64))


def _fillers(rng, n):
    """n keys spread over the level-1 bins of values in [1e-200, 1e-100): away from every cluster."""
    hi = int(rank_key(np.array([1e-100]))[0])
    return rng.integers(KEY_TINY, hi, n, dtype=np.uint64)


def _shuffle(rng, keys):
    return key_value(keys[rng.permutation(keys.size)])


def _clusters_plane(rng, n_clusters):
    """n_clusters clusters of kCap + 1 worlds, each alone in a level-1 bin (a range of level 2) whose keys fall
    8192 into one level-2 bin (a bucket) and 1 into the next (a run)."""
    c0 = KEY_ONE >> LEVEL0_SHIFT << LEVEL0_SHIFT
    keys = [U64(c0 + (c << LEVEL0_SHIFT)) + (np.arange(KCAP + 1, dtype=np.uint64) << U64(23))
            for c in range(n_clusters)]
    return _shuffle(rng, u64(*keys))


KEY_LOW, KEY_HIGH = (int(k) for k in rank_key(np.array([-np.finfo(np.float64).max, np.finfo(np.float64).max])))


def _slice_at_cap():
    """(nA, nD): groups whose two tasks (one plane, every world complete, on one rank) fill a slice to within 8 bytes
    of kScratchCap: the largest nA that fits beside a group of nD, for the first nD that leaves less than 8."""
    f = lambda n: task_bytes_of(n, n, n)  # noqa: E731
    for nD in range(20_000, 60_000):
        room = SCRATCH_CAP - HEADER - f(nD)
        lo, hi = 0, room // 40
        while lo < hi:
            mid = (lo + hi + 1) // 2
            lo, hi = (mid, hi) if f(mid) <= room else (lo, mid - 1)
        if room - f(lo) < 8:
            return lo, nD
    raise AssertionError("no fill within 8 bytes of the cap")


def catalogue():
    """[(name, values [M, p], sizes or None, planes, Split, want)]: want holds what each case is built to give: its
    rounds (run-length), reads and real ranks' launches where named."""
    rng = np.random.default_rng(31)
    cases = []
    # plan 0 at 1, 2, 8192 and 8193 complete worlds over 4 ranks, none holding more than 4097 of a group
    sizes = [1, 2, KCAP, KCAP + 1]
    v = rng.normal(0, 1, (sum(sizes), 2))
    cases.append(("plan0", v, sizes, [0, 1], Split(4, {0: (0, 4100), 1: (4100, 8195), 2: (8195, 12292),
                                                       3: (12292, 16388)}),
                  dict(reads=2 * (1 + 1 + 1 + 2))))
    # a bin of 8192 and of 8193 at each of the shifts 50, 36, 22, 8, and a run of 8193 signed zeros to shift 0, the
    # worlds shuffled over three ranks (none holding more than half of a bin)
    n_fill = 300
    M = KCAP + 2 + n_fill
    planes = []
    for level in (1, 2, 3, 4):
        for a in (KCAP, KCAP + 1):
            planes.append(_shuffle(rng, u64(_cluster(a, level, KCAP + 2 - a), _fillers(rng, n_fill))))
    zeros = np.concatenate([np.zeros(KCAP + 1), key_value(_fillers(rng, M - KCAP - 1))])[rng.permutation(M)]
    thirds = [0, M // 3, 2 * M // 3, M]
    zeros[:thirds[1]][zeros[:thirds[1]] == 0] = -0.0  # -0 on rank 0, +0 on ranks 1 and 2
    planes.append(zeros)
    cases.append(("levels", np.stack(planes, 1), None, list(range(9)),
                  Split(3, {r: (thirds[r], thirds[r + 1]) for r in range(3)}),
                  dict(reads=sum(2 * L + 3 for L in (1, 2, 3, 4)) + 6)))  # L + 1 and L + 2 reads at level L; the run
    # one histogram exchange of exactly 512 ranges (16 planes x 32): one round of 32 MiB; 2 ranks, so W is the first
    # term of its min, and the slice's 4,194,304 bucket keys take two windows
    v = np.stack([_clusters_plane(rng, 32) for _ in range(16)], 1)
    half = v.shape[0] // 2
    cases.append(("hist_512", v, None, list(range(16)), Split(2, {0: (0, half), 1: (half, v.shape[0])}),
                  dict(rounds=rle([16, 16 * KBINS * 4, ROUND_CAP, 4_186_111 * 8, (4_186_111 + KCAP) * 8, 8193 * 8,
                                   8193 * 8, 0]), reads=16 * 3)))
    # 525 ranges (25 planes x 21 = R of a group of 21 x 8193): rounds of 32 MiB and 851,968 bytes; real ranks 0 and 2
    # of 3, the middle one virtual
    v = np.stack([_clusters_plane(rng, 21) for _ in range(25)], 1)
    third = v.shape[0] // 3
    w3 = window_places(3)
    keys = 25 * 21 * KCAP
    cases.append(("hist_525", v, None, list(range(25)), Split(3, {0: (0, third), 2: (third, v.shape[0])}),
                  dict(rounds=[(24, 1), (25 * KBINS * 4, 1), (ROUND_CAP, 1), (851_968, 1), (w3 * 12, 1),
                               ((w3 + KCAP) * 8, 1), ((keys - w3) * 12, 1), ((keys - w3) * 8, 1), (0, 1)],
                       reads=25 * 3)))
    # 1024 groups of 2 worlds on 4096 and on 4097 ranks: the sizes in one round and in two; W = 2047 (a bucket on
    # place W - 1 and a last window of one place) and W = 2046 (a bucket on place W)
    sizes = [2] * 1024
    v = rng.normal(0, 1, (2048, 1))
    cases.append(("ranks_4096", v, sizes, [0], Split(4096, {0: (0, 2048)}),
                  dict(rounds=rle([ROUND_CAP, 2047 * 4096 * 4, 2048 * 8, 4096 * 4, 8, 0]),
                       reads=1024, launches={0: 2 + 2 + 1 + 8})))
    cases.append(("ranks_4097", v, sizes, [0], Split(4097, {4096: (0, 2048)}),
                  dict(rounds=[(ROUND_CAP, 1), (8192, 1), (2046 * 4097 * 4, 1), (2048 * 8, 1), (2 * 4097 * 4, 1),
                               (16, 1), (0, 1)], reads=1024)))
    # 5000 ranks, the real one last: W = 1676, 40,384 keys in 25 windows, the first buckets of 8192 keys spanning
    # windows where none starts
    sizes = [8192, 5000, 7000]
    v = rng.normal(0, 1, (sum(sizes), 2))
    keys, W = 2 * sum(sizes), 1676
    r = [3 * 5000 * 8]
    for s0 in range(0, keys, W):
        s1 = min(s0 + W, keys)
        r += [(s1 - s0) * 5000 * 4, (min(s1 + KCAP, keys) - s0) * 8]
    cases.append(("ranks_5000", v, sizes, [0, 1], Split(5000, {4999: (0, sum(sizes))}),
                  dict(rounds=rle(r + [0]), reads=6, launches={4999: 2 + 2 + 1 + 4 * 25})))
    # 2^22 and 2^22 + 1 ranks, a bucket of two worlds: W = 1, from the min - 1 and from the clamp; 2^23 - 1 ranks:
    # an offsets round 4 bytes below the cap
    v = np.array([[2.5], [-1.0]])
    for n in (1 << 22, (1 << 22) + 1, MAX_RANKS):
        cases.append((f"ranks_{n}", v, None, [0], Split(n, {n - 1 if n % 2 else 0: (0, 2)}),
                      dict(rounds=rle(rounds_of(n * 8) + [n * 4, 16, n * 4, 8, 0]), reads=1)))
    # several slices (1200 tasks of 8192 complete worlds over 2 ranks holding a third and two thirds)
    sizes = [KCAP] * 48
    v = rng.normal(0, 1, (sum(sizes), 25))
    cut = sum(sizes) // 3
    cases.append(("slices", v, sizes, list(range(25)), Split(2, {0: (0, cut), 1: (cut, sum(sizes))}),
                  dict(reads=1200)))
    # uneven splits: rank 0 holds only group 0, none of it complete, so none of the slice's groups (no pass, no
    # scatter), and rank 2, not rank 0, holds the most of group 2
    sizes = [3000, 9000, 20000]
    v = rng.normal(0, 1, (sum(sizes), 2))
    v[:3000, 1] = np.nan
    v[3000:3100, 0] = np.inf
    cases.append(("uneven", v, sizes, [0, 1], Split(3, {0: (0, 3000), 1: (3000, 18000), 2: (18000, 32000)}),
                  dict(launches={0: 2 + 2 + 1 + 4})))  # mask, sizes; init, plan 0; the level-1 plan; a window
    # slices: groups A and D fill the first slice to within 8 bytes of the cap on the rank holding them (its worlds
    # uniform over the keys, so level 1 resolves them into buckets), two groups of one world make a slice of their own,
    # which exchanges nothing, and group C's task alone needs more than the cap; with one world more in D, D's task
    # starts the second slice
    nA, nD = _slice_at_cap()
    nC = nA + nD + 10
    for name, d, want in (("slice_at_cap", nD, [2, 2, 1]), ("slice_past_cap", nD + 1, [1, 3, 1])):
        sizes = [nA, d, 1, 1, nC]
        keys = rng.integers(KEY_LOW, KEY_HIGH, sum(sizes), dtype=np.uint64, endpoint=True)
        v = key_value(keys)[:, None]
        cases.append((name, v, sizes, [0], Split(2, {0: (0, sum(sizes))}), dict(slices=want, reads=3 * 2 + 2)))
    # no group has a complete world: the sizes, then 0
    v = np.full((5000, 2), np.nan)
    v[::2, 0] = 1.0
    cases.append(("none_complete", v, [2000, 3000], [0, 1], Split(3, {0: (0, 2500), 2: (2500, 5000)}),
                  dict(rounds=[(2 * 3 * 8, 1), (0, 1)], reads=0, launches={0: 2, 2: 2})))
    return cases


_CASES = []


def cases():
    if not _CASES:
        _CASES.extend(catalogue())
    return _CASES


def report(case, fault=None):
    """(edges, failures, plan) of one case through the restatement."""
    name, values, sizes, planes, split, want = case
    P = sharded_plan(values, sizes, planes, split, fault)
    fails = [f"{name}: {e}" for e in P["errors"]]
    edges = set()
    if "rounds" in want and rle(P["rounds"]) != [tuple(x) for x in want["rounds"]]:
        fails.append(f"{name}: rounds {rle(P['rounds'])[:8]}, the case is built for {want['rounds'][:8]}")
    if "reads" in want and P.get("reads") != want["reads"]:
        fails.append(f"{name}: reads {P.get('reads')}, the case is built for {want['reads']}")
    if "slices" in want and P.get("slices") != want["slices"]:
        fails.append(f"{name}: slices of {P.get('slices')} tasks, the case is built for {want['slices']}")
    for r, n in want.get("launches", {}).items():
        if P["launches"].get(r) != n:
            fails.append(f"{name}: rank {r} launches {P['launches'].get(r)}, the case is built for {n}")
    if P["errors"] or "tasks" not in P:
        return edges, fails, P
    nR = split.n_ranks
    for (g, j), T in P["plans"].items():
        edges |= {f"plan 0 of {c}" for c in (1, 2, KCAP, KCAP + 1) if P["n_global"][g] == c}
        # a bin of kCap worlds is a bucket and one of kCap + 1 a range only by the counts summed over the ranks
        edges |= {f"bin of {c} at shift {s}" for c, k, s, most in T["cap_bins"]
                  if k == (1 if c == KCAP else 2) and 2 * most <= c}
        if any(c == KCAP + 1 for c in T["runs_at_0"]):
            edges.add("run of 8193 at shift 0")
        R = shard_ranges(P["n_global"][g])
        if R > 1 and max(T["ranges"]) == R:
            edges.add("R ranges at one level")
    if name == "levels":
        z = values[:, planes[-1]] == 0
        on0 = np.arange(values.shape[0]) < split.real[0][1]
        x = values[:, planes[-1]]
        if np.signbit(x[z & on0]).all() and not np.signbit(x[z & ~on0]).any():
            edges.add("-0 and +0 on different ranks in one run")
    edges |= {"histogram exchange of 512 ranges" for h in P["hist"] if h == 512 * KBINS * 4}
    edges |= {"histogram exchange in rounds" for h in P["hist"] if h > ROUND_CAP}
    G = len(P["n_global"])
    edges.add("sizes in one round" if G * nR * 8 <= ROUND_CAP else "sizes in rounds")
    W = P["W"]
    edges.add("W from the first term" if W == (ROUND_CAP - KCAP * 8) // 8 - 1 and P["windows"] else
              "W from the second term" if P["windows"] and W > 1 else "W clamped to 1" if W == 1 and
              ROUND_CAP // (4 * nR) <= 1 else "W of 1 from the min - 1" if W == 1 else "")
    for starts in P["bucket_starts"]:
        places = {s for s, c in starts if c > 1}
        if any(s % W == W - 1 for s in places) and W > 1:
            edges.add("bucket on place W - 1")
        if any(s % W == 0 and s > 0 for s in places):
            edges.add("bucket on place W")
    for s0, s1, keys in P["windows"]:
        if not any(s0 <= s < s1 for starts in P["bucket_starts"] for s, _ in starts):
            edges.add("window with no bucket start")
        if s1 - s0 == 1 and s1 == keys and W > 1:
            edges.add("last window of one place")
    if ROUND_CAP - 4 in P["rounds"]:
        edges.add("offsets round 4 bytes below the cap")
    if len(P["slices"]) > 1:
        edges.add("several slices")
    if any(not all(h.values()) for h in P["slice_holds"]):
        edges.add("a rank with none of a slice's groups")
    for k, (T, b) in enumerate(zip(P["slices"], P["slice_bytes"])):
        if SCRATCH_CAP - 8 < b <= SCRATCH_CAP:
            edges.add("slice within 8 bytes of the cap")
        if T == 1 and b > SCRATCH_CAP:
            edges.add("task alone over the cap")
        if 0 < k < len(P["slices"]) - 1 and P["slice_one_world"][k] and not P["slice_exchanges"][k] \
                and P["slice_exchanges"][k - 1] and P["slice_exchanges"][k + 1]:
            edges.add("slice of one-world tasks between slices that exchange")
    for g in range(G):
        if P["n_global"][g] and max(P["slots"], key=lambda r: P["slots"][r][g][0]) != 0:
            edges.add("the rank holding the most is not rank 0")
    if not P["tasks"]:
        edges.add("no complete world")
    edges.discard("")
    return edges, fails, P


EDGES = ({f"plan 0 of {c}" for c in (1, 2, KCAP, KCAP + 1)}
         | {f"bin of {c} at shift {s}" for c in (KCAP, KCAP + 1) for s in (50, 36, 22, 8)}
         | {"run of 8193 at shift 0", "-0 and +0 on different ranks in one run", "R ranges at one level",
            "histogram exchange of 512 ranges", "histogram exchange in rounds", "sizes in one round", "sizes in rounds",
            "W from the first term", "W from the second term", "W clamped to 1", "W of 1 from the min - 1",
            "bucket on place W - 1", "bucket on place W", "window with no bucket start", "last window of one place",
            "offsets round 4 bytes below the cap", "several slices", "a rank with none of a slice's groups",
            "the rank holding the most is not rank 0", "no complete world", "slice within 8 bytes of the cap",
            "task alone over the cap", "slice of one-world tasks between slices that exchange"})

_CLEAN = {}


def catalogue_outcome(fault=None):
    edges, fails = set(), []
    for case in cases():
        e, f, _ = report(case, fault)
        edges |= e
        fails += f
    return edges, fails + [f"edge not reached: {m}" for m in sorted(EDGES - edges)]


# --------------------------------------------------------------------------- CPU


def test_constants_match_the_sources():
    src, k = _constants(os.path.join(CSRC, "rank_kernels.cu"), os.path.join(CSRC, "order_stats.cuh"))
    for name, want in dict(kCap=KCAP, kBins=KBINS, kBinBits=KBINBITS, kLevels=RANK_LEVELS, kPassThreads=PASS_THREADS,
                           kScratchCap=SCRATCH_CAP, kHeader=HEADER, kRoundCap=ROUND_CAP,
                           kMaxSliceTasks=MAX_SLICE_TASKS).items():
        assert k[name] == want, name
    h = open(os.path.join(CSRC, "sixdof_internal.h")).read()
    ts = re.search(r"struct TaskState \{(.*?)\};", h, re.S).group(1)
    assert _struct_bytes("struct TaskState {" + re.sub(r"//[^\n]*", "", ts) + "};", "TaskState", k) == TASK_STATE
    assert _struct_bytes(src, "SRow", k) == SROW and _struct_bytes(src, "Piece", k) == PIECE
    assert _struct_bytes(src, "Range", k) == RANK_RANGE
    squash = lambda s: re.sub(r"\s+", "", s)  # noqa: E731
    S = squash(src)
    for text in (
            "return 2 * R * sizeof(Range) + lcn * sizeof(Piece) + align8(n * 4ull) + align8(lcn * 4ull) + lcn * 8ull;",
            "return sizeof(SRow) + sizeof(TaskState) + 24 + align8(shard_area_bytes(shard_ranges(N), lcn, n));",
            "uint64_t shard_ranges(uint64_t N) { return N > kCap ? ranges_of(N) : 0; }",
            "std::max<uint64_t>(1, n / (kCap + 1))",
            "A.rg1[0] = Range{0ull, 64 - kBinBits, 0};",
            "const bool run = r.N == 1;",
            "if (g <= 1 || R.shift == 0) continue; if (g <= kCap) {",
            "const uint32_t next_shift = R.shift > kBinBits ? R.shift - kBinBits : 0;",
            "if (bytes + most(t) > kScratchCap || t - Q.slices.back() == kMaxSliceTasks) break;",
            "return task_bytes_of(Q.n_global[g], Q.l_most[g], Q.w_most[g]);",
            "Q.wkeys = std::max<uint64_t>(2, std::min((kRoundCap - kCap * 8ull) / 8, "
            "kRoundCap / (4ull * Q.n_ranks))) - 1;",
            "const uint64_t bytes = (s1 - s0) * Q.n_ranks * 4;",
            "const uint64_t bytes = (std::min(s1 + kCap, Q.keys) - s0) * 8;",
            "const uint64_t bytes = G * Q.n_ranks * 8;",
            "words[t] = (uint64_t)Q.st[t].nr[next] * kBins;",
            "Q.reads += refine;", "Q.reads += T;",
            "if (r.grid) { shard_pass_kernel", "if (r.grid) { shard_scatter_kernel",
            "if (W) { rank_mask_kernel",
            "const uint64_t n = std::min(bytes, kRoundCap);",
            "uint64_t sharded_rank_max_worlds() { return (kPiece / kBins) * (kCap + 1ull) - 1; }"):
        assert squash(text) in S, text
    sh = S[S.index("cudaError_topen_window("):]  # the sharded host code: one launch counted per kernel or pair
    assert sh.count("*launches+=1;") == 5 and sh.count("*launches+=2;") == 3
    assert "constexpruint32_tkPiece=0x80000000u;" in S and MAX_WORLDS == 1_073_872_895
    abi = squash(open(os.path.join(CSRC, "sixdof_abi.cu")).read())
    assert squash("if ((uint64_t)n_ranks * 4 >= sharded_rank_round_bytes())") in abi
    # kMaxSliceTasks cannot be reached: a call has at most 1024 groups and 25 planes
    hdr = open(os.path.join(os.path.dirname(CSRC), "..", "include", "b200_sixdof.h")).read()
    groups = int(re.search(r"#define B200_MAX_WORLD_GROUPS (\d+)u", hdr).group(1))
    outcomes = int(re.search(r"#define B200_MAX_OUTCOMES (\d+)u", hdr).group(1))
    assert groups * outcomes == 25_600 < MAX_SLICE_TASKS


def test_restatement_on_hand_cases():
    assert window_places(1) == window_places(2) == 4_186_111 and window_places(3) == (1 << 23) // 3 - 1
    assert window_places(1 << 22) == 1 and window_places((1 << 22) + 1) == 1 and window_places(MAX_RANKS) == 1
    assert window_places((1 << 22) + 1, "w_without_max") == 0 and rounds_of(ROUND_CAP + 4) == [ROUND_CAP, 4]
    # a task of 9000 uniform worlds: one level at shift 50; a constant one: a run at shift 0 after five levels
    v = np.random.default_rng(1).uniform(1.0, 2.0, 9000)
    P, r = task_plan(rank_key(v))
    assert P["ranges"][1] == 1 and sum(map(bool, P["ranges"])) == 1 and same(r, scipy.stats.rankdata(v))
    P, r = task_plan(rank_key(np.full(9000, -3.0)))
    assert P["ranges"][1:6] == [1] * 5 and P["runs_at_0"] == [9000] and np.all(r == 4500.5)
    # the sizes of the smallest call
    P = sharded_plan(np.array([[1.0]]), None, [0], Split(1, {0: (0, 1)}))
    assert P["rounds"] == [8, 0] and P["reads"] == 1 and P["launches"] == {0: 5}


def test_sweep_reaches_every_boundary():
    edges, fails = catalogue_outcome()
    assert fails == []


@pytest.mark.parametrize("fault", FAULTS)
def test_each_fault_fails_a_case(fault):
    _, fails = catalogue_outcome(fault)
    assert fails, f"{fault} passes every case"


# --------------------------------------------------------------------------- GPU


def drive(handles, n_ranks, planes, grouped):
    """The rounds of the real handles {rank: ex} in lockstep over n_ranks ranks, the others virtual (all-zero
    partials), the partials summed (u32, wrapping).  Returns (the round sizes, {rank: kernel launches over the
    rounds})."""
    n0 = {r: ex.timings()["kernel_launches"] for r, ex in handles.items()}
    bound = {ex.sharded_ranks_begin(planes, grouped, r, n_ranks) for r, ex in handles.items()}
    assert bound == {ROUND_CAP}
    bufs = {r: np.zeros(ROUND_CAP // 4, np.uint32) for r in handles}
    rounds, n, red = [], 0, None
    while True:
        got = {ex.sharded_ranks_round(red, n, bufs[r]) for r, ex in handles.items()}
        assert len(got) == 1, got  # every rank makes the same rounds
        n = got.pop()
        rounds.append(n)
        if n == 0:
            break
        first, *rest = bufs.values()
        red = first[:n // 4].copy()
        for b in rest:
            red += b[:n // 4]
    return rounds, {r: ex.timings()["kernel_launches"] - n0[r] for r, ex in handles.items()}


def run_case(case, math="exact"):
    name, values, sizes, planes, split, want = case
    P = sharded_plan(values, sizes, planes, split)
    assert P["errors"] == []
    handles = {r: _only_values(np.ascontiguousarray(values[a:b]), math,
                               None if sizes is None else cut_groups(sizes, a, b)) for r, (a, b) in split.real.items()}
    try:
        rounds, launches = drive(handles, split.n_ranks, planes, sizes is not None)
        assert rounds == P["rounds"], (rle(rounds)[:8], rle(P["rounds"])[:8])  # R2
        assert launches == P["launches"], (launches, P["launches"])  # R4
        want_r = ref_ranks(values[:, planes], sizes)
        assert same(P["ranks"], want_r)
        tasks = len(sizes or [0]) * len(planes)
        for r, ex in handles.items():
            a, b = split.real[r]
            got, _ = ex.sharded_ranks_end()
            assert same(got, want_r[a:b]), (name, r)  # R1
            assert round(ex.rank_reads() * tasks) == P["reads"] and ex.rank_reads() == P["reads"] / tasks  # R3
            assert same(ex.outcome_values(), values[a:b])  # R5
        # R1: the rows of one handle holding every world (a real rank that holds them all serves, after its end)
        whole = [ex for r, ex in handles.items() if split.real[r] == (0, values.shape[0])]
        one = whole[0] if whole else handles.setdefault(-1, _only_values(values, math, sizes))
        assert same(one.outcome_group_ranks(planes) if sizes is not None else one.outcome_ranks(planes), want_r)
    finally:
        for ex in handles.values():
            ex.close()
    return rounds


def _case(name):
    return next(c for c in cases() if c[0] == name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c[0] for c in catalogue()])
def test_catalogue(name):
    need_gpu()
    run_case(_case(name))


@pytest.mark.gpu
def test_one_case_in_fast():
    need_gpu()
    run_case(_case("levels"), "fast")


@pytest.mark.gpu
def test_virtual_rank_equals_a_rank_of_incomplete_worlds():
    """A virtual rank 0 in the uneven case: the same rounds and ranks as a real rank 0 whose 3000 worlds are all
    incomplete (fewer than the largest rank's, so w_most is the same)."""
    need_gpu()
    name, values, sizes, planes, split, want = _case("uneven")
    real = run_case(_case("uneven"))
    virt = Split(split.n_ranks, {r: s for r, s in split.real.items() if r != 0})
    P = sharded_plan(values, sizes, planes, virt)
    assert P["rounds"] == real
    handles = {r: _only_values(np.ascontiguousarray(values[a:b]), "exact", cut_groups(sizes, a, b))
               for r, (a, b) in virt.real.items()}
    rounds, _ = drive(handles, 3, planes, True)
    assert rounds == real
    want = ref_ranks(values[:, planes], sizes)
    for r, ex in handles.items():
        a, b = virt.real[r]
        assert same(ex.sharded_ranks_end()[0], want[a:b])
        ex.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_ranks", [1 << 23, (1 << 23) + 1])
def test_rank_counts_past_the_window_bound_are_refused(n_ranks):
    need_gpu()
    with _only_values(np.array([[2.5], [-1.0]]), "exact") as ex:
        with pytest.raises(_lib.B200Error) as e:
            ex.sharded_ranks_begin([0], False, 0, n_ranks)
        assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        assert same(ex.outcome_ranks([0]), [[2.0], [1.0]])  # the handle stays usable


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [0, 1])
def test_group_size_refusal(extra):
    """One real rank of 3 complete worlds and a virtual rank whose size slot claims the rest of 1,073,872,895 (plus
    `extra`): at the limit the sizes round is accepted and the call goes on to its first histogram (the test then
    discards it with a new begin); one above, the sizes round fails and the handle stays usable."""
    need_gpu()
    with _only_values(np.array([[2.5], [-1.0], [7.0]]), "exact") as ex:
        claim = MAX_WORLDS - 3 + extra
        P = sharded_plan(np.array([[2.5], [-1.0], [7.0]]), None, [0], Split(2, {0: (0, 3)}, {1: [(claim, claim)]}))
        assert P.get("refused", False) == bool(extra)
        ex.sharded_ranks_begin([0], False, 0, 2)
        buf = np.zeros(ROUND_CAP // 4, np.uint32)
        n = ex.sharded_ranks_round(None, 0, buf)
        assert n == 16
        red = buf[:4].copy()
        red[2], red[3] = claim, claim  # rank 1's slots of group 0
        if extra:
            with pytest.raises(_lib.B200Error) as e:
                ex.sharded_ranks_round(red, n, buf)
            assert e.value.code == _lib.ERR_INVALID_ARGUMENT
        else:
            assert ex.sharded_ranks_round(red, n, buf) == KBINS * 4  # level 1: one range
            ex.sharded_ranks_begin([0], False, 0, 1)  # discards the call: no histogram sum is made up
        assert same(ex.outcome_ranks([0]), [[2.0], [1.0], [3.0]])
