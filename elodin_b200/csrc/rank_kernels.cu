// Midranks of a Monte-Carlo batch's outcomes: for every task (world group g, selected outcome plane j) the midrank of
// every complete world of the group (include/b200_sixdof.h b200_sixdof_outcome_ranks and _rank_correlation).  A world
// is complete when its n_p selected values are all finite; its midrank in plane j is less + (eq + 1) / 2, less and eq
// the complete worlds of its group with a smaller and an equal value (scipy.stats.rankdata(method="average")).  Values
// compare numerically: rank_key maps -0 to +0 before the totalOrder key, so unlike the quantile and top-worlds kernels
// the two zeros are one value.  A midrank does not depend on the order among tied worlds, so nothing breaks ties: the
// rank planes are a function of the data alone, whatever the route, launch shape, slicing or atomic order.
//
//  - mask pass: one read of every selected plane; a byte per world (complete or not), NaN into every rank plane of an
//    incomplete world.
//  - small groups (n <= kSmallMax, quantile_order's routes): a warp (n <= 256, empty groups included) or a block per
//    task loads the complete (key, world) pairs into shared memory, sorts them (bitonic) and writes each world's
//    midrank from its tie run's bounds (two binary searches of the sorted keys).  One read of the plane, no scratch.
//  - large groups: an MSD bucket pass over the keys:
//      count    per task: complete count and min / max key; every world's state: bin 0 of level 0, or none
//      plan 0   the task whole: a tie run (one key, or one world), a bucket (at most kCap worlds), or a range to refine
//      pass l   per task with a range to refine, one histogram of kBins equal-width bins per range; every world in one
//               moves to its bin, every world whose bin the last plan resolved takes the bin's piece
//      plan l   a block per range: each bin's exclusive prefix is its base `less`; a bin one key wide (or of one world)
//               becomes a tie run, a bin of at most kCap worlds a bucket, a larger one a range of the next level.  A
//               piece (tie run or bucket) is named by its base, unique within the task.
//      scatter  a tie run's worlds take base + (count + 1) / 2; a bucket's go, as (key, world), to the bucket area at
//               [base, base + count)
//      finish   a block per bucket sorts it in shared memory and writes base + its in-bucket midranks
//    Bound: a level over a range of b bits of key leaves bins of b - 14 bits (kBins = 2^14), so after at most 5
//    histogram levels (shifts <= 50, 36, 22, 8, 0) every bin is one key wide: at most 1 + 5 + 1 = 7 reads of the
//    plane on any data, 3 where the first level leaves no bin above kCap worlds, and one read of the bucket area.  A
//    pass reads nothing of a task with nothing to refine.
//    Scratch per task of n worlds: its plan, 2 x R ranges and histograms of kBins u32 (R = max(1, n / (kCap + 1)),
//    the most ranges a level can hold), and per world a state (u32), a piece word (u64), a bucket list slot (u32 per
//    two worlds) and a bucket area slot (u64, u32): about 42 bytes per world.  The large tasks run in slices of at
//    most kScratchCap = 256 MiB, the same launch sequence per slice; a task that alone needs more runs alone.
//
// A world-sharded call (sharded_rank_round, below) runs the same bucket pass over every task, in rounds whose u32 words
// the ranks sum: the plan sees the summed counts, so every rank resolves the same ranges, tie runs and buckets, and the
// buckets' keys travel summed too (each rank writes its own, the others leave those words 0).
#include <algorithm>
#include <cooperative_groups.h>
#include <cub/block/block_scan.cuh>

#include "order_stats.cuh"
#include "sixdof_internal.h"

namespace b200 {
namespace {

namespace cg = cooperative_groups;

constexpr unsigned kBins = 1u << 14;  // histogram bins per range and level
constexpr unsigned kBinBits = 14;
constexpr unsigned kCap = 8192;       // a bin of at most this many worlds is a bucket, sorted in shared memory
constexpr int kLevels = 5;            // histogram levels after the count pass
constexpr unsigned kPassThreads = 256;
constexpr unsigned kPlanThreads = 1024;
constexpr uint32_t kNone = 0xffffffffu;      // world state: not complete
constexpr uint32_t kPiece = 0x80000000u;     // world state / bin code: the piece whose base is the low 31 bits
constexpr unsigned long long kRun = 1ull << 63;  // piece word: a tie run (count in bits 32..62, bucket fill in 0..31)

// the key of a finite value: ascending keys are ascending values, equal keys equal values (-0 == +0)
__device__ __forceinline__ unsigned long long rank_key(double x) { return order_key(x == 0.0 ? 0.0 : x); }

// the midrank, within the sorted keys a[0, n), of position i: its tie run [s, e) found by two binary searches
__device__ __forceinline__ double midrank_at(const unsigned long long *a, uint32_t n, uint32_t i)
{
    const unsigned long long k = a[i];
    uint32_t lo = 0, hi = i;  // first position whose key is k
    while (lo < hi) {
        const uint32_t m = (lo + hi) / 2;
        if (a[m] < k) lo = m + 1;
        else hi = m;
    }
    const uint32_t s = lo;
    lo = i + 1, hi = n;       // first position past the run
    while (lo < hi) {
        const uint32_t m = (lo + hi) / 2;
        if (a[m] <= k) lo = m + 1;
        else hi = m;
    }
    return (double)(s + lo + 1) * 0.5;  // s + (e - s + 1) / 2, a half-integer, exact
}

__device__ __forceinline__ const double *plane_of(const RankParams &S, uint32_t j)
{
    return S.planes + S.plane[j] * S.ld;
}

__device__ __forceinline__ double *rank_plane(const RankParams &S, uint32_t j) { return S.ranks + j * S.ld; }

// ---- mask pass ------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(256) rank_mask_kernel(RankParams S, uint64_t n_worlds)
{
    for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < n_worlds; w += (uint64_t)gridDim.x * blockDim.x) {
        bool ok = true;
        for (uint32_t j = 0; j < S.n_p; ++j) ok = ok && finite(plane_of(S, j)[w]);
        S.mask[w] = ok;
        if (!ok)
            for (uint32_t j = 0; j < S.n_p; ++j) rank_plane(S, j)[w] = __longlong_as_double(0x7ff8000000000000ll);
    }
}

// ---- small groups ---------------------------------------------------------------------------------------------------

// task (group wg, selected plane j): load the complete pairs into (a, b), pad to a power of two with ~0 (no finite
// value's key), sort, write every complete world's midrank
template <class Sync>
__device__ void rank_small(const RankParams &S, const WorldGroup &wg, uint32_t j, unsigned long long *a, uint32_t *b,
                           uint32_t *cnt, uint32_t tid, uint32_t team, Sync sync)
{
    if (tid == 0) *cnt = 0;
    sync();
    const double *p = plane_of(S, j) + wg.o;
    const uint8_t *m = S.mask + wg.o;
    for (uint32_t w = tid; w < wg.n; w += team) {
        if (m[w]) {
            const uint32_t slot = atomicAdd(cnt, 1u);
            a[slot] = rank_key(p[w]);
            b[slot] = w;
        }
    }
    sync();
    const uint32_t n = *cnt, P = pow2_at_least(n);
    for (uint32_t k = n + tid; k < P; k += team) {
        a[k] = ~0ull;
        b[k] = ~0u;
    }
    sync();
    bitonic_pairs(a, b, P, tid, team, sync);
    double *r = rank_plane(S, j) + wg.o;
    for (uint32_t i = tid; i < n; i += team) r[b[i]] = midrank_at(a, n, i);
    sync();
}

// a warp per task, eight tasks per block (groups of at most kWarpMax worlds); task x of the route: group
// order[first + x / n_p], selected plane x % n_p
__global__ void __launch_bounds__(256) rank_warp_kernel(RankParams S, uint32_t first, uint64_t n_groups)
{
    __shared__ unsigned long long keys[8][kWarpMax];
    __shared__ uint32_t idx[8][kWarpMax];
    __shared__ uint32_t cnt[8];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t T = n_groups * S.n_p;
    for (uint64_t x = blockIdx.x * 8ull + wid; x < T; x += gridDim.x * 8ull) {
        const uint32_t g = S.order[first + x / S.n_p], j = (uint32_t)(x % S.n_p);
        rank_small(S, S.groups[g], j, keys[wid], idx[wid], &cnt[wid], lane, 32, []() { __syncwarp(); });
    }
}

// a block per task (groups of kWarpMax < n <= kSmallMax worlds); dynamic shared memory: P (u64, u32) pairs, P the
// power of two at least the route's largest group
__global__ void __launch_bounds__(512) rank_block_kernel(RankParams S, uint32_t first, uint64_t n_groups, uint32_t P)
{
    extern __shared__ unsigned long long keys[];
    __shared__ uint32_t cnt;
    uint32_t *idx = (uint32_t *)(keys + P);
    const uint64_t T = n_groups * S.n_p;
    for (uint64_t x = blockIdx.x; x < T; x += gridDim.x) {
        const uint32_t g = S.order[first + x / S.n_p], j = (uint32_t)(x % S.n_p);
        rank_small(S, S.groups[g], j, keys, idx, &cnt, threadIdx.x, blockDim.x, []() { __syncthreads(); });
    }
}

// ---- large groups ---------------------------------------------------------------------------------------------------

// One task of a slice: group g's worlds [o, o + n) of selected plane j, in C chunks of Wc worlds, k0 = the chunks of
// the slice's tasks before it; R ranges per level; its scratch at `off` bytes into the slice's
struct TRow {
    uint64_t off;
    uint32_t o, n, Wc, C, k0, j, R, pad;
};

// The plan of a task
struct TState {
    unsigned long long kmin, kmax;
    uint32_t n;                 // complete worlds
    uint32_t level;             // the level whose codes the states that name a bin refer to
    uint32_t n_buckets;
    uint32_t nr[kLevels + 2];   // ranges of each level
};

// A range of keys [lo, lo + (kBins << shift)) refined at a level; its worlds' less starts at base
struct Range {
    unsigned long long lo;
    uint32_t shift, base;
};

// The scratch of one task
struct TaskArea {
    TState *st;
    Range *rg0, *rg1;          // [R] per level parity
    uint32_t *hist0, *hist1;   // [R][kBins] per level parity: a level's counts, then its bins' codes
    unsigned long long *piece; // [n]: piece words, at each piece's base
    unsigned long long *bk;    // [n]: bucket area keys, at [base, base + count)
    uint32_t *wst;             // [n]: world states
    uint32_t *blist;           // [n / 2 + 1]: the bases of the buckets
    uint32_t *bi;              // [n]: bucket area worlds
};

__host__ __device__ inline uint64_t align8(uint64_t x) { return (x + 7) / 8 * 8; }

__host__ __device__ inline uint64_t task_bytes(uint64_t n, uint64_t R)
{
    return align8(sizeof(TState)) + 2 * R * sizeof(Range) + 2 * R * kBins * 4ull + n * 16ull + align8(n * 4ull) +
           align8((n / 2 + 1) * 4ull) + align8(n * 4ull);
}

__device__ inline TaskArea area_of(void *base, const TRow &r)
{
    TaskArea A;
    char *p = (char *)base + r.off;
    A.st = (TState *)p;
    p += align8(sizeof(TState));
    A.rg0 = (Range *)p;
    p += r.R * sizeof(Range);
    A.rg1 = (Range *)p;
    p += r.R * sizeof(Range);
    A.piece = (unsigned long long *)p;
    p += r.n * 8ull;
    A.bk = (unsigned long long *)p;
    p += r.n * 8ull;
    A.hist0 = (uint32_t *)p;
    p += r.R * kBins * 4ull;
    A.hist1 = (uint32_t *)p;
    p += r.R * kBins * 4ull;
    A.wst = (uint32_t *)p;
    p += align8(r.n * 4ull);
    A.blist = (uint32_t *)p;
    p += align8((r.n / 2 + 1) * 4ull);
    A.bi = (uint32_t *)p;
    return A;
}

// the ranges and histograms of a level, by its parity
__device__ __forceinline__ Range *rg_of(const TaskArea &A, int level) { return (level & 1) ? A.rg1 : A.rg0; }
__device__ __forceinline__ uint32_t *hist_of(const TaskArea &A, int level) { return (level & 1) ? A.hist1 : A.hist0; }

struct Layout {
    uint64_t T;                 // tasks of the slice
    unsigned long long *reads;  // reads of the planes, summed over the tasks of the call
    const TRow *rows;           // [T]
    void *base;                 // the tasks' areas, at rows[t].off
};

// zero every task's plan and both histograms
__global__ void rank_init_kernel(Layout L, bool first, unsigned long long reads0)
{
    if (first && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *L.reads = reads0;
    const TRow r = L.rows[blockIdx.y];
    const TaskArea A = area_of(L.base, r);
    const uint64_t t0 = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x, step = (uint64_t)gridDim.x * blockDim.x;
    if (t0 == 0) {
        A.st->kmin = ~0ull;
        A.st->kmax = 0;
        A.st->n = 0;
        A.st->level = 0;
        A.st->n_buckets = 0;
        for (int l = 0; l < kLevels + 2; ++l) A.st->nr[l] = 0;
    }
    // hist[0] and hist[1] are adjacent
    for (uint64_t i = t0; i < 2ull * r.R * kBins; i += step) A.hist0[i] = 0;
}

// count: complete count and min / max key per task, and every world's state; a block per chunk
__global__ void __launch_bounds__(kPassThreads) rank_count_kernel(RankParams S, uint64_t K, Layout L)
{
    __shared__ uint32_t sn[kPassThreads / 32];
    __shared__ unsigned long long smn[kPassThreads / 32], smx[kPassThreads / 32];
    const uint32_t t = threadIdx.x;
    for (uint64_t c = blockIdx.x; c < K; c += gridDim.x) {
        const uint32_t ti = row_of_chunk(L.rows, L.T, c);
        const TRow r = L.rows[ti];
        const TaskArea A = area_of(L.base, r);
        const double *p = plane_of(S, r.j) + r.o;
        const uint8_t *m = S.mask + r.o;
        const uint32_t w0 = (uint32_t)(c - r.k0) * r.Wc, w1 = min(w0 + r.Wc, r.n);
        uint32_t n = 0;
        unsigned long long mn = ~0ull, mx = 0;
        for (uint32_t w = w0 + t; w < w1; w += kPassThreads) {
            const bool ok = m[w];
            A.wst[w] = ok ? 0u : kNone;
            if (ok) {
                const unsigned long long s = rank_key(p[w]);
                ++n;
                mn = min(mn, s);
                mx = max(mx, s);
            }
        }
        for (int o = 16; o > 0; o >>= 1) {
            n += __shfl_xor_sync(0xffffffffu, n, o);
            mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if ((t & 31) == 0) {
            sn[t >> 5] = n;
            smn[t >> 5] = mn;
            smx[t >> 5] = mx;
        }
        __syncthreads();
        if (t == 0) {
            for (uint32_t w = 1; w < kPassThreads / 32; ++w) {
                n += sn[w];
                mn = min(mn, smn[w]);
                mx = max(mx, smx[w]);
            }
            if (n) {
                atomicAdd(&A.st->n, n);
                atomicMin(&A.st->kmin, mn);
                atomicMax(&A.st->kmax, mx);
            }
        }
        __syncthreads();
    }
}

// A bin of `count` worlds (count > 0) whose less is `base`, one key wide when shift == 0: its code, after writing its
// piece word or its range of the next level
__device__ __forceinline__ uint32_t resolve_bin(const TaskArea &A, uint32_t count, uint32_t base, unsigned long long lo,
                                                uint32_t shift, uint32_t next_shift, int next)
{
    if (count == 1 || shift == 0 || count <= kCap) {
        const bool run = count == 1 || shift == 0;
        A.piece[base] = ((unsigned long long)count << 32) | (run ? kRun : 0ull);
        if (!run) A.blist[atomicAdd(&A.st->n_buckets, 1u)] = base;
        return kPiece | base;
    }
    const uint32_t r = atomicAdd(&A.st->nr[next], 1u);
    rg_of(A, next)[r] = Range{lo, next_shift, base};
    return r;
}

__device__ __forceinline__ uint32_t level_shift(unsigned long long span)
{
    const uint32_t len = bit_len(span);
    return len > kBinBits ? len - kBinBits : 0;
}

// plan 0: one thread per task; the task whole is bin 0 of level 0, its code in hist[0][0]
__global__ void rank_plan0_kernel(Layout L)
{
    const uint64_t ti = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (ti >= L.T) return;
    const TRow r = L.rows[ti];
    const TaskArea A = area_of(L.base, r);
    const TState &s = *A.st;
    atomicAdd(L.reads, 1ull);  // the count pass
    if (s.n == 0) return;
    atomicAdd(L.reads, 1ull);  // the scatter
    const uint32_t shift = s.kmin == s.kmax ? 0 : 1 + level_shift(s.kmax - s.kmin);  // > 0: more than one key
    A.hist0[0] = resolve_bin(A, s.n, 0, s.kmin, shift, shift ? shift - 1 : 0, 1);
}

// pass l >= 1: every world of a task that has ranges at level l leaves its level l - 1 bin: for a range, into its
// level l bin (counted); for a piece, into the piece; a block per chunk, the bins in global memory
__global__ void __launch_bounds__(kPassThreads) rank_pass_kernel(RankParams S, uint64_t K, Layout L, int level)
{
    const uint32_t t = threadIdx.x;
    for (uint64_t c = blockIdx.x; c < K; c += gridDim.x) {
        const uint32_t ti = row_of_chunk(L.rows, L.T, c);
        const TRow r = L.rows[ti];
        const TaskArea A = area_of(L.base, r);
        if (A.st->nr[level] == 0) continue;  // uniform over the block
        if (c == r.k0 && t == 0) atomicAdd(L.reads, 1ull);
        const uint32_t *code = hist_of(A, level - 1);
        uint32_t *hist = hist_of(A, level);
        const Range *rg = rg_of(A, level);
        const double *p = plane_of(S, r.j) + r.o;
        const uint32_t w0 = (uint32_t)(c - r.k0) * r.Wc, w1 = min(w0 + r.Wc, r.n);
        for (uint32_t w = w0 + t; w < w1; w += kPassThreads) {
            const uint32_t st = A.wst[w];
            if (st & kPiece) continue;  // a piece, or not complete
            const uint32_t cd = code[st];
            if (cd & kPiece) {
                A.wst[w] = cd;
                continue;
            }
            const Range R = rg[cd];
            const uint32_t b = cd * kBins + (uint32_t)((rank_key(p[w]) - R.lo) >> R.shift);
            // one atomic per bin among the lanes here: heavy ties put most of a warp in one bin
            const cg::coalesced_group same = cg::labeled_partition(cg::coalesced_threads(), b);
            if (same.thread_rank() == 0) atomicAdd(&hist[b], same.size());
            A.wst[w] = b;
        }
    }
}

// plan l >= 1: block (range x, task y) of a task with ranges at level l clears its range x of the level l - 1 codes
// (the next pass counts there) and, for a range of level l, turns its bins' counts into codes
__global__ void __launch_bounds__(kPlanThreads) rank_plan_kernel(Layout L, int level)
{
    using Scan = cub::BlockScan<uint32_t, kPlanThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    constexpr uint32_t kItems = kBins / kPlanThreads;
    const TRow row = L.rows[blockIdx.y];
    const TaskArea A = area_of(L.base, row);
    TState &s = *A.st;
    const uint32_t nr = s.nr[level], x = blockIdx.x, t = threadIdx.x;
    if (nr == 0) return;  // the task is done: its codes stay for the scatter
    if (x == 0 && t == 0) s.level = level;
    if (x < (level == 1 ? 1u : s.nr[level - 1])) {  // level 0 is one range (of one bin)
        uint32_t *old = hist_of(A, level - 1) + (uint64_t)x * kBins;
        for (uint32_t k = t; k < kBins; k += kPlanThreads) old[k] = 0;
    }
    if (x >= nr) return;
    const Range R = rg_of(A, level)[x];
    uint32_t *hist = hist_of(A, level) + (uint64_t)x * kBins;
    uint32_t sum = 0, bins[kItems];
#pragma unroll
    for (uint32_t k = 0; k < kItems; ++k) {
        bins[k] = hist[t * kItems + k];
        sum += bins[k];
    }
    uint32_t base;
    Scan(scan_tmp).ExclusiveSum(sum, base);
    const uint32_t next_shift = R.shift > kBinBits ? R.shift - kBinBits : 0;
#pragma unroll
    for (uint32_t k = 0; k < kItems; ++k) {
        const uint32_t b = t * kItems + k;
        if (bins[k])
            hist[b] = resolve_bin(A, bins[k], R.base + base, R.lo + ((unsigned long long)b << R.shift), R.shift,
                                  next_shift, level + 1);
        base += bins[k];
    }
}

// scatter: every complete world takes its piece: a tie run's midrank, or a slot of its bucket's area
__global__ void __launch_bounds__(kPassThreads) rank_scatter_kernel(RankParams S, uint64_t K, Layout L)
{
    const uint32_t t = threadIdx.x;
    for (uint64_t c = blockIdx.x; c < K; c += gridDim.x) {
        const uint32_t ti = row_of_chunk(L.rows, L.T, c);
        const TRow r = L.rows[ti];
        const TaskArea A = area_of(L.base, r);
        const uint32_t *code = hist_of(A, A.st->level);
        const double *p = plane_of(S, r.j) + r.o;
        double *out = rank_plane(S, r.j) + r.o;
        const uint32_t w0 = (uint32_t)(c - r.k0) * r.Wc, w1 = min(w0 + r.Wc, r.n);
        for (uint32_t w = w0 + t; w < w1; w += kPassThreads) {
            uint32_t st = A.wst[w];
            if (st == kNone) continue;
            if (!(st & kPiece)) st = code[st];
            const uint32_t base = st & ~kPiece;
            const unsigned long long pw = A.piece[base];
            if (pw & kRun) {
                out[w] = (double)base + (double)(((pw >> 32) & 0x7fffffffull) + 1) * 0.5;
                continue;
            }
            const uint32_t slot = (uint32_t)atomicAdd(&A.piece[base], 1ull);
            A.bk[base + slot] = rank_key(p[w]);
            A.bi[base + slot] = w;
        }
    }
}

// finish: block (x, task y) sorts buckets x, x + gridDim.x, .. of the task in shared memory and writes base + the
// in-bucket midranks
__global__ void __launch_bounds__(kPlanThreads) rank_finish_kernel(RankParams S, Layout L)
{
    extern __shared__ unsigned long long keys[];  // kCap keys, then kCap worlds
    uint32_t *idx = (uint32_t *)(keys + kCap);
    const TRow r = L.rows[blockIdx.y];
    const TaskArea A = area_of(L.base, r);
    const uint32_t nb = A.st->n_buckets, t = threadIdx.x;
    double *out = rank_plane(S, r.j) + r.o;
    for (uint32_t x = blockIdx.x; x < nb; x += gridDim.x) {
        const uint32_t base = A.blist[x];
        const uint32_t n = (uint32_t)((A.piece[base] >> 32) & 0x7fffffffull), P = pow2_at_least(n);
        for (uint32_t k = t; k < P; k += blockDim.x) {
            keys[k] = k < n ? A.bk[base + k] : ~0ull;
            idx[k] = k < n ? A.bi[base + k] : ~0u;
        }
        __syncthreads();
        bitonic_pairs(keys, idx, P, t, blockDim.x, []() { __syncthreads(); });
        for (uint32_t i = t; i < n; i += blockDim.x) out[idx[i]] = (double)base + midrank_at(keys, n, i);
        __syncthreads();
    }
}

// correlation: group g's covariance record [n, mean[n_p], M[n_p][n_p]] into [n, rho[n_p][n_p]]
__global__ void rank_corr_kernel(const double *cov, double *out, uint64_t G, uint32_t n_p)
{
    const uint64_t per = (uint64_t)n_p * n_p;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < G * (1 + per);
         i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t g = i / (1 + per), e = i % (1 + per);
        const double *c = cov + g * (1 + n_p + per);
        if (e == 0) {
            out[i] = c[0];
            continue;
        }
        const uint32_t a = (uint32_t)((e - 1) / n_p), b = (uint32_t)((e - 1) % n_p);
        const double *M = c + 1 + n_p;
        const double maa = M[a * n_p + a], mbb = M[b * n_p + b];
        out[i] = c[0] >= 2.0 && maa > 0.0 && mbb > 0.0
                     ? __ddiv_rn(M[a * n_p + b], __dsqrt_rn(__dmul_rn(maa, mbb)))
                     : __longlong_as_double(0x7ff8000000000000ll);
    }
}

// ---- world-sharded calls ----------------------------------------------------------------------------------------------

using TaskState = RankShard::TaskState;
constexpr uint32_t kNoBucket = 0xffffffffu;

// One task of a sharded slice: the rank's worlds [o, o + n) of group g and selected plane j, in C chunks of Wc worlds
// (k0 = the chunks of the slice's tasks before it); R ranges at most per level, from N, the group's complete worlds over
// every rank; lcn of them on this rank; its area at `off` bytes into the slice's
struct SRow {
    uint64_t off;
    uint32_t o, n, Wc, C, k0, j, R, N, lcn, pad;
};

// A piece (tie run or bucket) that holds worlds of this rank.  Only such pieces are kept, so a task keeps at most lcn.
// base, count: its less and its worlds over every rank; a bucket's number b (kNoBucket: a tie run), where its keys
// start in the task's key words (kb) and where this rank's start (ko), its worlds on this rank (lc) and where they start
// in the rank's bucket list (lb), and the slots of the list filled so far
struct Piece {
    uint32_t base, count, b, kb, ko, lc, lb, fill;
};

// The area of one sharded task: the ranges of the two level parities (R each: a range holds more than kCap worlds over
// every rank), then the rank's part: its pieces, its worlds' states and its bucket worlds and their keys.  The level
// histograms live in the slice's pools, sized by the ranges that exist.
struct SArea {
    Range *rg0, *rg1;
    Piece *pc;                  // [lcn]
    uint32_t *wst;              // [n]
    uint32_t *bi;               // [lcn]
    unsigned long long *bkey;   // [lcn]
};

__host__ __device__ inline uint64_t shard_area_bytes(uint64_t R, uint64_t lcn, uint64_t n)
{
    return 2 * R * sizeof(Range) + lcn * sizeof(Piece) + align8(n * 4ull) + align8(lcn * 4ull) + lcn * 8ull;
}

__device__ inline SArea shard_area_of(void *base, const SRow &r)
{
    SArea A;
    char *p = (char *)base + r.off;
    A.rg0 = (Range *)p;
    p += r.R * sizeof(Range);
    A.rg1 = (Range *)p;
    p += r.R * sizeof(Range);
    A.pc = (Piece *)p;
    p += r.lcn * sizeof(Piece);
    A.wst = (uint32_t *)p;
    p += align8(r.n * 4ull);
    A.bi = (uint32_t *)p;
    p += align8(r.lcn * 4ull);
    A.bkey = (unsigned long long *)p;
    return A;
}

__device__ __forceinline__ Range *srg_of(const SArea &A, int level) { return (level & 1) ? A.rg1 : A.rg0; }

struct SLayout {
    uint64_t T;                 // tasks of the slice
    const SRow *rows;           // [T]
    TaskState *st;              // [T]
    const uint64_t *hoff0, *hoff1;  // [T] per level parity: where each task's histograms start in the pool (u32 words)
    const uint64_t *xk;         // [T]: where each task's keys start in the slice's key words
    void *base;                 // the tasks' areas, at rows[t].off
    uint32_t *pool0, *pool1;    // per level parity: the level's histograms, [ranges][kBins] per task; then codes
    uint32_t *x;                // the exchange
    uint32_t rank, n_ranks;
};

__device__ __forceinline__ uint32_t *shist(const SLayout &L, int level, uint64_t t)
{
    // selected, not indexed: an indexed parameter array would be copied to the stack
    return (level & 1) ? L.pool1 + L.hoff1[t] : L.pool0 + L.hoff0[t];
}

// the sizes: the complete worlds and the worlds of every group on this rank, into its slots
// x[(g * n_ranks + rank) * 2 + {0, 1}] (x zeroed)
__global__ void __launch_bounds__(256) shard_size_kernel(RankParams S, uint64_t G, uint32_t *x, uint32_t rank,
                                                         uint32_t n_ranks)
{
    __shared__ uint32_t part[8];
    for (uint64_t g = blockIdx.x; g < G; g += gridDim.x) {
        const WorldGroup wg = S.groups[g];
        uint32_t n = 0;
        for (uint64_t w = threadIdx.x; w < wg.n; w += blockDim.x) n += S.mask[wg.o + w];
        for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = n;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int k = 1; k < 8; ++k) n += part[k];
            x[(g * n_ranks + rank) * 2] = n;
            x[(g * n_ranks + rank) * 2 + 1] = (uint32_t)wg.n;
        }
        __syncthreads();
    }
}

// every world's state: bin 0 of level 0, the task's one piece (a task of at most kCap worlds), or none
__global__ void shard_init_kernel(SLayout L, const uint8_t *mask)
{
    const SRow r = L.rows[blockIdx.y];
    const SArea A = shard_area_of(L.base, r);
    const uint32_t first = r.N <= kCap ? kPiece : 0u;
    for (uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; w < r.n; w += (uint64_t)gridDim.x * blockDim.x)
        A.wst[w] = mask[r.o + w] ? first : kNone;
}

// plan 0: one thread per task; the task whole, over the whole key range (min and max do not add over the ranks), is a
// tie run of one world, a bucket, or the range of level 1
__global__ void shard_plan0_kernel(SLayout L)
{
    const uint64_t ti = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (ti >= L.T) return;
    const SRow r = L.rows[ti];
    const SArea A = shard_area_of(L.base, r);
    TaskState s{};
    s.N = r.N;
    s.lcn = r.lcn;
    if (r.N <= kCap) {
        const bool run = r.N == 1;
        if (r.lcn) {
            A.pc[0] = Piece{0, r.N, run ? kNoBucket : 0u, 0, 0, r.lcn, 0, 0};
            s.n_pieces = 1;
        }
        if (!run) {
            s.n_buckets = 1;
            s.bucket_worlds = r.N;
            s.local_worlds = r.lcn;
        }
    } else {
        A.rg1[0] = Range{0ull, 64 - kBinBits, 0};
        s.nr[1] = 1;
    }
    L.st[ti] = s;
}

// pass l >= 1, as rank_pass_kernel: the rank's worlds of a task with ranges at level l leave their level l - 1 bin (at
// level 1, the task's one range) for a piece or a level l bin, counted in the level's pool
__global__ void __launch_bounds__(kPassThreads) shard_pass_kernel(RankParams S, uint64_t K, SLayout L, int level)
{
    const uint32_t t = threadIdx.x;
    for (uint64_t c = blockIdx.x; c < K; c += gridDim.x) {
        const uint32_t ti = row_of_chunk(L.rows, L.T, c);
        const SRow r = L.rows[ti];
        const SArea A = shard_area_of(L.base, r);
        const uint32_t w0 = (uint32_t)(c - r.k0) * r.Wc, w1 = min(w0 + r.Wc, r.n);
        const TaskState &ts = L.st[ti];
        const uint32_t *code = level > 1 ? shist(L, level - 1, ti) : nullptr;
        if (ts.nr[level] == 0) {  // uniform over the block
            // a task whose last plan was l - 1: its worlds take their pieces now, before the pool of l - 1 is reused
            if (level > 1 && ts.level == (uint32_t)(level - 1))
                for (uint32_t w = w0 + t; w < w1; w += kPassThreads) {
                    const uint32_t st = A.wst[w];
                    if (!(st & kPiece)) A.wst[w] = code[st];
                }
            continue;
        }
        uint32_t *hist = shist(L, level, ti);
        const Range *rg = srg_of(A, level);
        const double *p = plane_of(S, r.j) + r.o;
        for (uint32_t w = w0 + t; w < w1; w += kPassThreads) {
            const uint32_t st = A.wst[w];
            if (st & kPiece) continue;
            const uint32_t cd = code ? code[st] : 0u;
            if (cd & kPiece) {
                A.wst[w] = cd;
                continue;
            }
            const Range R = rg[cd];
            const uint32_t b = cd * kBins + (uint32_t)((rank_key(p[w]) - R.lo) >> R.shift);
            const cg::coalesced_group same = cg::labeled_partition(cg::coalesced_threads(), b);
            if (same.thread_rank() == 0) atomicAdd(&hist[b], same.size());
            A.wst[w] = b;
        }
    }
}

// Per-thread sums of a run of bins, scanned over the block: the less of the bins before it, and the buckets, their
// worlds over every rank and on this one, and the ranges they hold.  Scanned as three primitive words (less | ranges,
// bucket worlds | buckets, local bucket worlds): no half reaches 2^32 over a task of fewer than 2^31 worlds.
struct PlanSum {
    uint32_t less, nb, bw, lw, nr;
};

__device__ __forceinline__ PlanSum plan_add(const PlanSum &a, const PlanSum &b)
{
    return PlanSum{a.less + b.less, a.nb + b.nb, a.bw + b.bw, a.lw + b.lw, a.nr + b.nr};
}

constexpr unsigned kShardPlanThreads = 512;

// plan l >= 1: a block per task with ranges at level l resolves its ranges in order, from the summed counts in the
// exchange (laid out as the pool) and the local ones in the pool, writing the bins' codes over the local counts: every
// rank numbers the next level's ranges and the buckets in the same order, so the ranks' words line up in the next
// exchange.  Only the pieces that hold worlds of this rank are kept.
__global__ void __launch_bounds__(kShardPlanThreads) shard_plan_kernel(SLayout L, int level)
{
    using Scan64 = cub::BlockScan<unsigned long long, kShardPlanThreads>;
    using Scan32 = cub::BlockScan<uint32_t, kShardPlanThreads>;
    __shared__ union {
        typename Scan64::TempStorage s64;
        typename Scan32::TempStorage s32;
    } scan_tmp;
    constexpr uint32_t kItems = kBins / kShardPlanThreads;
    const uint64_t ti = blockIdx.y;
    const SRow row = L.rows[ti];
    const SArea A = shard_area_of(L.base, row);
    TaskState &s = L.st[ti];
    const uint32_t nr = s.nr[level], t = threadIdx.x;
    if (nr == 0) return;  // the task is done: its codes stay for the scatter
    const uint32_t next_level = level + 1;
    PlanSum carry{0, s.n_buckets, s.bucket_worlds, s.local_worlds, 0};
    const uint32_t *sums = L.x + ((level & 1) ? L.hoff1[ti] : L.hoff0[ti]);
    for (uint32_t x = 0; x < nr; ++x) {
        const Range R = srg_of(A, level)[x];
        const uint32_t next_shift = R.shift > kBinBits ? R.shift - kBinBits : 0;
        // the bins are read twice (the second time from cache) rather than held across the scan
        const uint32_t *sum = sums + (uint64_t)x * kBins + t * kItems;
        uint32_t *code = shist(L, level, ti) + (uint64_t)x * kBins + t * kItems;
        PlanSum mine{0, 0, 0, 0, 0};
        for (uint32_t k = 0; k < kItems; ++k) {
            const uint32_t g = sum[k];
            mine.less += g;
            if (g <= 1 || R.shift == 0) continue;
            if (g <= kCap) {
                mine.nb += 1;
                mine.bw += g;
                mine.lw += code[k];
            } else {
                mine.nr += 1;
            }
        }
        unsigned long long a0, a1, t0, t1;
        uint32_t a2, t2;
        Scan64(scan_tmp.s64).ExclusiveSum(mine.less | (unsigned long long)mine.nr << 32, a0, t0);
        __syncthreads();
        Scan64(scan_tmp.s64).ExclusiveSum(mine.bw | (unsigned long long)mine.nb << 32, a1, t1);
        __syncthreads();
        Scan32(scan_tmp.s32).ExclusiveSum(mine.lw, a2, t2);
        const PlanSum total{(uint32_t)t0, (uint32_t)(t1 >> 32), (uint32_t)t1, t2, (uint32_t)(t0 >> 32)};
        PlanSum at{(uint32_t)a0, (uint32_t)(a1 >> 32), (uint32_t)a1, a2, (uint32_t)(a0 >> 32)};
        at = plan_add(carry, at);  // carry.less is 0: less restarts at every range's base
        at.less += R.base;
        for (uint32_t k = 0; k < kItems; ++k) {
            const uint32_t g = sum[k];
            if (g == 0) continue;
            const uint32_t base = at.less, b = t * kItems + k, lc = code[k];
            at.less += g;
            if (g > kCap && R.shift != 0) {
                srg_of(A, next_level)[at.nr] = Range{R.lo + ((unsigned long long)b << R.shift), next_shift, base};
                code[k] = at.nr;
                at.nr += 1;
                continue;
            }
            const bool run = g == 1 || R.shift == 0;
            if (lc) {
                const uint32_t id = atomicAdd(&s.n_pieces, 1u);
                A.pc[id] = run ? Piece{base, g, kNoBucket, 0, 0, lc, 0, 0} : Piece{base, g, at.nb, at.bw, at.bw, lc, at.lw, 0};
                code[k] = kPiece | id;
            }
            if (!run) {
                at.nb += 1;
                at.bw += g;
                at.lw += lc;
            }
        }
        carry = plan_add(carry, total);
        carry.less = 0;
        __syncthreads();  // scan_tmp is reused
    }
    if (t == 0) {
        s.level = level;
        s.n_buckets = carry.nb;
        s.bucket_worlds = carry.bw;
        s.local_worlds = carry.lw;
        s.nr[next_level] = carry.nr;
    }
}

// scatter: every complete world of the rank takes its piece: a tie run's midrank, or its bucket's next slot in the
// rank's bucket list, with its key
__global__ void __launch_bounds__(kPassThreads) shard_scatter_kernel(RankParams S, uint64_t K, SLayout L)
{
    const uint32_t t = threadIdx.x;
    for (uint64_t c = blockIdx.x; c < K; c += gridDim.x) {
        const uint32_t ti = row_of_chunk(L.rows, L.T, c);
        const SRow r = L.rows[ti];
        const SArea A = shard_area_of(L.base, r);
        const uint32_t level = L.st[ti].level;
        const uint32_t *code = level ? shist(L, level, ti) : nullptr;
        const double *p = plane_of(S, r.j) + r.o;
        double *out = rank_plane(S, r.j) + r.o;
        const uint32_t w0 = (uint32_t)(c - r.k0) * r.Wc, w1 = min(w0 + r.Wc, r.n);
        for (uint32_t w = w0 + t; w < w1; w += kPassThreads) {
            uint32_t st = A.wst[w];
            if (st == kNone) continue;
            if (!(st & kPiece)) st = code[st];
            Piece &P = A.pc[st & ~kPiece];
            if (P.b == kNoBucket) {
                out[w] = (double)P.base + (double)(P.count + 1) * 0.5;
                continue;
            }
            const uint32_t slot = atomicAdd(&P.fill, 1u);
            A.bi[P.lb + slot] = w;
            A.bkey[P.lb + slot] = rank_key(p[w]);
        }
    }
}

// is piece P a bucket whose keys start in the window [s0, s1) of the slice's key words (its task's from xk)?
__device__ __forceinline__ bool in_window(const Piece &P, uint64_t xk, uint64_t s0, uint64_t s1)
{
    return P.b != kNoBucket && xk + P.kb >= s0 && xk + P.kb < s1;
}

// the window [s0, s1) of the buckets' keys: mode 0, every bucket's count on this rank into its slot
// x[(its first key - s0) * n_ranks + rank] (x zeroed); mode 1, from the sums, where this rank's keys of the bucket go:
// after those of the ranks before it; mode 2, this rank's keys there, from s0 on (x zeroed)
__global__ void shard_window_kernel(SLayout L, uint64_t s0, uint64_t s1, int mode)
{
    const SArea A = shard_area_of(L.base, L.rows[blockIdx.y]);
    const uint32_t np = L.st[blockIdx.y].n_pieces;
    const uint64_t xk = L.xk[blockIdx.y];
    unsigned long long *keys = (unsigned long long *)L.x;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < np; i += gridDim.x * blockDim.x) {
        Piece &P = A.pc[i];
        if (!in_window(P, xk, s0, s1)) continue;
        const uint64_t slot = (xk + P.kb - s0) * L.n_ranks;
        if (mode == 0) {
            L.x[slot + L.rank] = P.lc;
        } else if (mode == 1) {
            uint32_t off = 0;
            for (uint32_t r = 0; r < L.rank; ++r) off += L.x[slot + r];
            P.ko = P.kb + off;
        } else {
            for (uint32_t k = 0; k < P.lc; ++k) keys[xk + P.ko - s0 + k] = A.bkey[P.lb + k];
        }
    }
}

// the midrank within the sorted keys a[0, n) of key k, which a holds: its tie run [s, e) from two binary searches
__device__ __forceinline__ double midrank_of(const unsigned long long *a, uint32_t n, unsigned long long k)
{
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t m = (lo + hi) / 2;
        if (a[m] < k) lo = m + 1;
        else hi = m;
    }
    const uint32_t s = lo;
    hi = n;
    while (lo < hi) {
        const uint32_t m = (lo + hi) / 2;
        if (a[m] <= k) lo = m + 1;
        else hi = m;
    }
    return (double)(s + lo + 1) * 0.5;
}

// finish of the window [s0, s1): block (x, task y) sorts the task's buckets there that hold worlds of this rank (pieces
// x, x + gridDim.x, ..) from every rank's keys in the summed exchange, and writes base + the in-bucket midrank of each
// of the rank's worlds
__global__ void __launch_bounds__(kPlanThreads) shard_finish_kernel(RankParams S, SLayout L, uint64_t s0, uint64_t s1)
{
    extern __shared__ unsigned long long keys[];  // kCap keys, then kCap slots for bitonic_pairs
    uint32_t *idx = (uint32_t *)(keys + kCap);
    const SRow r = L.rows[blockIdx.y];
    const SArea A = shard_area_of(L.base, r);
    const uint32_t np = L.st[blockIdx.y].n_pieces, t = threadIdx.x;
    const uint64_t xk = L.xk[blockIdx.y];
    const unsigned long long *x = (const unsigned long long *)L.x;
    double *out = rank_plane(S, r.j) + r.o;
    for (uint32_t i = blockIdx.x; i < np; i += gridDim.x) {
        const Piece P = A.pc[i];
        if (!in_window(P, xk, s0, s1)) continue;  // uniform over the block
        const uint32_t n2 = pow2_at_least(P.count);
        for (uint32_t k = t; k < n2; k += blockDim.x) {
            keys[k] = k < P.count ? x[xk + P.kb - s0 + k] : ~0ull;
            idx[k] = k;
        }
        __syncthreads();
        bitonic_pairs(keys, idx, n2, t, blockDim.x, []() { __syncthreads(); });
        for (uint32_t k = t; k < P.lc; k += blockDim.x)
            out[A.bi[P.lb + k]] = (double)P.base + midrank_of(keys, P.count, A.bkey[P.lb + k]);
        __syncthreads();
    }
}

constexpr uint64_t kScratchCap = 256ull << 20;  // device scratch of a large-group call, unless one task needs more
constexpr uint64_t kHeader = 256;               // the reads counter

inline uint64_t ranges_of(uint64_t n) { return std::max<uint64_t>(1, n / (kCap + 1)); }

// The large tasks (large groups of order[block ..] outermost, then the selected planes) cut into slices: each slice
// the longest run of tasks whose rows and areas fit in kScratchCap, at least one task
struct Slice {
    uint64_t t0, T, bytes;
};

std::vector<Slice> slices_of(const RankParams &S, const std::vector<WorldGroup> &table,
                             const std::vector<uint32_t> &order, uint32_t block)
{
    std::vector<Slice> out;
    const uint64_t n_tasks = (order.size() - block) * S.n_p;
    for (uint64_t t = 0; t < n_tasks;) {
        Slice s{t, 0, kHeader};
        while (t < n_tasks) {
            const uint64_t n = table[order[block + t / S.n_p]].n;
            const uint64_t add = sizeof(TRow) + task_bytes(n, ranges_of(n));
            if (s.T > 0 && s.bytes + add > kScratchCap) break;
            s.bytes += add;
            ++s.T;
            ++t;
        }
        out.push_back(s);
    }
    return out;
}

} // namespace

uint64_t rank_scratch_bytes(const RankParams &S, const std::vector<WorldGroup> &table, const std::vector<uint32_t> &order)
{
    uint64_t most = 0;
    for (const Slice &s : slices_of(S, table, order, routes_of(table, order).block)) most = std::max(most, s.bytes);
    return most;
}

cudaError_t launch_ranks(const RankParams &S, uint64_t n_worlds, const std::vector<WorldGroup> &table,
                         const std::vector<uint32_t> &order, void *scratch, int *launches, unsigned long long *reads,
                         cudaStream_t s)
{
    *launches = 0;
    if (n_worlds == 0) return cudaSuccess;
    rank_mask_kernel<<<(unsigned)std::min<uint64_t>((n_worlds + 255) / 256, kGridCap), 256, 0, s>>>(S, n_worlds);
    *launches += 1;
    const Routes rt = routes_of(table, order);
    const uint32_t warp = rt.warp, block = rt.block;
    cudaError_t e = cudaSuccess;
    if (warp > 0) {
        rank_warp_kernel<<<(unsigned)std::min((warp * (uint64_t)S.n_p + 7) / 8, kGridCap), 256, 0, s>>>(S, 0, warp);
        *launches += 1;
    }
    if (block > warp) {
        const uint32_t P = block_keys(table, order, rt);
        const size_t smem = P * 12ull;
        e = cudaFuncSetAttribute(rank_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        rank_block_kernel<<<(unsigned)std::min((block - warp) * (uint64_t)S.n_p, kGridCap), 512, smem, s>>>(S, warp, block - warp, P);
        *launches += 1;
    }
    if (order.size() == block) return cudaGetLastError();
    e = cudaFuncSetAttribute(rank_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kCap * 12));
    if (e != cudaSuccess) return e;
    Layout L;
    L.reads = (unsigned long long *)scratch;
    for (const Slice &sl : slices_of(S, table, order, block)) {
        L.T = sl.T;
        L.rows = (const TRow *)((char *)scratch + kHeader);
        L.base = (char *)scratch;
        std::vector<TRow> rows(sl.T);
        uint64_t K = 0, off = align8(kHeader + sl.T * sizeof(TRow)), Rmax = 1;
        for (uint64_t i = 0; i < sl.T; ++i) {
            const uint64_t t = sl.t0 + i;
            const WorldGroup &wg = table[order[block + t / S.n_p]];
            const uint32_t Wc = chunk_of(wg.n, sl.T, kPassThreads), C = (uint32_t)((wg.n + Wc - 1) / Wc);
            const uint64_t R = ranges_of(wg.n);
            rows[i] = TRow{off, (uint32_t)wg.o, (uint32_t)wg.n, Wc, C, (uint32_t)K, (uint32_t)(t % S.n_p), (uint32_t)R, 0};
            off += task_bytes(wg.n, R);
            K += C;
            Rmax = std::max(Rmax, R);
        }
        // in stream order, into the scratch the previous slice is done with
        e = cudaMemcpyAsync((void *)L.rows, rows.data(), sl.T * sizeof(TRow), cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) return e;
        const unsigned grid = (unsigned)std::min(K, kGridCap);
        const unsigned per_task = (unsigned)std::max<uint64_t>(1, 8ull * kNumSMs / sl.T);
        rank_init_kernel<<<dim3(per_task, (unsigned)sl.T), 256, 0, s>>>(L, sl.t0 == 0, block * (uint64_t)S.n_p);
        rank_count_kernel<<<grid, kPassThreads, 0, s>>>(S, K, L);
        rank_plan0_kernel<<<(unsigned)((sl.T + 127) / 128), 128, 0, s>>>(L);
        for (int level = 1; level <= kLevels; ++level) {
            rank_pass_kernel<<<grid, kPassThreads, 0, s>>>(S, K, L, level);
            rank_plan_kernel<<<dim3((unsigned)Rmax, (unsigned)sl.T), kPlanThreads, 0, s>>>(L, level);
        }
        rank_scatter_kernel<<<grid, kPassThreads, 0, s>>>(S, K, L);
        rank_finish_kernel<<<dim3(per_task, (unsigned)sl.T), kPlanThreads, kCap * 12, s>>>(S, L);
        *launches += 5 + 2 * kLevels;
    }
    e = cudaGetLastError();
    // the reads counter, 8 bytes, lands before the caller's stream synchronise
    if (e == cudaSuccess) e = cudaMemcpyAsync(reads, scratch, sizeof *reads, cudaMemcpyDeviceToHost, s);
    return e;
}

cudaError_t launch_rank_correlation(const double *cov, double *out, uint64_t G, uint32_t n_p, int *launches,
                                    cudaStream_t s)
{
    const uint64_t total = G * (1ull + (uint64_t)n_p * n_p);
    rank_corr_kernel<<<(unsigned)std::min<uint64_t>((total + 255) / 256, kGridCap), 256, 0, s>>>(cov, out, G, n_p);
    *launches = 1;
    return cudaGetLastError();
}

// ---- world-sharded calls ----------------------------------------------------------------------------------------------
// Every (group, plane) task whose group holds a complete world on some rank takes the MSD bucket pass (the small routes
// would see only this rank's worlds), in slices cut alike on every rank, with an exchange before every step that needs
// the other ranks' counts or keys:
//   sizes     once per call: every group's complete worlds and worlds, rank-slotted (G x n_ranks x 2 u32)
//   open      per slice: the world states, then plan 0 from the global size alone
//   hist l    pass l counts the rank's worlds into the level's pool; out: the pool (each task's counts of the level's
//             ranges); in: their sums, then plan l
//   scatter   after the last plan: tie runs' midranks, and the rank's bucket worlds with their keys in its bucket list
//   windows   the buckets in windows of their first key in the slice's key words, so that no exchange passes kRoundCap:
//             offsets  each bucket's count on this rank, rank-slotted: where this rank's keys of the bucket go
//             keys     each rank's keys (u64) at the bucket's place plus its offset, the other ranks leaving those words
//                      0; in: every key of the window's buckets, then the finish
// A step that finds no work skips the exchange.  Every rank plans from the same sums, numbers ranges and buckets in the
// same order and so makes the same exchanges, each of the same size.  The sizes and the histograms are sent in rounds of
// at most kRoundCap bytes.
namespace {

enum : int { kStart = 0, kSizes, kHist, kOffsets, kKeys, kDone };
constexpr uint64_t kRoundCap = 32ull << 20;
constexpr uint64_t kMaxSliceTasks = 65535;  // a slice's tasks are a grid's y extent

// the slice's header: rows, task states, the pools' offsets of the two level parities and the key offsets, then the
// tasks' areas
struct SliceHeader {
    uint64_t rows, st, hoff0, hoff1, xk, areas;
};

SliceHeader slice_header(uint64_t T)
{
    SliceHeader H;
    H.rows = kHeader;
    H.st = align8(H.rows + T * sizeof(SRow));
    H.hoff0 = align8(H.st + T * sizeof(TaskState));
    H.hoff1 = H.hoff0 + T * 8;
    H.xk = H.hoff1 + T * 8;
    H.areas = H.xk + T * 8;
    return H;
}

// a task of at most kCap worlds over every rank is one piece: no ranges
uint64_t shard_ranges(uint64_t N) { return N > kCap ? ranges_of(N) : 0; }

// a task's bytes in a slice, for a rank with lcn complete worlds of n
uint64_t task_bytes_of(uint64_t N, uint64_t lcn, uint64_t n)
{
    return sizeof(SRow) + sizeof(TaskState) + 24 + align8(shard_area_bytes(shard_ranges(N), lcn, n));
}

// the tasks (group << 32 | plane: the groups with complete worlds, in table order, then the selected planes), and the
// slices: each the longest run of tasks that fit in kScratchCap on the rank holding the most of each group (at least
// one task), from the rank-slotted sizes alone, so alike on every rank; Q.slices = their first tasks, then the count
void cut_slices(RankShard &Q)
{
    Q.tasks.clear();
    for (uint32_t g = 0; g < Q.n_global.size(); ++g)
        if (Q.n_global[g])
            for (uint32_t j = 0; j < Q.S.n_p; ++j) Q.tasks.push_back((uint64_t)g << 32 | j);
    Q.slices.clear();
    const auto most = [&](uint64_t t) {
        const uint64_t g = Q.tasks[t] >> 32;
        return task_bytes_of(Q.n_global[g], Q.l_most[g], Q.w_most[g]);
    };
    for (uint64_t t = 0; t < Q.tasks.size();) {
        Q.slices.push_back(t);
        uint64_t bytes = kHeader + most(t);
        for (++t; t < Q.tasks.size(); ++t) {
            if (bytes + most(t) > kScratchCap || t - Q.slices.back() == kMaxSliceTasks) break;
            bytes += most(t);
        }
    }
    Q.slices.push_back(Q.tasks.size());
}

// the rows of slice k (their areas: this rank's) and the slice's bytes of scratch
std::vector<SRow> slice_rows(const RankShard &Q, uint64_t k, uint64_t *bytes)
{
    const uint64_t t0 = Q.slices[k], T = Q.slices[k + 1] - t0;
    std::vector<SRow> rows(T);
    uint64_t off = slice_header(T).areas, K = 0;
    for (uint64_t i = 0; i < T; ++i) {
        const uint32_t g = (uint32_t)(Q.tasks[t0 + i] >> 32), j = (uint32_t)Q.tasks[t0 + i];
        const WorldGroup &wg = Q.table[g];
        const uint64_t N = Q.n_global[g], R = shard_ranges(N), lcn = Q.n_local[g];
        const uint32_t Wc = chunk_of(wg.n, T, kPassThreads), C = (uint32_t)((wg.n + Wc - 1) / Wc);
        rows[i] = SRow{off, (uint32_t)wg.o, (uint32_t)wg.n, Wc, C, (uint32_t)K, j, (uint32_t)R, (uint32_t)N,
                       (uint32_t)lcn, 0};
        off += align8(shard_area_bytes(R, lcn, wg.n));
        K += C;
    }
    *bytes = off;
    return rows;
}

struct SliceRun {
    SLayout L;
    uint64_t K;           // chunks of the rank's worlds
    unsigned grid, per_task;
    std::vector<SRow> rows;
};

SliceRun slice_run(const RankShard &Q)
{
    SliceRun r;
    uint64_t bytes = 0;
    r.rows = slice_rows(Q, Q.slice, &bytes);
    const uint64_t T = r.rows.size();
    const SliceHeader H = slice_header(T);
    char *base = (char *)Q.area;
    r.L = SLayout{T, (const SRow *)(base + H.rows), (TaskState *)(base + H.st),
                  (const uint64_t *)(base + H.hoff0), (const uint64_t *)(base + H.hoff1),
                  (const uint64_t *)(base + H.xk), base, Q.pool[0], Q.pool[1], Q.x, Q.rank, Q.n_ranks};
    r.K = 0;
    for (const SRow &row : r.rows) r.K += row.C;
    r.grid = (unsigned)std::min(r.K, kGridCap);
    r.per_task = (unsigned)std::max<uint64_t>(1, 8ull * kNumSMs / T);
    return r;
}

// a grow-only buffer of at least `need` bytes, once the stream is done with the old one
cudaError_t grow(void **p, uint64_t *have, uint64_t need, cudaStream_t s)
{
    if (*have >= need) return cudaSuccess;
    CUDA_TRY(cudaStreamSynchronize(s));
    if (*p) CUDA_TRY(cudaFree(*p));
    *p = nullptr;
    *have = 0;
    CUDA_TRY(cudaMalloc(p, need));
    *have = need;
    return cudaSuccess;
}

// offsets packed in task order, words[t] each, into the header's array at `where`; their total
uint64_t set_offsets(const RankShard &Q, uint64_t where, const std::vector<uint64_t> &words, cudaStream_t s,
                     cudaError_t *e)
{
    std::vector<uint64_t> off(words.size());
    uint64_t total = 0;
    for (size_t t = 0; t < words.size(); ++t) {
        off[t] = total;
        total += words[t];
    }
    *e = cudaMemcpyAsync((char *)Q.area + where, off.data(), off.size() * 8, cudaMemcpyHostToDevice, s);
    return total;
}

// start exchange `step` of `bytes` (> 0) whose words the stream is writing into Q.x: its first round
cudaError_t start(RankShard &Q, int step, uint64_t bytes, void *partial, uint64_t *partial_bytes, cudaStream_t s)
{
    Q.step = step;
    Q.xbytes = bytes;
    Q.xpos = 0;
    const uint64_t n = std::min(bytes, kRoundCap);
    CUDA_TRY(cudaMemcpyAsync(partial, Q.x, n, cudaMemcpyDefault, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    *partial_bytes = n;
    return cudaGetLastError();
}

// the slice's task states, after a plan
cudaError_t read_states(RankShard &Q, const SliceRun &r, cudaStream_t s)
{
    Q.st.resize(r.L.T);
    CUDA_TRY(cudaMemcpyAsync(Q.st.data(), r.L.st, r.L.T * sizeof(TaskState), cudaMemcpyDeviceToHost, s));
    return cudaStreamSynchronize(s);
}

// the window of the slice's buckets whose first key is in [s0, s1) (keys <= kCap past s1): its offsets exchange
cudaError_t open_window(RankShard &Q, void *partial, uint64_t *partial_bytes, int *launches, cudaStream_t s)
{
    const uint64_t s0 = Q.window * Q.wkeys, s1 = std::min(s0 + Q.wkeys, Q.keys);
    const uint64_t bytes = (s1 - s0) * Q.n_ranks * 4;
    // room for the keys exchange too: it follows in the same words, without a sync in between
    CUDA_TRY(grow((void **)&Q.x, &Q.x_bytes, std::max(bytes, (std::min(s1 + kCap, Q.keys) - s0) * 8), s));
    SliceRun r = slice_run(Q);
    CUDA_TRY(cudaMemsetAsync(Q.x, 0, bytes, s));
    shard_window_kernel<<<dim3(r.per_task, (unsigned)r.L.T), 256, 0, s>>>(r.L, s0, s1, 0);
    *launches += 1;
    return start(Q, kOffsets, bytes, partial, partial_bytes, s);
}

// after plan `level` of the slice: the next level's histogram exchange, or the scatter and the windows of the buckets,
// or the slice's end (Q.step = kDone)
cudaError_t after_plan(RankShard &Q, int level, void *partial, uint64_t *partial_bytes, int *launches, cudaStream_t s)
{
    SliceRun r = slice_run(Q);
    CUDA_TRY(read_states(Q, r, s));
    const uint64_t T = r.L.T;
    const SliceHeader H = slice_header(T);
    std::vector<uint64_t> words(T);
    uint64_t refine = 0, keys = 0;
    for (uint64_t t = 0; t < T; ++t) {
        refine += Q.st[t].nr[level + 1] > 0;
        keys += Q.st[t].bucket_worlds;
    }
    cudaError_t e = cudaSuccess;
    if (refine && level < kLevels) {
        const int next = level + 1, p = next & 1;
        for (uint64_t t = 0; t < T; ++t) words[t] = (uint64_t)Q.st[t].nr[next] * kBins;
        const uint64_t total = set_offsets(Q, p ? H.hoff1 : H.hoff0, words, s, &e);
        CUDA_TRY(e);
        CUDA_TRY(grow((void **)&Q.pool[p], &Q.pool_bytes[p], total * 4, s));
        CUDA_TRY(grow((void **)&Q.x, &Q.x_bytes, total * 4, s));
        r = slice_run(Q);
        CUDA_TRY(cudaMemsetAsync(Q.pool[p], 0, total * 4, s));
        Q.reads += refine;
        if (r.grid) {
            shard_pass_kernel<<<r.grid, kPassThreads, 0, s>>>(Q.S, r.K, r.L, next);
            *launches += 1;
        }
        CUDA_TRY(cudaMemcpyAsync(Q.x, Q.pool[p], total * 4, cudaMemcpyDeviceToDevice, s));
        Q.level = next;
        return start(Q, kHist, total * 4, partial, partial_bytes, s);
    }
    Q.reads += T;
    if (r.grid) {
        shard_scatter_kernel<<<r.grid, kPassThreads, 0, s>>>(Q.S, r.K, r.L);
        *launches += 1;
    }
    if (keys) {
        for (uint64_t t = 0; t < T; ++t) words[t] = Q.st[t].bucket_worlds;
        Q.keys = set_offsets(Q, H.xk, words, s, &e);
        CUDA_TRY(e);
        // an offsets window of wkeys * n_ranks u32 and its keys (up to kCap past it) are both one round below the cap;
        // at least one place (the begin refuses n_ranks >= kRoundCap / 4, where even one place reaches the cap), and
        // the max before the - 1 so that a min of 0 cannot wrap
        Q.wkeys = std::max<uint64_t>(2, std::min((kRoundCap - kCap * 8ull) / 8, kRoundCap / (4ull * Q.n_ranks))) - 1;
        Q.window = 0;
        return open_window(Q, partial, partial_bytes, launches, s);
    }
    Q.step = kDone;  // the caller opens the next slice
    return cudaGetLastError();
}

cudaError_t open_slice(RankShard &Q, void *partial, uint64_t *partial_bytes, int *launches, cudaStream_t s)
{
    const SliceRun r = slice_run(Q);
    CUDA_TRY(cudaMemcpyAsync((void *)r.L.rows, r.rows.data(), r.rows.size() * sizeof(SRow), cudaMemcpyHostToDevice, s));
    shard_init_kernel<<<dim3(r.per_task, (unsigned)r.L.T), 256, 0, s>>>(r.L, Q.S.mask);
    shard_plan0_kernel<<<(unsigned)((r.L.T + 127) / 128), 128, 0, s>>>(r.L);
    *launches += 2;
    return after_plan(Q, 0, partial, partial_bytes, launches, s);
}

} // namespace

uint64_t sharded_rank_round_bytes() { return kRoundCap; }

// a world state names a bin of its task's ranges below the piece flag: R * kBins < 2^31
uint64_t sharded_rank_max_worlds() { return (kPiece / kBins) * (kCap + 1ull) - 1; }

void rank_shard_free(RankShard &Q)
{
    for (void *p : {Q.area, (void *)Q.x, (void *)Q.pool[0], (void *)Q.pool[1]})
        if (p) cudaFree(p);
    Q.area = nullptr;
    Q.x = Q.pool[0] = Q.pool[1] = nullptr;
    Q.area_bytes = Q.x_bytes = Q.pool_bytes[0] = Q.pool_bytes[1] = 0;
}

cudaError_t sharded_rank_round(RankShard &Q, const void *reduced, void *partial, uint64_t *partial_bytes, int *launches,
                               cudaStream_t s)
{
    *partial_bytes = 0;
    *launches = 0;
    const uint64_t G = Q.table.size();
    if (Q.step == kStart) {  // the completeness mask, then the sizes
        const uint64_t bytes = G * Q.n_ranks * 8;
        CUDA_TRY(grow((void **)&Q.x, &Q.x_bytes, bytes, s));
        CUDA_TRY(cudaMemsetAsync(Q.x, 0, bytes, s));
        uint64_t W = 0;
        for (const WorldGroup &wg : Q.table) W = std::max(W, wg.o + wg.n);
        if (W) {
            rank_mask_kernel<<<(unsigned)std::min<uint64_t>((W + 255) / 256, kGridCap), 256, 0, s>>>(Q.S, W);
            shard_size_kernel<<<(unsigned)std::min<uint64_t>(G, kGridCap), 256, 0, s>>>(Q.S, G, Q.x, Q.rank, Q.n_ranks);
            *launches += 2;
        }
        return start(Q, kSizes, bytes, partial, partial_bytes, s);
    }
    if (Q.step == kDone) return cudaSuccess;
    // the sums of the round last sent
    const uint64_t n = std::min(Q.xbytes - Q.xpos, kRoundCap);
    CUDA_TRY(cudaMemcpyAsync((char *)Q.x + Q.xpos, reduced, n, cudaMemcpyDefault, s));
    Q.xpos += n;
    if (Q.xpos < Q.xbytes) {  // the exchange's next round
        const uint64_t m = std::min(Q.xbytes - Q.xpos, kRoundCap);
        CUDA_TRY(cudaMemcpyAsync(partial, (char *)Q.x + Q.xpos, m, cudaMemcpyDefault, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        *partial_bytes = m;
        return cudaGetLastError();
    }
    if (Q.step == kSizes) {
        std::vector<uint32_t> words(G * Q.n_ranks * 2);
        CUDA_TRY(cudaMemcpyAsync(words.data(), Q.x, words.size() * 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        Q.n_global.assign(G, 0);
        Q.n_local.assign(G, 0);
        Q.l_most.assign(G, 0);
        Q.w_most.assign(G, 0);
        for (uint64_t g = 0; g < G; ++g) {
            for (uint32_t k = 0; k < Q.n_ranks; ++k) {
                const uint32_t *w = &words[(g * Q.n_ranks + k) * 2];
                Q.n_global[g] += w[0];
                Q.l_most[g] = std::max<uint64_t>(Q.l_most[g], w[0]);
                Q.w_most[g] = std::max<uint64_t>(Q.w_most[g], w[1]);
            }
            Q.n_local[g] = words[(g * Q.n_ranks + Q.rank) * 2];
            if (Q.bad_group == ~0ull && Q.n_global[g] > sharded_rank_max_worlds()) Q.bad_group = g;
        }
        if (Q.bad_group != ~0ull) {
            Q.step = kDone;
            return cudaSuccess;
        }
        cut_slices(Q);
        uint64_t most = 0;
        for (Q.slice = 0; Q.slice + 1 < Q.slices.size(); ++Q.slice) {
            uint64_t bytes = 0;
            slice_rows(Q, Q.slice, &bytes);
            most = std::max(most, bytes);
        }
        CUDA_TRY(grow(&Q.area, &Q.area_bytes, std::max<uint64_t>(most, 8), s));
        Q.slice = 0;
        Q.step = kDone;
    } else {
        SliceRun r = slice_run(Q);
        const uint64_t T = r.L.T;
        if (Q.step == kHist) {
            shard_plan_kernel<<<dim3(1, (unsigned)T), kShardPlanThreads, 0, s>>>(r.L, Q.level);
            *launches += 1;
            CUDA_TRY(after_plan(Q, Q.level, partial, partial_bytes, launches, s));
            if (Q.step != kDone) return cudaSuccess;
        } else {
            const uint64_t s0 = Q.window * Q.wkeys, s1 = std::min(s0 + Q.wkeys, Q.keys);
            if (Q.step == kOffsets) {  // the offsets applied, then this rank's keys of the window
                const uint64_t bytes = (std::min(s1 + kCap, Q.keys) - s0) * 8;
                shard_window_kernel<<<dim3(r.per_task, (unsigned)T), 256, 0, s>>>(r.L, s0, s1, 1);
                CUDA_TRY(cudaMemsetAsync(Q.x, 0, bytes, s));
                shard_window_kernel<<<dim3(r.per_task, (unsigned)T), 256, 0, s>>>(r.L, s0, s1, 2);
                *launches += 2;
                return start(Q, kKeys, bytes, partial, partial_bytes, s);
            }
            CUDA_TRY(cudaFuncSetAttribute(shard_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)(kCap * 12)));
            shard_finish_kernel<<<dim3(r.per_task, (unsigned)T), kPlanThreads, kCap * 12, s>>>(Q.S, r.L, s0, s1);
            *launches += 1;
            if (s1 < Q.keys) {
                ++Q.window;
                return open_window(Q, partial, partial_bytes, launches, s);
            }
        }
        ++Q.slice;
    }
    // the slice just ended (or the sizes): open slices until one makes an exchange
    while (Q.slice + 1 < Q.slices.size()) {
        CUDA_TRY(open_slice(Q, partial, partial_bytes, launches, s));
        if (Q.step != kDone) return cudaSuccess;
        ++Q.slice;
    }
    Q.step = kDone;
    CUDA_TRY(cudaStreamSynchronize(s));
    return cudaGetLastError();
}

} // namespace b200
