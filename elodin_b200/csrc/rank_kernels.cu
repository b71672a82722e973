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
// The order helpers and bitonic_pairs are duplicated from topk_kernels.cu (the top-worlds kernels keep their registers
// and this file's rank key differs at zero).
#include <algorithm>
#include <cfloat>
#include <cooperative_groups.h>
#include <cub/block/block_scan.cuh>

#include "sixdof_internal.h"

namespace b200 {
namespace {

namespace cg = cooperative_groups;

constexpr unsigned kSmallMax = 8192;  // largest group sorted in shared memory by the small routes
constexpr unsigned kWarpMax = 256;    // up to this size a warp sorts a task, eight tasks per block
constexpr unsigned kBins = 1u << 14;  // histogram bins per range and level
constexpr unsigned kBinBits = 14;
constexpr unsigned kCap = 8192;       // a bin of at most this many worlds is a bucket, sorted in shared memory
constexpr int kLevels = 5;            // histogram levels after the count pass
constexpr unsigned kPassThreads = 256;
constexpr unsigned kPlanThreads = 1024;
constexpr uint32_t kNone = 0xffffffffu;      // world state: not complete
constexpr uint32_t kPiece = 0x80000000u;     // world state / bin code: the piece whose base is the low 31 bits
constexpr unsigned long long kRun = 1ull << 63;  // piece word: a tie run (count in bits 32..62, bucket fill in 0..31)

__device__ __forceinline__ unsigned long long order_key(double x)
{
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__device__ __forceinline__ bool finite(double x) { return fabs(x) <= DBL_MAX; }

// the key of a finite value: ascending keys are ascending values, equal keys equal values (-0 == +0)
__device__ __forceinline__ unsigned long long rank_key(double x) { return order_key(x == 0.0 ? 0.0 : x); }

__device__ __forceinline__ bool ck_less(unsigned long long a, uint32_t ai, unsigned long long b, uint32_t bi)
{
    return a < b || (a == b && ai < bi);
}

__device__ __forceinline__ uint32_t pow2_at_least(uint32_t n)
{
    return n <= 1 ? 1 : 1u << (32 - __clz(n - 1));
}

__device__ __forceinline__ uint32_t bit_len(unsigned long long x) { return 64 - __clzll(x); }

// ascending bitonic sort of the pairs (a[], b[])[0, P) (P a power of two) by `team` threads; sync() is the team barrier
template <class Sync>
__device__ void bitonic_pairs(unsigned long long *a, uint32_t *b, uint32_t P, uint32_t tid, uint32_t team, Sync sync)
{
    for (uint32_t k = 2; k <= P; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t t = tid; t < P / 2; t += team) {
                const uint32_t i = 2 * j * (t / j) + t % j, l = i + j;
                const unsigned long long x = a[i], y = a[l];
                const uint32_t xi = b[i], yi = b[l];
                if (ck_less(y, yi, x, xi) == ((i & k) == 0)) {
                    a[i] = y; a[l] = x;
                    b[i] = yi; b[l] = xi;
                }
            }
            sync();
        }
    }
}

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

__device__ inline uint32_t row_of_chunk(const TRow *rows, uint64_t T, uint64_t k)
{
    uint64_t lo = 0, hi = T - 1;
    while (lo < hi) {
        const uint64_t mid = (lo + hi + 1) / 2;
        if (rows[mid].k0 <= k) lo = mid;
        else hi = mid - 1;
    }
    return (uint32_t)lo;
}

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

constexpr uint64_t kScratchCap = 256ull << 20;  // device scratch of a large-group call, unless one task needs more
constexpr uint64_t kHeader = 256;               // the reads counter
constexpr uint64_t kGridCap = 64ull * kNumSMs * 8;

inline uint64_t ranges_of(uint64_t n) { return std::max<uint64_t>(1, n / (kCap + 1)); }

// the world chunk of a task of n worlds in a slice of T tasks: about 8 blocks per SM over the slice, at least 16
// worlds per thread
inline uint32_t chunk_of(uint64_t n, uint64_t T)
{
    const uint64_t want = std::max<uint64_t>(1, 8ull * kNumSMs / std::max<uint64_t>(1, T));
    uint64_t per = (n + want - 1) / want;
    per = std::max<uint64_t>(per, 16ull * kPassThreads);
    return (uint32_t)((per + kPassThreads - 1) / kPassThreads * kPassThreads);
}

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

uint32_t small_routes(const std::vector<WorldGroup> &table, const std::vector<uint32_t> &order, uint32_t *warp)
{
    uint32_t block = 0;
    *warp = 0;
    for (uint32_t g : order) {
        *warp += table[g].n <= kWarpMax;
        block += table[g].n <= kSmallMax;
    }
    return block;
}

} // namespace

uint64_t rank_scratch_bytes(const RankParams &S, const std::vector<WorldGroup> &table, const std::vector<uint32_t> &order)
{
    uint32_t warp;
    const uint32_t block = small_routes(table, order, &warp);
    uint64_t most = 0;
    for (const Slice &s : slices_of(S, table, order, block)) most = std::max(most, s.bytes);
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
    uint32_t warp;
    const uint32_t block = small_routes(table, order, &warp);
    cudaError_t e = cudaSuccess;
    if (warp > 0) {
        rank_warp_kernel<<<(unsigned)std::min((warp * (uint64_t)S.n_p + 7) / 8, kGridCap), 256, 0, s>>>(S, 0, warp);
        *launches += 1;
    }
    if (block > warp) {
        uint64_t n = 0;
        for (uint32_t k = warp; k < block; ++k) n = std::max(n, table[order[k]].n);
        uint32_t P = 1;
        while (P < n) P <<= 1;
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
            const uint32_t Wc = chunk_of(wg.n, sl.T), C = (uint32_t)((wg.n + Wc - 1) / Wc);
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

} // namespace b200
