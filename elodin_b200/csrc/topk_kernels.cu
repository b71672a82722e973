// Worst worlds of a Monte-Carlo batch: for every task (world group g, selected outcome plane p) the first min(k, count)
// worlds of the group whose value is finite, in the order of the IEEE totalOrder key (order_key: -0 < +0), ascending
// or (largest) descending, ties broken by ascending world index (include/b200_sixdof.h b200_sixdof_outcome_top_worlds
// and _group_top_worlds).  A world group is a contiguous range [o, o + n) of the group table (WorldGroup; only o and n
// are read).  Every world is ranked by its composite key (s, i): s = order_key(x), complemented for largest, and i its
// index within the group, so the order is a total order of the data alone and no route, launch shape, slicing or
// atomic order changes a record.
//
// Routes, chosen per group from its size n (route_of in order_stats.cuh; quantile_order lists the groups by route):
//  - small groups (n <= kSmallMax): a warp (n <= 256, empty groups included) or a block per task loads the task's
//    finite (s, i) pairs into shared memory, sorts them (bitonic) and writes the first k.  One read of the plane, one
//    launch per route that has groups, no scratch.
//  - large groups: a radix select of the composite key of rank kk - 1 (kk = min(k, count)), then one gather:
//      pass 0   per task: finite count and min / max of s (integer atomics)
//      plan 0   kk; a task of at most kCap finite worlds goes straight to the gather, the others refine [min s, max s]
//      pass l   per refining task, one histogram of kBins equal-width bins over its range: of s while the range holds
//               more than one value key, of i among the worlds of that one key once it holds one ("heavy ties": dwell
//               row counts, clamped values, saturated ticks)
//      plan l   the range moves to the bin holding rank kk - 1; every bin before it is selected whole (fewer than kk
//               worlds).  A range of at most kCap worlds goes to the gather; a range of one value key that still holds
//               more continues on i.
//      gather   per task, every world before the range to the `below` area (< kk <= 1024 of them) and every world in it
//               to the `range` area (<= kCap)
//      finish   one block per task sorts each area in shared memory and writes the record
//    Bound: a pass over a range of b bits of key leaves at most b - 14 bits (kBins = 2^14), so a range of value keys
//    (b <= 64) holds one key after at most 5 passes (shifts 50, 36, 22, 8, 0) and a range of indices (b <= 32) one
//    world after at most 3 more (shifts 18, 4, 0): kLevels = 8 histogram passes, so at most 1 + 8 + 1 = 10 reads of the
//    plane on any data.  On continuous data the first histogram leaves a bin of a few thousand worlds: 3 reads (count,
//    histogram, gather).  A pass reads nothing of a task that is not refining.
//    Scratch per task: its plan (TState), kBins u32 of histogram, kBelow + kCap (u64, u32) pairs of areas, about 172 KB;
//    the large tasks run in slices of at most kSliceTasks tasks, the same launch sequence per slice, so the scratch
//    stays under kScratchCap = 256 MiB whatever G x p is.
#include <algorithm>
#include <cub/block/block_scan.cuh>

#include "order_stats.cuh"
#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kBins = 1u << 14;  // histogram bins per task and pass
constexpr unsigned kBinBits = 14;
constexpr unsigned kCap = 8192;                      // a range of at most this many worlds is gathered and sorted
constexpr unsigned kBelow = B200_MAX_TOP_WORLDS;     // worlds before the range: fewer than kk <= k
constexpr int kLevels = 8;                           // histogram passes after pass 0
constexpr unsigned kPassThreads = 256;
constexpr unsigned kPlanThreads = 1024;

enum : uint32_t { kDone = 0, kRefine = 1, kGather = 2 };

// the sort key of x: ascending s is the task's order
__device__ __forceinline__ unsigned long long sort_key(double x, int largest)
{
    const unsigned long long k = order_key(x);
    return largest ? ~k : k;
}

// the record of task (g, j): [count, value_0 .. value_{k-1}, world_0 .. world_{k-1}]
__device__ __forceinline__ double *record_of(const TopkParams &S, uint64_t g, uint32_t j)
{
    return S.out + (g * S.n_p + j) * (1ull + 2ull * S.k);
}

// slot l of a record from the sorted pair (s, i) of a world of the group at o, or the empty slot (NaN, -1)
__device__ __forceinline__ void write_slot(const TopkParams &S, double *rec, uint32_t l, bool live, unsigned long long s,
                                           uint32_t i, uint64_t o)
{
    rec[1 + l] = live ? key_value(S.largest ? ~s : s) : __longlong_as_double(0x7ff8000000000000ll);
    rec[1 + S.k + l] = live ? (double)(o + i) : -1.0;
}

__device__ __forceinline__ const double *plane_of(const TopkParams &S, uint32_t j)
{
    return S.planes + S.plane[j] * S.ld;
}

// ---- small groups ---------------------------------------------------------------------------------------------------

// load the finite pairs of task (group wg, selected plane j) into (a, b), pad to a power of two with (~0, ~0) (after
// every finite pair: ~0 is no finite value's key, whichever the direction), sort; returns the finite count
template <class Sync>
__device__ uint32_t load_sort(const TopkParams &S, const WorldGroup &wg, uint32_t j, unsigned long long *a, uint32_t *b,
                              uint32_t *cnt, uint32_t tid, uint32_t team, Sync sync)
{
    if (tid == 0) *cnt = 0;
    sync();
    const double *p = plane_of(S, j) + wg.o;
    for (uint32_t w = tid; w < wg.n; w += team) {
        const double x = p[w];
        if (finite(x)) {
            const uint32_t slot = atomicAdd(cnt, 1u);
            a[slot] = sort_key(x, S.largest);
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
    return n;
}

__device__ __forceinline__ void write_sorted(const TopkParams &S, double *rec, uint32_t n, const unsigned long long *a,
                                             const uint32_t *b, uint64_t o, uint32_t tid, uint32_t team)
{
    const uint32_t kk = min(n, S.k);
    if (tid == 0) rec[0] = (double)n;
    for (uint32_t l = tid; l < S.k; l += team) write_slot(S, rec, l, l < kk, l < kk ? a[l] : 0, l < kk ? b[l] : 0, o);
}

// a warp per task, eight tasks per block (groups of at most kWarpMax worlds); task x of the route: group
// order[first + x / n_p], selected plane x % n_p
__global__ void __launch_bounds__(256) topk_warp_kernel(TopkParams S, uint32_t first, uint64_t n_groups)
{
    __shared__ unsigned long long keys[8][kWarpMax];
    __shared__ uint32_t idx[8][kWarpMax];
    __shared__ uint32_t cnt[8];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t T = n_groups * S.n_p;
    for (uint64_t x = blockIdx.x * 8ull + wid; x < T; x += gridDim.x * 8ull) {
        const uint32_t g = S.order[first + x / S.n_p], j = (uint32_t)(x % S.n_p);
        const WorldGroup wg = S.groups[g];
        const uint32_t n = load_sort(S, wg, j, keys[wid], idx[wid], &cnt[wid], lane, 32, []() { __syncwarp(); });
        write_sorted(S, record_of(S, g, j), n, keys[wid], idx[wid], wg.o, lane, 32);
        __syncwarp();
    }
}

// a block per task (groups of kWarpMax < n <= kSmallMax worlds); dynamic shared memory: P (u64, u32) pairs, P the
// power of two at least the route's largest group
__global__ void __launch_bounds__(512) topk_block_kernel(TopkParams S, uint32_t first, uint64_t n_groups, uint32_t P)
{
    extern __shared__ unsigned long long keys[];
    __shared__ uint32_t cnt;
    uint32_t *idx = (uint32_t *)(keys + P);
    const uint64_t T = n_groups * S.n_p;
    for (uint64_t x = blockIdx.x; x < T; x += gridDim.x) {
        const uint32_t g = S.order[first + x / S.n_p], j = (uint32_t)(x % S.n_p);
        const WorldGroup wg = S.groups[g];
        const uint32_t n = load_sort(S, wg, j, keys, idx, &cnt, threadIdx.x, blockDim.x, []() { __syncthreads(); });
        write_sorted(S, record_of(S, g, j), n, keys, idx, wg.o, threadIdx.x, blockDim.x);
        __syncthreads();
    }
}

// ---- large groups ---------------------------------------------------------------------------------------------------

// One task of a radix slice: group g's worlds [o, o + n) of selected plane j, in C chunks of Wc worlds, k0 = the chunks
// of the slice's tasks before it
struct TRow {
    uint32_t o, n, Wc, C, k0, g, j, pad;
};

// The plan of a task: the composite range [(lo, ilo), (hi, ihi)] that holds rank kk - 1 (phase 0: a range of value
// keys, ilo = 0, ihi = ~0; phase 1: one value key lo = hi and a range of indices), `below` worlds before it
struct TState {
    unsigned long long lo, hi, kmin, kmax;
    uint32_t ilo, ihi;
    uint32_t n, kk;          // finite worlds, min(k, n)
    uint32_t r;              // rank of kk - 1 within the range
    uint32_t count;          // worlds in the range
    uint32_t below;          // worlds before it
    uint32_t state, phase, shift;
    uint32_t fill_below, fill_range;  // the gather's area fills
};

struct Layout {
    uint64_t T;                        // tasks of the slice
    unsigned long long *reads;         // reads of the planes, summed over the tasks of the call
    const TRow *rows;                  // [T]
    TState *st;                        // [T]
    uint32_t *hist;                    // [T][kBins]
    unsigned long long *bk, *rk;       // [T][kBelow], [T][kCap]: the areas' keys
    uint32_t *bi, *ri;                 // and indices
};

// pass 0: finite count and min / max sort key per task; a block per chunk
__global__ void __launch_bounds__(kPassThreads) topk_count_kernel(TopkParams S, uint64_t K, Layout L)
{
    __shared__ uint32_t sn[kPassThreads / 32];
    __shared__ unsigned long long smn[kPassThreads / 32], smx[kPassThreads / 32];
    const uint32_t t = threadIdx.x;
    for (uint64_t c = blockIdx.x; c < K; c += gridDim.x) {
        const uint32_t ti = row_of_chunk(L.rows, L.T, c);
        const TRow r = L.rows[ti];
        const double *p = plane_of(S, r.j) + r.o;
        const uint32_t w0 = (uint32_t)(c - r.k0) * r.Wc, w1 = min(w0 + r.Wc, r.n);
        uint32_t n = 0;
        unsigned long long mn = ~0ull, mx = 0;
        for (uint32_t w = w0 + t; w < w1; w += kPassThreads) {
            const double x = p[w];
            if (finite(x)) {
                const unsigned long long s = sort_key(x, S.largest);
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
                TState &s = L.st[ti];
                atomicAdd(&s.n, n);
                atomicMin(&s.kmin, mn);
                atomicMax(&s.kmax, mx);
            }
        }
        __syncthreads();
    }
}

// pass l >= 1: the histogram of every refining task's range; a block per chunk, the bins in shared memory
__global__ void __launch_bounds__(kPassThreads) topk_pass_kernel(TopkParams S, uint64_t K, Layout L)
{
    extern __shared__ uint32_t sh_hist[];  // kBins
    const uint32_t t = threadIdx.x;
    for (uint64_t c = blockIdx.x; c < K; c += gridDim.x) {
        const uint32_t ti = row_of_chunk(L.rows, L.T, c);
        const TState &s = L.st[ti];
        if (s.state != kRefine) continue;  // uniform over the block
        const TRow r = L.rows[ti];
        const unsigned long long lo = s.lo, hi = s.hi;
        const uint32_t ilo = s.ilo, ihi = s.ihi, shift = s.shift, phase = s.phase;
        const uint32_t nb = (uint32_t)(((phase ? (unsigned long long)(ihi - ilo) : hi - lo) >> shift) + 1);
        for (uint32_t b = t; b < nb; b += kPassThreads) sh_hist[b] = 0;
        __syncthreads();
        const double *p = plane_of(S, r.j) + r.o;
        const uint32_t w0 = (uint32_t)(c - r.k0) * r.Wc, w1 = min(w0 + r.Wc, r.n);
        for (uint32_t w = w0 + t; w < w1; w += kPassThreads) {
            const double x = p[w];
            if (!finite(x)) continue;
            const unsigned long long k = sort_key(x, S.largest);
            if (k < lo || k > hi) continue;
            if (!phase) atomicAdd(&sh_hist[(uint32_t)((k - lo) >> shift)], 1u);
            else if (w >= ilo && w <= ihi) atomicAdd(&sh_hist[(w - ilo) >> shift], 1u);
        }
        __syncthreads();
        uint32_t *hist = L.hist + (uint64_t)ti * kBins;
        for (uint32_t b = t; b < nb; b += kPassThreads)
            if (sh_hist[b]) atomicAdd(&hist[b], sh_hist[b]);
        __syncthreads();
    }
}

// the next pass's reads of a task of state `st` that moved to it in this plan
__device__ __forceinline__ void count_read(const Layout &L, uint32_t st)
{
    if (st != kDone) atomicAdd(L.reads, 1ull);
}

// What the next pass does with a task whose range holds s.count worlds: gather them when they fit, else refine the
// range (on the index among the group's n worlds once it holds one value key) with at most kBins bins
__device__ __forceinline__ void next_pass(TState &s, uint32_t n)
{
    if (s.count <= kCap) {
        s.state = kGather;
        return;
    }
    s.state = kRefine;
    if (!s.phase && s.lo == s.hi) {
        s.phase = 1;
        s.ilo = 0;
        s.ihi = n - 1;
    }
    const uint32_t len = bit_len(s.phase ? (unsigned long long)(s.ihi - s.ilo) : s.hi - s.lo);
    s.shift = len > kBinBits ? len - kBinBits : 0;
}


// Plan after pass `level`: one block per task.  Level 0 starts the task from its count; a later level moves a refining
// range into the bin that holds rank r, counts the bins before it as selected, decides the next pass and clears the
// bins for it.
__global__ void __launch_bounds__(kPlanThreads) topk_plan_kernel(TopkParams S, Layout L, int level)
{
    using Scan = cub::BlockScan<uint32_t, kPlanThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ uint32_t hit_bin, hit_below, hit_count;
    constexpr uint32_t kItems = kBins / kPlanThreads;
    TState &s = L.st[blockIdx.x];
    const uint32_t t = threadIdx.x;
    if (level == 0) {
        if (t == 0) {
            s.kk = min(s.n, S.k);
            s.below = 0;
            s.phase = 0;
            s.ilo = 0;
            s.ihi = ~0u;
            s.count = s.n;
            s.fill_below = s.fill_range = 0;
            s.r = s.kk - 1;
            // every finite world is in the range [(kmin, 0), (kmax, ~0)]; a range that fits is gathered whole
            s.lo = s.n <= kCap ? 0 : s.kmin;
            s.hi = s.n <= kCap ? ~0ull : s.kmax;
            if (s.n == 0) s.state = kDone;
            else next_pass(s, L.rows[blockIdx.x].n);
            atomicAdd(L.reads, 1ull);  // pass 0
            count_read(L, s.state);
        }
        return;
    }
    if (s.state != kRefine) return;  // uniform over the block
    uint32_t *hist = L.hist + (uint64_t)blockIdx.x * kBins;
    const uint32_t r = s.r;
    uint32_t sum = 0, bins[kItems];
#pragma unroll
    for (uint32_t k = 0; k < kItems; ++k) {
        bins[k] = hist[t * kItems + k];
        sum += bins[k];
    }
    uint32_t base;
    Scan(scan_tmp).ExclusiveSum(sum, base);  // worlds of the range in the bins before this thread's
    if (r >= base && r < base + sum) {      // exactly one thread holds rank r; its bins are cleared below, after this
        uint32_t below = base, k = 0;
        while (r >= below + hist[t * kItems + k]) below += hist[t * kItems + k++];
        hit_bin = t * kItems + k;
        hit_below = below;
        hit_count = hist[t * kItems + k];
    }
#pragma unroll
    for (uint32_t k = 0; k < kItems; ++k) hist[t * kItems + k] = 0;  // the next pass adds to zeros
    __syncthreads();
    if (t == 0) {
        const uint32_t b = hit_bin;
        const unsigned long long span = s.shift ? (1ull << s.shift) - 1 : 0;
        if (!s.phase) {
            s.lo += (unsigned long long)b << s.shift;
            s.hi = min(s.hi, s.lo + span);
        } else {
            const unsigned long long ilo = s.ilo + ((unsigned long long)b << s.shift);
            s.ihi = (uint32_t)min((unsigned long long)s.ihi, ilo + span);
            s.ilo = (uint32_t)ilo;
        }
        s.r = r - hit_below;
        s.below += hit_below;
        s.count = hit_count;
        next_pass(s, L.rows[blockIdx.x].n);
        count_read(L, s.state);
    }
}

// gather: every world of a gathering task before its range to the below area, every world in it to the range area; a
// block per chunk
__global__ void __launch_bounds__(kPassThreads) topk_gather_kernel(TopkParams S, uint64_t K, Layout L)
{
    const uint32_t t = threadIdx.x;
    for (uint64_t c = blockIdx.x; c < K; c += gridDim.x) {
        const uint32_t ti = row_of_chunk(L.rows, L.T, c);
        TState &s = L.st[ti];
        if (s.state != kGather) continue;  // uniform over the block
        const TRow r = L.rows[ti];
        const unsigned long long lo = s.lo, hi = s.hi;
        const uint32_t ilo = s.ilo, ihi = s.ihi;
        const double *p = plane_of(S, r.j) + r.o;
        const uint32_t w0 = (uint32_t)(c - r.k0) * r.Wc, w1 = min(w0 + r.Wc, r.n);
        for (uint32_t w = w0 + t; w < w1; w += kPassThreads) {
            const double x = p[w];
            if (!finite(x)) continue;
            const unsigned long long k = sort_key(x, S.largest);
            if (ck_less(k, w, lo, ilo)) {
                const uint32_t slot = atomicAdd(&s.fill_below, 1u);
                L.bk[(uint64_t)ti * kBelow + slot] = k;
                L.bi[(uint64_t)ti * kBelow + slot] = w;
            } else if (!ck_less(hi, ihi, k, w)) {
                const uint32_t slot = atomicAdd(&s.fill_range, 1u);
                L.rk[(uint64_t)ti * kCap + slot] = k;
                L.ri[(uint64_t)ti * kCap + slot] = w;
            }
        }
    }
}

// finish: one block per task sorts its below area (all selected) and its range area (the first kk - below selected)
// in shared memory and writes the record
__global__ void __launch_bounds__(kPlanThreads) topk_finish_kernel(TopkParams S, Layout L)
{
    extern __shared__ unsigned long long keys[];  // kCap keys, then kCap indices
    uint32_t *idx = (uint32_t *)(keys + kCap);
    const TState &s = L.st[blockIdx.x];
    const TRow r = L.rows[blockIdx.x];
    const uint32_t t = threadIdx.x;
    double *rec = record_of(S, r.g, r.j);
    const uint32_t kk = s.kk, nb = s.below;
    if (t == 0) rec[0] = (double)s.n;
    for (uint32_t l = kk + t; l < S.k; l += blockDim.x) write_slot(S, rec, l, false, 0, 0, r.o);
    if (s.state == kDone) return;
    for (int a = 0; a < 2; ++a) {
        const uint32_t n = a ? s.count : nb, P = pow2_at_least(n);
        const unsigned long long *ak = a ? L.rk + (uint64_t)blockIdx.x * kCap : L.bk + (uint64_t)blockIdx.x * kBelow;
        const uint32_t *ai = a ? L.ri + (uint64_t)blockIdx.x * kCap : L.bi + (uint64_t)blockIdx.x * kBelow;
        for (uint32_t k = t; k < P; k += blockDim.x) {
            keys[k] = k < n ? ak[k] : ~0ull;
            idx[k] = k < n ? ai[k] : ~0u;
        }
        __syncthreads();
        bitonic_pairs(keys, idx, P, t, blockDim.x, []() { __syncthreads(); });
        const uint32_t l0 = a ? nb : 0, l1 = a ? kk : nb;  // record slots [l0, l1) from the sorted area
        for (uint32_t l = l0 + t; l < l1; l += blockDim.x) write_slot(S, rec, l, true, keys[l - l0], idx[l - l0], r.o);
        __syncthreads();
    }
}

constexpr uint64_t kScratchCap = 256ull << 20;  // device scratch of a large-group call, whatever G x p is
constexpr uint64_t kTaskBytes = sizeof(TRow) + (sizeof(TState) + 7) / 8 * 8 + kBins * 4ull + (kBelow + kCap) * 12ull;
constexpr uint64_t kSliceTasks = (kScratchCap - 256) / kTaskBytes;  // about 1500 tasks per slice
static_assert(256 + kSliceTasks * kTaskBytes <= kScratchCap, "a slice's scratch must fit in kScratchCap");

// The scratch of a slice of T tasks: a 256-byte header (the reads counter), then per task its row, plan, histogram and
// areas (keys before indices, so every u64 array is 8-byte aligned)
inline Layout layout_of(uint64_t T, void *scratch)
{
    Layout L;
    L.T = T;
    char *p = (char *)scratch;
    L.reads = (unsigned long long *)p;
    p += 256;
    L.rows = (const TRow *)p;
    p += T * sizeof(TRow);
    L.st = (TState *)p;
    p += T * ((sizeof(TState) + 7) / 8 * 8);
    L.bk = (unsigned long long *)p;
    p += T * kBelow * 8ull;
    L.rk = (unsigned long long *)p;
    p += T * kCap * 8ull;
    L.hist = (uint32_t *)p;
    p += T * kBins * 4ull;
    L.bi = (uint32_t *)p;
    p += T * kBelow * 4ull;
    L.ri = (uint32_t *)p;
    return L;
}

// first: the reads counter starts at `reads0`, the reads of the small routes' tasks
__global__ void topk_init_kernel(Layout L, bool first, unsigned long long reads0)
{
    if (first && blockIdx.x == 0 && threadIdx.x == 0) *L.reads = reads0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < L.T; i += (uint64_t)gridDim.x * blockDim.x) {
        TState &s = L.st[i];
        s.kmin = ~0ull;
        s.kmax = 0;
        s.n = 0;
        s.state = kDone;
    }
    // a fresh histogram for pass 1 (each plan clears the bins it read for the next pass)
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < L.T * kBins; i += (uint64_t)gridDim.x * blockDim.x)
        L.hist[i] = 0;
}

} // namespace

uint64_t topk_scratch_bytes(const TopkParams &S, const std::vector<WorldGroup> &table)
{
    uint64_t large = 0;
    for (const WorldGroup &wg : table) large += route_of(wg.n) == kRadixRoute;
    if (large == 0) return 0;
    return 256 + std::min<uint64_t>(kSliceTasks, large * S.n_p) * kTaskBytes;
}

cudaError_t launch_top_worlds(const TopkParams &S, const std::vector<WorldGroup> &table,
                              const std::vector<uint32_t> &order, void *scratch, int *launches,
                              unsigned long long *reads, cudaStream_t s)
{
    *launches = 0;
    const Routes rt = routes_of(table, order);
    const uint32_t warp = rt.warp, block = rt.block;
    cudaError_t e = cudaSuccess;
    if (warp > 0) {
        topk_warp_kernel<<<(unsigned)std::min((warp * (uint64_t)S.n_p + 7) / 8, kGridCap), 256, 0, s>>>(S, 0, warp);
        *launches += 1;
    }
    if (block > warp) {
        const uint32_t P = block_keys(table, order, rt);
        const size_t smem = P * 12ull;
        e = cudaFuncSetAttribute(topk_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        topk_block_kernel<<<(unsigned)std::min((block - warp) * (uint64_t)S.n_p, kGridCap), 512, smem, s>>>(S, warp, block - warp, P);
        *launches += 1;
    }
    const uint64_t large = order.size() - block;
    if (large == 0) return cudaGetLastError();
    e = cudaFuncSetAttribute(topk_pass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kBins * 4));
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(topk_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kCap * 12));
    if (e != cudaSuccess) return e;
    // The same fixed sequence on every slice of the large tasks (large group outermost, then the selected planes)
    const uint64_t n_tasks = large * S.n_p;
    for (uint64_t t0 = 0; t0 < n_tasks; t0 += kSliceTasks) {
        const uint64_t T = std::min<uint64_t>(kSliceTasks, n_tasks - t0);
        const Layout L = layout_of(T, scratch);
        std::vector<TRow> rows(T);
        uint64_t K = 0;
        for (uint64_t i = 0; i < T; ++i) {
            const uint32_t g = order[block + (t0 + i) / S.n_p];
            const WorldGroup &wg = table[g];
            const uint32_t Wc = chunk_of(wg.n, T, kPassThreads), C = (uint32_t)((wg.n + Wc - 1) / Wc);
            rows[i] = TRow{(uint32_t)wg.o, (uint32_t)wg.n, Wc, C, (uint32_t)K, g, (uint32_t)((t0 + i) % S.n_p), 0};
            K += C;
        }
        // in stream order, into the scratch the previous slice is done with
        e = cudaMemcpyAsync((void *)L.rows, rows.data(), T * sizeof(TRow), cudaMemcpyHostToDevice, s);
        if (e != cudaSuccess) return e;
        const unsigned grid = (unsigned)std::min(K, kGridCap);
        topk_init_kernel<<<(unsigned)std::min((T * kBins + 255) / 256, kGridCap), 256, 0, s>>>(L, t0 == 0, block * (uint64_t)S.n_p);
        topk_count_kernel<<<grid, kPassThreads, 0, s>>>(S, K, L);
        topk_plan_kernel<<<(unsigned)T, kPlanThreads, 0, s>>>(S, L, 0);
        for (int level = 1; level <= kLevels; ++level) {
            topk_pass_kernel<<<grid, kPassThreads, kBins * 4, s>>>(S, K, L);
            topk_plan_kernel<<<(unsigned)T, kPlanThreads, 0, s>>>(S, L, level);
        }
        topk_gather_kernel<<<grid, kPassThreads, 0, s>>>(S, K, L);
        topk_finish_kernel<<<(unsigned)T, kPlanThreads, kCap * 12, s>>>(S, L);
        *launches += 5 + 2 * kLevels;
    }
    e = cudaGetLastError();
    // the reads counter, 8 bytes, lands before the caller's stream synchronise
    if (e == cudaSuccess) e = cudaMemcpyAsync(reads, layout_of(0, scratch).reads, sizeof *reads, cudaMemcpyDeviceToHost, s);
    return e;
}

} // namespace b200
