// Ensemble quantiles over the world axis: for every (world group, plane, entity) triple and every level q, numpy's
// default ("linear") quantile of the finite values of the group's worlds (include/b200_sixdof.h
// b200_sixdof_trajectory_quantiles / _state_quantiles and the _group_quantiles entries).  A world group is a contiguous
// world range [o, o + n) of the group table (WorldGroup; only o and n are read here); the ungrouped entries are the
// one-group case [0, n_worlds).  The result is two order statistics and a fixed lerp, so it needs no floating-point
// reduction: it is exact, and independent of the route, the launch shape and the order of any atomic, so a triple has
// the bits of the ungrouped call on a batch of exactly its group's worlds whatever the other groups of the call.
//
// Values are ordered by the IEEE totalOrder key (key(-0) < key(+0); NaN and +-inf are dropped before).  Three routes,
// chosen per world group from its size n alone (route_of in order_stats.cuh; quantile_order lists the groups by route);
// one call can take all three:
//  - small groups (n <= kSmallMax): a warp (n <= 256, empty groups included) or a block per triple loads the triple's
//    finite keys into shared memory, sorts them (bitonic) and reads off the ranks.  One read of the planes, one launch
//    per route that has groups, no scratch; the block route's shared memory is sized by its largest group.
//  - large groups: a radix select on the key with a fixed launch sequence, pass 0 and passes 1..kLevels:
//      pass 0   per group: finite count n and min / max key (integer atomics)
//      plan     every rank a level needs is in [kmin, kmax]
//      pass k   per group, one histogram of kBins bins over the key ranges that still hold a rank too large to finish
//               (each range gets kBins / 2^ceil(log2 ranges) bins, equal-width in key space); a range small enough is
//               instead copied to scratch ("compacted") in the same pass
//      plan     each rank moves to its bin: a range of one key is finished, a range of <= kBucketCap keys is compacted
//               by the next pass, the others are refined by the next pass
//      finish   per group, each compacted range is sorted in shared memory and its ranks read off
//    A range of 2^64 keys takes at most 14 + 6 * 9 = 68 bits of refinement in passes 1..7 (kBins = 2^14 bins for one
//    range, at least 2^9 for up to 32), so every rank is finished after pass kLevels = 7: at most 8 reads of the planes
//    on any data.  On continuous data pass 1 leaves buckets of a few thousand keys, so the planes are read 3 times
//    (count, histogram, compaction).  A pass reads nothing of a group whose ranks are all finished.
//    Scratch per triple: kBins u32 + kGroupCap u64 keys + the plan (QGroup), about 198 KB.  The triples of the large
//    groups form rows (large group, plane), large group outermost; they run in slices of at most kSliceGroups triples
//    (whole rows, or entity ranges of one row when a row has more entities), the same launch sequence per slice, so the
//    scratch stays under kScratchCap = 256 MiB whatever the ring, group or entity count.  Each row of a slice is chunked
//    by pass_shape over its own group's size; a block task finds its row through the slice's row table (QRow, copied
//    to the scratch ahead of the slice's launches) by binary search over the rows' first chunks.
// Counts and keys are integers, so the order in which atomics land changes no result.
#include <algorithm>
#include <cub/block/block_scan.cuh>

#include "order_stats.cuh"
#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kBins = 1u << 14;   // histogram bins per group and pass (64 KB of u32, in shared memory when E = 1)
constexpr unsigned kBinBits = 14;
constexpr unsigned kBucketCap = 8192;  // a range of at most this many keys is compacted and sorted in shared memory
constexpr unsigned kGroupCap = 16384;  // compacted keys per group
constexpr int kLevels = 7;             // histogram passes after pass 0
constexpr unsigned kSlots = 2 * B200_MAX_QUANTILES;
constexpr unsigned kPassThreads = 256;
constexpr unsigned kPlanThreads = 1024;

enum : uint32_t { kDone = 0, kRefine = 1, kCompact = 2, kCompacted = 3, kUnused = 4 };

// one rank a level needs: x_(rank) is the key in [lo, hi] of rank rr among the group's keys in that range
struct QSlot {
    unsigned long long lo, hi;
    uint32_t rr, count, state, owner;  // owner: the first slot of the same range (shares its bins / compaction)
    uint32_t bin0, shift, cofs, fill;  // refine: bins [bin0, bin0 + (hi - lo) >> shift]; compact: area[cofs ..]
};

struct QGroup {
    unsigned long long kmin, kmax;
    uint32_t n, todo, used;         // todo: the next pass has work here; used: compacted keys
    uint32_t n_act, n_refine;       // the next pass's ranges (refine or compact owners): slot[act[0 .. n_act)]
    uint8_t act[kSlots];
    QSlot slot[kSlots];
};

// One row (large world group g, plane i) of a radix slice: the group's worlds [o, o + n) in C chunks of Wc worlds
// (pass_shape), k0 = the chunks of the slice's rows before it
struct QRow {
    uint32_t o, n, Wc, C, k0, g, i, pad;
};

// A slice of the triples the fixed launch sequence runs on: rows [r0, r0 + nr) of the large groups' (group, plane)
// rows x entities [e0, e0 + ne), K chunks over its rows (Cu chunks each where every row has as many, else 0, and a
// task searches the row table); local triple t = (r - r0) * ne + (e - e0).  Slices keep the scratch under kScratchCap
// whatever the ring, group or entity count.
struct Slice {
    uint64_t r0, nr, e0, ne, K, Cu;
};

struct Layout {
    uint64_t G;                   // triples of the slice
    unsigned long long *reads;    // reads of the planes, summed over the triples of the call
    const QRow *rows;             // [nr] the slice's rows
    QGroup *grp;                  // [G]
    uint32_t *hist;               // [G][kBins]
    unsigned long long *area;     // [G][area_stride]: kGroupCap, or kSlots when sharded (right after hist)
    uint64_t area_stride;
    // sharded (a rank's part of a world-sharded call, b200_sixdof_sharded_quantiles_*): pass 0 counts into cnt[G], the
    // plans start from the whole key range and compact only ranges of one key, and every plan adds its groups' todo
    // flags to *todo
    bool sharded;
    uint32_t *cnt;
    uint32_t *todo;
};

__device__ __forceinline__ double *out_of(const QuantileParams &S, uint64_t g, uint64_t i, uint64_t e)
{
    const uint64_t W = S.planes_per_sample;
    return S.out + ((((i / W) * S.n_groups + g) * S.n_entities + e) * W + i % W) * S.n_q;
}

// numpy's linear quantile of the n sorted keys, rank -> key given by `at`
template <class At>
__device__ double quantile_of(uint32_t n, double q, At at)
{
    if (n == 0) return __longlong_as_double(0x7ff8000000000000ll);
    const double h = __dmul_rn((double)(n - 1), q);
    if (h >= (double)(n - 1)) return key_value(at(n - 1));
    const uint32_t i = (uint32_t)floor(h);
    const double t = __dsub_rn(h, (double)i);
    const double a = key_value(at(i)), b = key_value(at(i + 1));
    const double d = __dsub_rn(b, a);
    return t >= 0.5 ? __dsub_rn(b, __dmul_rn(d, __dsub_rn(1.0, t))) : __dadd_rn(a, __dmul_rn(d, t));
}

// ranks (i, i + 1) of level l, or (n - 1, unused) when h >= n - 1
__device__ inline void ranks_of(uint32_t n, double q, uint32_t &r0, uint32_t &r1, bool &two)
{
    const double h = __dmul_rn((double)(n - 1), q);
    two = h < (double)(n - 1);
    r0 = two ? (uint32_t)floor(h) : n - 1;
    r1 = r0 + 1;
}

// ascending bitonic sort of a[0, P) (P a power of two) by `team` threads; sync() is the team barrier
template <class Sync>
__device__ void bitonic(unsigned long long *a, uint32_t P, uint32_t tid, uint32_t team, Sync sync)
{
    for (uint32_t k = 2; k <= P; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t t = tid; t < P / 2; t += team) {
                const uint32_t i = 2 * j * (t / j) + t % j, l = i + j;
                const unsigned long long x = a[i], y = a[l];
                if ((x > y) == ((i & k) == 0)) { a[i] = y; a[l] = x; }
            }
            sync();
        }
    }
}

// ---- small groups ---------------------------------------------------------------------------------------------------

// load the finite keys of triple (world group wg, i, e) into a[], pad to a power of two with ~0 (above every finite
// key), sort
template <class Sync>
__device__ uint32_t load_sort(const QuantileParams &S, const WorldGroup &wg, uint64_t i, uint64_t e,
                              unsigned long long *a, uint32_t *cnt, uint32_t tid, uint32_t team, Sync sync)
{
    if (tid == 0) *cnt = 0;
    sync();
    const double *p = stats_plane(S, i) + wg.o * S.n_entities + e;
    for (uint64_t w = tid; w < wg.n; w += team) {
        const double x = p[w * S.n_entities];
        if (finite(x)) a[atomicAdd(cnt, 1u)] = order_key(x);
    }
    sync();
    const uint32_t n = *cnt, P = pow2_at_least(n);
    for (uint32_t k = n + tid; k < P; k += team) a[k] = ~0ull;
    sync();
    bitonic(a, P, tid, team, sync);
    return n;
}

// Item x of a small route over the world groups order[first .. first + n_groups): triple (group order[first + x / PE],
// plane (x % PE) / E, entity x % E), PE = planes x entities
struct Item {
    uint64_t g, i, e;
    WorldGroup wg;
};

__device__ __forceinline__ Item item_of(const QuantileParams &S, uint32_t first, uint64_t x)
{
    const uint64_t PE = S.n_planes * S.n_entities;
    Item it;
    it.g = S.order[first + x / PE];
    it.i = (x % PE) / S.n_entities;
    it.e = x % S.n_entities;
    it.wg = S.groups[it.g];
    return it;
}

// a warp per triple, eight triples per block (groups of at most kWarpMax worlds)
__global__ void __launch_bounds__(256) quantile_warp_kernel(QuantileParams S, uint32_t first, uint64_t n_groups)
{
    __shared__ unsigned long long keys[8][kWarpMax];
    __shared__ uint32_t cnt[8];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t G = n_groups * S.n_planes * S.n_entities;
    for (uint64_t x = blockIdx.x * 8ull + wid; x < G; x += gridDim.x * 8ull) {
        const Item it = item_of(S, first, x);
        const uint32_t n = load_sort(S, it.wg, it.i, it.e, keys[wid], &cnt[wid], lane, 32, []() { __syncwarp(); });
        double *o = out_of(S, it.g, it.i, it.e);
        for (uint32_t l = lane; l < S.n_q; l += 32)
            o[l] = quantile_of(n, S.q[l], [&](uint32_t r) { return keys[wid][r]; });
        __syncwarp();
    }
}

// a block per triple (groups of kWarpMax < n <= kSmallMax worlds); dynamic shared memory: pow2 of the largest group's
// size in keys
__global__ void __launch_bounds__(512) quantile_block_kernel(QuantileParams S, uint32_t first, uint64_t n_groups)
{
    extern __shared__ unsigned long long keys[];
    __shared__ uint32_t cnt;
    const uint64_t G = n_groups * S.n_planes * S.n_entities;
    for (uint64_t x = blockIdx.x; x < G; x += gridDim.x) {
        const Item it = item_of(S, first, x);
        const uint32_t n = load_sort(S, it.wg, it.i, it.e, keys, &cnt, threadIdx.x, blockDim.x, []() { __syncthreads(); });
        double *o = out_of(S, it.g, it.i, it.e);
        for (uint32_t l = threadIdx.x; l < S.n_q; l += blockDim.x)
            o[l] = quantile_of(n, S.q[l], [&](uint32_t r) { return keys[r]; });
        __syncthreads();
    }
}

// ---- large groups ---------------------------------------------------------------------------------------------------

// Thread mapping of the passes (as in stats_kernels.cu): a task is (row, world chunk, tile of Et entities); thread t
// takes entity t % Et of the tile and every J-th world of the chunk, so a warp reads consecutive doubles.  The chunking
// of a row is pass_shape over its group's size, the entities and the rows of its slice.
struct PassShape {
    uint64_t Et, J, T, Wc, C;
};

inline PassShape pass_shape(uint64_t n_worlds, uint64_t E, uint64_t n_planes)
{
    PassShape s;
    s.Et = E <= kPassThreads ? E : kPassThreads;
    s.J = E <= kPassThreads ? kPassThreads / E : 1;
    s.T = (E + s.Et - 1) / s.Et;
    // about 4 blocks per SM in all, at least 4096 values per thread-lane group (a block's histogram flush is amortised)
    const uint64_t want = std::max<uint64_t>(1, 4ull * kNumSMs / std::max<uint64_t>(1, n_planes * s.T));
    uint64_t per = (n_worlds + want * s.J - 1) / (want * s.J);
    per = std::max<uint64_t>(per, 16);
    s.Wc = per * s.J;
    s.C = (n_worlds + s.Wc - 1) / s.Wc;
    return s;
}

// pass 0: finite count and min / max key per triple
__global__ void __launch_bounds__(kPassThreads) quantile_count_kernel(QuantileParams S, Slice sl, PassShape sp, Layout L)
{
    const uint64_t E = S.n_entities;
    const unsigned t = threadIdx.x, el = t % (unsigned)sp.Et, j = t / (unsigned)sp.Et;
    const uint64_t n_tasks = sl.K * sp.T;
    for (uint64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
        const uint64_t tile = task % sp.T, k = task / sp.T, il = sl.Cu ? k / sl.Cu : row_of_chunk(L.rows, sl.nr, k);
        const QRow r = L.rows[il];
        const uint64_t c = k - r.k0;
        const uint64_t e = tile * sp.Et + el;  // within the slice
        uint32_t n = 0;
        unsigned long long mn = ~0ull, mx = 0;
        const bool live = j < sp.J && e < sl.ne;
        if (live) {
            const double *p = stats_plane(S, r.i) + sl.e0 + e;
            const uint64_t w1 = r.o + min((c + 1) * r.Wc, (uint64_t)r.n);
            for (uint64_t w = r.o + c * r.Wc + j; w < w1; w += sp.J) {
                const double x = p[w * E];
                if (finite(x)) {
                    const unsigned long long k = order_key(x);
                    ++n;
                    mn = min(mn, k);
                    mx = max(mx, k);
                }
            }
        }
        if (sl.ne == 1) {  // one group per block: reduce the warp first
            for (int o = 16; o > 0; o >>= 1) {
                n += __shfl_xor_sync(0xffffffffu, n, o);
                mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
                mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            }
            if ((t & 31) != 0) n = 0;
        }
        if (live && n) {
            QGroup &G = L.grp[il * sl.ne + e];
            atomicAdd(L.sharded ? &L.cnt[il * sl.ne + e] : &G.n, n);
            atomicMin(&G.kmin, mn);
            atomicMax(&G.kmax, mx);
        }
    }
}

// pass k >= 1: histogram of the refined ranges, copy of the compacted ones
__global__ void __launch_bounds__(kPassThreads) quantile_pass_kernel(QuantileParams S, Slice sl, PassShape sp, Layout L)
{
    extern __shared__ uint32_t sh_hist[];  // kBins counters when ne == 1 (one group per block), else unused
    __shared__ unsigned long long sh_lo[kSlots], sh_hi[kSlots];  // ne == 1: the group's active ranges
    __shared__ uint32_t sh_bin0[kSlots], sh_shift[kSlots], sh_slot[kSlots];
    const uint64_t E = S.n_entities;
    const bool shared_hist = sl.ne == 1;
    const unsigned t = threadIdx.x, el = t % (unsigned)sp.Et, j = t / (unsigned)sp.Et;
    const uint64_t n_tasks = sl.K * sp.T;
    for (uint64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
        const uint64_t tile = task % sp.T, k = task / sp.T, il = sl.Cu ? k / sl.Cu : row_of_chunk(L.rows, sl.nr, k);
        const QRow r = L.rows[il];
        const uint64_t c = k - r.k0;
        const uint64_t e = tile * sp.Et + el;  // within the slice
        const bool live = j < sp.J && e < sl.ne;
        const uint64_t g = il * sl.ne + (live ? e : 0);
        QGroup &G = L.grp[g];
        if (shared_hist) {
            if (!G.todo) continue;  // the whole block is this group: uniform
            for (uint32_t b = t; b < kBins; b += blockDim.x) sh_hist[b] = 0;
            if (t < G.n_act) {
                const QSlot &q = G.slot[G.act[t]];
                sh_lo[t] = q.lo;
                sh_hi[t] = q.hi;
                sh_bin0[t] = q.state == kRefine ? q.bin0 : ~0u;  // ~0: compact
                sh_shift[t] = q.shift;
                sh_slot[t] = G.act[t];
            }
            __syncthreads();
        }
        if (live && G.todo) {
            uint32_t *hist = L.hist + g * kBins;
            unsigned long long *area = L.area + g * L.area_stride;
            const double *p = stats_plane(S, r.i) + sl.e0 + e;
            const uint64_t w1 = r.o + min((c + 1) * r.Wc, (uint64_t)r.n);
            const unsigned long long kmin = G.kmin, kmax = G.kmax;
            const uint32_t n_act = G.n_act;
            for (uint64_t w = r.o + c * r.Wc + j; w < w1; w += sp.J) {
                const double x = p[w * E];
                if (!finite(x)) continue;
                const unsigned long long k = order_key(x);
                if (k < kmin || k > kmax) continue;
                for (uint32_t r = 0; r < n_act; ++r) {
                    if (shared_hist) {
                        if (k < sh_lo[r] || k > sh_hi[r]) continue;
                        if (sh_bin0[r] != ~0u) atomicAdd(&sh_hist[sh_bin0[r] + (uint32_t)((k - sh_lo[r]) >> sh_shift[r])], 1u);
                        else area[G.slot[sh_slot[r]].cofs + atomicAdd(&G.slot[sh_slot[r]].fill, 1u)] = k;
                        break;
                    }
                    QSlot &q = G.slot[G.act[r]];
                    if (k < q.lo || k > q.hi) continue;
                    if (q.state == kRefine) atomicAdd(&hist[q.bin0 + (uint32_t)((k - q.lo) >> q.shift)], 1u);
                    else area[q.cofs + atomicAdd(&q.fill, 1u)] = k;
                    break;
                }
            }
        }
        if (shared_hist) {
            __syncthreads();
            uint32_t *hist = L.hist + g * kBins;
            for (uint32_t b = t; b < kBins; b += blockDim.x)
                if (sh_hist[b]) atomicAdd(&hist[b], sh_hist[b]);
            __syncthreads();
        }
    }
}

// Plan after pass `level`: one block per group.  Moves each refined rank into its bin, then (thread 0) groups the ranks
// into ranges and decides what the next pass does with each; clears the histogram for the next pass.
__global__ void __launch_bounds__(kPlanThreads) quantile_plan_kernel(QuantileParams S, Layout L, int level)
{
    using Scan = cub::BlockScan<uint32_t, kPlanThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ bool dirty;  // the histogram holds counts: the pass before this plan refined a range (or fresh scratch)
    extern __shared__ uint32_t bins[];  // kBins: the counts of the range being scanned
    constexpr uint32_t kItems = kBins / kPlanThreads;
    QGroup &G = L.grp[blockIdx.x];
    uint32_t *hist = L.hist + (uint64_t)blockIdx.x * kBins;
    unsigned long long *area = L.area + blockIdx.x * L.area_stride;
    const uint32_t t = threadIdx.x;
    if (t == 0) dirty = level == 0 || (G.todo && G.n_refine);
    if (level == 0) {
        if (t == 0) {
            // sharded: n is the ranks' sum, and min / max do not add, so every rank starts from the whole key range
            if (L.sharded) G.n = L.cnt[blockIdx.x];
            const unsigned long long lo = L.sharded ? 0 : G.kmin, hi = L.sharded ? ~0ull : G.kmax;
            for (uint32_t s = 0; s < kSlots; ++s) {
                QSlot &q = G.slot[s];
                q = QSlot{lo, hi, 0, G.n, kUnused, s, 0, 0, 0, 0};
                if (G.n == 0 || s / 2 >= S.n_q) continue;
                uint32_t r0, r1;
                bool two;
                ranks_of(G.n, S.q[s / 2], r0, r1, two);
                if (s % 2 == 1 && !two) continue;
                q.rr = s % 2 ? r1 : r0;
                q.state = kRefine;
            }
        }
    } else {
        __shared__ QSlot moved[kSlots];  // the new range of each refined rank, applied once every bin is scanned
        __shared__ uint32_t hit[kSlots];
        if (t < kSlots) hit[t] = 0;
        for (uint32_t a = 0; a < kSlots; ++a) {  // each refined range: exclusive scan of its bins, ranks into bins
            const QSlot o = G.slot[a];
            if (o.owner != a || o.state != kRefine) continue;  // uniform over the block
            const uint32_t nb = (uint32_t)((o.hi - o.lo) >> o.shift) + 1;
            uint32_t sum = 0;
            for (uint32_t k = 0; k < kItems; ++k) {
                const uint32_t b = t * kItems + k;
                bins[b] = b < nb ? hist[o.bin0 + b] : 0;
                sum += bins[b];
            }
            uint32_t base;
            Scan(scan_tmp).ExclusiveSum(sum, base);  // keys of the range below this thread's bins
            __syncthreads();
            for (uint32_t s = a; s < kSlots; ++s) {
                const QSlot q = G.slot[s];
                if (q.owner != a || q.state != kRefine || q.rr < base || q.rr >= base + sum) continue;
                uint32_t below = base, k = 0;
                while (q.rr >= below + bins[t * kItems + k]) below += bins[t * kItems + k++];
                const unsigned long long lo = o.lo + ((unsigned long long)(t * kItems + k) << o.shift);
                const unsigned long long span = o.shift ? (1ull << o.shift) - 1 : 0;
                QSlot m = q;
                m.lo = lo;
                m.hi = min(o.hi, lo + span);
                m.count = bins[t * kItems + k];
                m.rr = q.rr - below;
                moved[s] = m;
                hit[s] = 1;
            }
            __syncthreads();
        }
        if (t < kSlots && hit[t]) {
            G.slot[t] = moved[t];
            G.slot[t].state = 5;  // moved: regrouped below
        }
    }
    __syncthreads();
    if (t == 0) {
        const bool last = level == kLevels;
        uint32_t n_refine = 0;
        for (uint32_t s = 0; s < kSlots; ++s) {
            QSlot &q = G.slot[s];
            if (q.state == kCompact && L.sharded) {  // a range of one key: the ranks' summed area words are that key
                q.lo = q.hi = area[G.slot[q.owner].cofs];
                q.state = kDone;
            }
            if (q.state == kCompact) q.state = kCompacted;  // the pass that just ran copied it
            if (q.state != 5 && q.state != kRefine) continue;
            q.state = kRefine;
            q.owner = s;
            for (uint32_t r = 0; r < s; ++r) {
                const QSlot &o = G.slot[r];
                if (o.owner == r && (o.state == kRefine || o.state == kCompact || o.state == kDone) && o.lo == q.lo && o.hi == q.hi) {
                    q.owner = r;
                    q.state = o.state;
                    break;
                }
            }
            if (q.owner != s) continue;
            if (q.lo == q.hi) {
                q.state = kDone;
            } else if (!last && (L.sharded ? q.count == 1 : q.count <= kBucketCap && G.used + q.count <= kGroupCap)) {
                q.state = kCompact;
                q.cofs = G.used;
                q.fill = 0;
                G.used += q.count;
            } else {
                ++n_refine;
            }
        }
        const uint32_t per = kBins / pow2_at_least(n_refine), bits = kBinBits - (31 - __clz(kBins / per));
        uint32_t k = 0, n_act = 0;
        for (uint32_t s = 0; s < kSlots; ++s) {
            QSlot &q = G.slot[s];
            if (q.owner != s) continue;
            if (q.state == kRefine) {
                const uint32_t len = bit_len(q.hi - q.lo);
                q.shift = len > bits ? len - bits : 0;
                q.bin0 = k++ * per;
            }
            if (q.state == kRefine || q.state == kCompact) G.act[n_act++] = (uint8_t)s;
        }
        G.n_act = n_act;
        G.n_refine = n_refine;
        const uint32_t todo = n_act > 0;
        G.todo = todo;
        atomicAdd(L.reads, (unsigned long long)(todo + (level == 0)));  // level 0: pass 0 read the group too
        if (L.sharded && todo) atomicAdd(L.todo, 1u);
    }
    __syncthreads();
    if (dirty)
        for (uint32_t b = t; b < kBins; b += blockDim.x) hist[b] = 0;
    // sharded: the keys read off above are in the slots now; a rank that does not hold the next pass's keys sends zeros
    if (L.sharded && t < kSlots) area[t] = 0;
}

// finish: one block per group sorts each compacted range in shared memory, then writes the group's quantiles
__global__ void __launch_bounds__(kPlanThreads) quantile_finish_kernel(QuantileParams S, Slice sl, Layout L)
{
    extern __shared__ unsigned long long keys[];  // kBucketCap
    __shared__ unsigned long long rank_key[kSlots];
    QGroup &G = L.grp[blockIdx.x];
    const unsigned long long *area = L.area + blockIdx.x * L.area_stride;
    const uint32_t t = threadIdx.x;
    if (t < kSlots) rank_key[t] = G.slot[t].lo;  // a finished range holds one key
    __syncthreads();
    for (uint32_t a = 0; a < kSlots; ++a) {
        const QSlot &o = G.slot[a];
        if (o.owner != a || o.state != kCompacted) continue;
        const uint32_t n = o.count, P = pow2_at_least(n);
        for (uint32_t k = t; k < P; k += blockDim.x) keys[k] = k < n ? area[o.cofs + k] : ~0ull;
        __syncthreads();
        bitonic(keys, P, t, blockDim.x, []() { __syncthreads(); });
        if (t < kSlots && G.slot[t].owner == a) rank_key[t] = keys[G.slot[t].rr];
        __syncthreads();
    }
    const QRow &r = L.rows[blockIdx.x / sl.ne];
    double *out = out_of(S, r.g, r.i, sl.e0 + blockIdx.x % sl.ne);
    for (uint32_t l = t; l < S.n_q; l += blockDim.x) {
        // slot 2l holds rank i (or n - 1), slot 2l + 1 rank i + 1: map the two ranks quantile_of asks for onto them
        uint32_t r0 = 0, r1 = 0;
        bool two = false;
        if (G.n) ranks_of(G.n, S.q[l], r0, r1, two);
        out[l] = quantile_of(G.n, S.q[l], [&](uint32_t r) { return rank_key[2 * l + (r == r0 ? 0 : 1)]; });
    }
}

constexpr uint64_t kScratchCap = 256ull << 20;  // device scratch of a large-group call, whatever the ring holds
constexpr uint64_t kGroupBytes = (sizeof(QGroup) + 7) / 8 * 8 + kBins * 4ull + kGroupCap * 8ull;
constexpr uint64_t kSliceGroups = (kScratchCap - 256) / kGroupBytes;  // about 1350 triples per slice
constexpr uint64_t kRowBytes = kSliceGroups * sizeof(QRow);           // a slice has at most kSliceGroups rows
static_assert(256 + kRowBytes + kSliceGroups * kGroupBytes <= kScratchCap, "a slice's scratch must fit in kScratchCap");

// The scratch of a slice of G triples: a 256-byte header (the reads counter, then the sharded todo counter), the row
// table, then per triple its plan, histogram and compaction area; a sharded slice's areas (kSlots keys: it compacts
// ranges of one key only) follow the histograms directly, so a round's counters and keys are one run of u32 words, and
// its pass 0 counts follow them.
constexpr uint64_t kExchangeBytes = kBins * 4ull + kSlots * 8ull;  // a sharded triple's words of a histogram round
constexpr uint64_t kShardGroupBytes = (sizeof(QGroup) + 7) / 8 * 8 + kExchangeBytes + 4;

inline Layout layout_of(uint64_t G, void *scratch, bool sharded)
{
    Layout L;
    L.G = G;
    char *p = (char *)scratch;
    L.reads = (unsigned long long *)p;
    L.todo = sharded ? (uint32_t *)(p + 8) : nullptr;
    p += 256;
    L.rows = (const QRow *)p;
    p += kRowBytes;
    L.grp = (QGroup *)p;
    p += G * ((sizeof(QGroup) + 7) / 8 * 8);
    L.hist = (uint32_t *)p;
    p += G * kBins * sizeof(uint32_t);
    L.area = (unsigned long long *)p;
    L.area_stride = sharded ? kSlots : kGroupCap;
    p += G * L.area_stride * 8;
    L.sharded = sharded;
    L.cnt = sharded ? (uint32_t *)p : nullptr;
    return L;
}

// first: the reads counter starts at `reads0`, the reads of the small routes' triples
__global__ void quantile_init_kernel(Layout L, bool first, unsigned long long reads0)
{
    if (first && blockIdx.x == 0 && threadIdx.x == 0) *L.reads = reads0;
    for (uint64_t g = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; g < L.G; g += (uint64_t)gridDim.x * blockDim.x) {
        L.grp[g].kmin = ~0ull;
        L.grp[g].kmax = 0;
        L.grp[g].n = 0;
        L.grp[g].todo = 0;
        L.grp[g].used = 0;
        L.grp[g].n_act = 0;
        L.grp[g].n_refine = 0;
        if (L.sharded) L.cnt[g] = 0;
    }
}

// triples per slice along each axis: whole rows while a row's entities fit, else entity ranges of one row
inline Slice slice_shape(uint64_t E)
{
    if (E <= kSliceGroups) return Slice{0, std::max<uint64_t>(1, kSliceGroups / E), 0, E, 0, 0};
    return Slice{0, 1, 0, kSliceGroups, 0, 0};
}

// One slice of the radix sequence over the large groups large[0 .. n_large) of a table (slice_shape; row slices
// outermost, then entity slices): its triples, row table, scratch layout and pass launch shape.
struct SliceRun {
    Slice sl;
    Layout L;
    PassShape sp;
    unsigned grid;
    size_t hist_smem;
    std::vector<QRow> rows;
};

inline uint64_t slices_of(const QuantileParams &S, uint64_t n_large)
{
    const Slice sh = slice_shape(S.n_entities);
    const uint64_t n_rows = n_large * S.n_planes;
    return (n_rows + sh.nr - 1) / sh.nr * ((S.n_entities + sh.ne - 1) / sh.ne);
}

SliceRun slice_run(const QuantileParams &S, const std::vector<WorldGroup> &table, const uint32_t *large,
                   uint64_t n_large, uint64_t k, void *scratch, bool sharded)
{
    const Slice sh = slice_shape(S.n_entities);
    const uint64_t n_rows = n_large * S.n_planes, n_e = (S.n_entities + sh.ne - 1) / sh.ne;
    const uint64_t r0 = k / n_e * sh.nr, e0 = k % n_e * sh.ne;
    SliceRun run;
    Slice &sl = run.sl;
    sl = Slice{r0, std::min(sh.nr, n_rows - r0), e0, std::min(sh.ne, S.n_entities - e0), 0, 0};
    for (uint64_t r = r0; r < r0 + sl.nr; ++r) {
        const uint32_t g = large[r / S.n_planes];
        const WorldGroup &wg = table[g];
        const PassShape sp = pass_shape(wg.n, sl.ne, sl.nr);
        run.rows.push_back(QRow{(uint32_t)wg.o, (uint32_t)wg.n, (uint32_t)sp.Wc, (uint32_t)sp.C, (uint32_t)sl.K, g,
                                (uint32_t)(r % S.n_planes), 0});
        sl.K += sp.C;
        sl.Cu = r == r0 || sl.Cu == sp.C ? sp.C : 0;
    }
    run.L = layout_of(sl.nr * sl.ne, scratch, sharded);
    run.sp = pass_shape(0, sl.ne, sl.nr);  // the tiles (Et, J, T): the slice's entities alone
    run.grid = (unsigned)std::min(sl.K * run.sp.T, kGridCap);
    run.hist_smem = sl.ne == 1 ? kBins * 4ull : 0;
    return run;
}

cudaError_t radix_attributes()
{
    cudaError_t e = cudaFuncSetAttribute(quantile_pass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kBins * 4));
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(quantile_plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kBins * 4));
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(quantile_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kBucketCap * 8));
    return e;
}

// The slice's row table, copied in stream order into the scratch the previous slice is done with, then its init and
// pass 0 (no pass 0 launch when no row of the slice holds a world: a sharded rank's empty groups)
cudaError_t launch_open(const QuantileParams &S, const SliceRun &r, bool first, unsigned long long reads0, cudaStream_t s)
{
    const cudaError_t e = cudaMemcpyAsync((void *)r.L.rows, r.rows.data(), r.rows.size() * sizeof(QRow),
                                          cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return e;
    quantile_init_kernel<<<(unsigned)std::min((r.L.G + 255) / 256, kGridCap), 256, 0, s>>>(r.L, first, reads0);
    if (r.grid) quantile_count_kernel<<<r.grid, kPassThreads, 0, s>>>(S, r.sl, r.sp, r.L);
    return cudaSuccess;
}

void launch_plan(const QuantileParams &S, const SliceRun &r, int level, cudaStream_t s)
{
    quantile_plan_kernel<<<(unsigned)r.L.G, kPlanThreads, kBins * 4, s>>>(S, r.L, level);
}

void launch_pass(const QuantileParams &S, const SliceRun &r, cudaStream_t s)
{
    if (r.grid) quantile_pass_kernel<<<r.grid, kPassThreads, r.hist_smem, s>>>(S, r.sl, r.sp, r.L);
}

void launch_finish(const QuantileParams &S, const SliceRun &r, cudaStream_t s)
{
    quantile_finish_kernel<<<(unsigned)r.L.G, kPlanThreads, kBucketCap * 8, s>>>(S, r.sl, r.L);
}

} // namespace

std::vector<uint32_t> quantile_order(const std::vector<WorldGroup> &table)
{
    std::vector<uint32_t> order;
    for (int route = kWarpRoute; route <= kRadixRoute; ++route)
        for (uint32_t g = 0; g < table.size(); ++g) {
            if (route_of(table[g].n) == route) order.push_back(g);
        }
    return order;
}

uint64_t quantile_scratch_bytes(const QuantileParams &S, const std::vector<WorldGroup> &table)
{
    uint64_t large = 0;
    for (const WorldGroup &wg : table) large += route_of(wg.n) == kRadixRoute;
    if (S.n_planes == 0 || S.n_entities == 0 || large == 0) return 0;
    const Slice sh = slice_shape(S.n_entities);
    return 256 + kRowBytes + std::min(sh.nr, large * S.n_planes) * sh.ne * kGroupBytes;
}

cudaError_t launch_quantiles(const QuantileParams &S, const std::vector<WorldGroup> &table,
                             const std::vector<uint32_t> &order, void *scratch, int *launches,
                             unsigned long long *reads, cudaStream_t s)
{
    *launches = 0;
    if (S.n_planes == 0 || S.n_entities == 0) return cudaSuccess;
    const uint64_t PE = S.n_planes * S.n_entities;
    const Routes rt = routes_of(table, order);
    cudaError_t e = cudaSuccess;
    if (rt.warp > 0) {
        quantile_warp_kernel<<<(unsigned)std::min((rt.warp * PE + 7) / 8, kGridCap), 256, 0, s>>>(S, 0, rt.warp);
        *launches += 1;
    }
    if (rt.block > rt.warp) {
        const size_t smem = block_keys(table, order, rt) * 8ull;
        e = cudaFuncSetAttribute(quantile_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        quantile_block_kernel<<<(unsigned)std::min((rt.block - rt.warp) * PE, kGridCap), 512, smem, s>>>(S, rt.warp,
                                                                                                         rt.block - rt.warp);
        *launches += 1;
    }
    const uint64_t large = order.size() - rt.block;
    if (large == 0) return cudaGetLastError();
    e = radix_attributes();
    if (e != cudaSuccess) return e;
    // The same fixed sequence on every slice (one slice unless the triples need more than kScratchCap of scratch);
    // each plan clears the histograms it leaves for the next pass, so the scratch needs no clearing in between.
    const uint64_t n_slices = slices_of(S, large);
    for (uint64_t k = 0; k < n_slices; ++k) {
        const SliceRun r = slice_run(S, table, order.data() + rt.block, large, k, scratch, false);
        e = launch_open(S, r, k == 0, rt.block * PE, s);
        if (e != cudaSuccess) return e;
        launch_plan(S, r, 0, s);
        *launches += 3;
        for (int level = 1; level <= kLevels; ++level) {
            launch_pass(S, r, s);
            launch_plan(S, r, level, s);
            *launches += 2;
        }
        launch_finish(S, r, s);
        *launches += 1;
    }
    e = cudaGetLastError();
    // the reads counter, 8 bytes, lands before the caller's stream synchronise
    if (e == cudaSuccess) e = cudaMemcpyAsync(reads, layout_of(0, scratch, false).reads, sizeof *reads, cudaMemcpyDeviceToHost, s);
    return e;
}

// ---- world-sharded calls ---------------------------------------------------------------------------------------------
// Every group takes the radix route (the route would follow the global world count, which no rank knows before the count
// round) and every slice runs the launch sequence above with the sharded layout, a round between a pass and its plan:
//   count round   open the slice; out: the pass 0 counts cnt[G]; in: their sums, then plan 0 from the whole key range
//   pass round k  pass k; out: the slice's histograms and compaction keys; in: their sums, then plan k
// A plan whose slice has nothing left to do ends the slice (finish) and opens the next one.  Every rank plans from the
// same sums, so every rank makes the same rounds and ends on the same order statistics: those of the union of the
// worlds.  A range whose global count is 1 is compacted: the one rank that holds its key copies it to the cleared area
// and the others send zeros, so the summed words are the key; larger ranges are refined down to one key.

uint64_t sharded_quantile_scratch_bytes(const QuantileParams &S, uint64_t n_groups)
{
    if (S.n_planes == 0 || S.n_entities == 0 || n_groups == 0) return 0;
    const Slice sh = slice_shape(S.n_entities);
    return (256 + kRowBytes + std::min(sh.nr, n_groups * S.n_planes) * sh.ne * kShardGroupBytes + 255) / 256 * 256;
}

uint64_t sharded_quantile_round_bytes(const QuantileParams &S, uint64_t n_groups)
{
    if (S.n_planes == 0 || S.n_entities == 0 || n_groups == 0) return 0;
    const Slice sh = slice_shape(S.n_entities);
    return std::min(sh.nr, n_groups * S.n_planes) * sh.ne * kExchangeBytes;
}

cudaError_t sharded_quantile_round(QuantileShard &Q, const void *reduced, void *partial, uint64_t *partial_bytes,
                                   int *launches, cudaStream_t s)
{
    *partial_bytes = 0;
    *launches = 0;
    const QuantileParams &S = Q.S;
    const uint64_t n_groups = Q.table.size();
    const uint64_t n_slices = S.n_planes && S.n_entities ? slices_of(S, n_groups) : 0;
    std::vector<uint32_t> all(n_groups);
    for (uint32_t g = 0; g < n_groups; ++g) all[g] = g;
    CUDA_TRY(radix_attributes());
    if (Q.level >= 0) {  // the sums of the last round's words, then the plan of the pass they count
        const SliceRun r = slice_run(S, Q.table, all.data(), n_groups, Q.slice, Q.scratch, true);
        const uint64_t G = r.L.G;
        CUDA_TRY(cudaMemcpyAsync(Q.level == 0 ? (void *)r.L.cnt : (void *)r.L.hist, reduced,
                                 Q.level == 0 ? G * 4 : G * kExchangeBytes, cudaMemcpyDefault, s));
        CUDA_TRY(cudaMemsetAsync(r.L.todo, 0, 4, s));
        launch_plan(S, r, Q.level, s);
        uint32_t todo = 0;
        CUDA_TRY(cudaMemcpyAsync(&todo, r.L.todo, 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        *launches += 1;
        if (todo && Q.level < kLevels) {
            launch_pass(S, r, s);
            ++Q.level;
            *launches += 1;
            CUDA_TRY(cudaMemcpyAsync(partial, r.L.hist, G * kExchangeBytes, cudaMemcpyDefault, s));
            CUDA_TRY(cudaStreamSynchronize(s));
            *partial_bytes = G * kExchangeBytes;
            return cudaGetLastError();
        }
        launch_finish(S, r, s);
        *launches += 1;
        ++Q.slice;
        Q.level = -1;
    }
    if (Q.slice < n_slices) {
        const SliceRun r = slice_run(S, Q.table, all.data(), n_groups, Q.slice, Q.scratch, true);
        CUDA_TRY(launch_open(S, r, Q.slice == 0, 0, s));
        *launches += r.grid ? 2 : 1;
        Q.level = 0;
        CUDA_TRY(cudaMemcpyAsync(partial, r.L.cnt, r.L.G * 4, cudaMemcpyDefault, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        *partial_bytes = r.L.G * 4;
        return cudaGetLastError();
    }
    if (n_slices)
        CUDA_TRY(cudaMemcpyAsync(&Q.reads, layout_of(0, Q.scratch, true).reads, 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    return cudaGetLastError();
}

} // namespace b200
