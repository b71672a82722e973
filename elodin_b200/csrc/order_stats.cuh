// The building blocks of the order-statistic kernels (quantile_kernels.cu, topk_kernels.cu, rank_kernels.cu): the
// IEEE totalOrder key, the composite (key, index) order and its pair sort, the chunk walk of a radix slice, and the
// route split of the groups by size.  Everything here has internal linkage (an anonymous namespace), so each includer
// compiles its own copy, as if it were written in that file, and its kernels' code is what it would be then.
#pragma once
#include <algorithm>
#include <cfloat>
#include <vector>

#include "sixdof_internal.h"

namespace b200 {
namespace {

// ---- route split ----------------------------------------------------------------------------------------------------
// Each world group takes a route from its size n alone: up to kWarpMax worlds (empty groups included) a warp sorts it
// in shared memory, eight groups per block; up to kSmallMax a block does; larger groups take the file's radix route.
// quantile_order lists a table's groups by route once per table, and every launch counts the routes of that order with
// routes_of, so the order and the counts cannot disagree.

constexpr unsigned kWarpMax = 256;
constexpr unsigned kSmallMax = 8192;

enum : int { kWarpRoute = 0, kBlockRoute = 1, kRadixRoute = 2 };

inline int route_of(uint64_t n) { return n <= kWarpMax ? kWarpRoute : n <= kSmallMax ? kBlockRoute : kRadixRoute; }

// the groups of each route of an order listed by route: order[0 .. warp) warp, [warp, block) block, [block, size) radix
struct Routes {
    uint32_t warp, block;
};

inline Routes routes_of(const std::vector<WorldGroup> &table, const std::vector<uint32_t> &order)
{
    Routes r{0, 0};
    for (uint32_t g : order) {
        r.warp += route_of(table[g].n) == kWarpRoute;
        r.block += route_of(table[g].n) <= kBlockRoute;
    }
    return r;
}

// the keys a block of the block route sorts: the power of two at least the route's largest group
inline uint32_t block_keys(const std::vector<WorldGroup> &table, const std::vector<uint32_t> &order, const Routes &r)
{
    uint64_t n = 0;
    for (uint32_t k = r.warp; k < r.block; ++k) n = std::max(n, table[order[k]].n);
    uint32_t P = 1;
    while (P < n) P <<= 1;
    return P;
}

// ---- keys and their order -------------------------------------------------------------------------------------------

// the IEEE totalOrder key of x: ascending keys are ascending values, -0 < +0
__device__ __forceinline__ unsigned long long order_key(double x)
{
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__device__ __forceinline__ double key_value(unsigned long long k)
{
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

__device__ __forceinline__ bool finite(double x) { return fabs(x) <= DBL_MAX; }

// (a, ai) < (b, bi) in the composite order
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

// ---- radix slices ---------------------------------------------------------------------------------------------------

// the row of chunk k of a slice: the last of rows[0 .. nr) whose first chunk (k0) is at most k
template <class Row>
__device__ inline uint64_t row_of_chunk(const Row *rows, uint64_t nr, uint64_t k)
{
    uint64_t lo = 0, hi = nr - 1;
    while (lo < hi) {
        const uint64_t mid = (lo + hi + 1) / 2;
        if (rows[mid].k0 <= k) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

constexpr uint64_t kGridCap = 64ull * kNumSMs * 8;

// the world chunk of a task of n worlds in a slice of T tasks, for blocks of `threads` threads that each take every
// threads-th world: about 8 blocks per SM over the slice, at least 16 worlds per thread (a block's histogram clear and
// flush is amortised)
inline uint32_t chunk_of(uint64_t n, uint64_t T, uint64_t threads)
{
    const uint64_t want = std::max<uint64_t>(1, 8ull * kNumSMs / std::max<uint64_t>(1, T));
    uint64_t per = (n + want - 1) / want;
    per = std::max<uint64_t>(per, 16ull * threads);
    return (uint32_t)((per + threads - 1) / threads * threads);
}

// return the error of a CUDA runtime call from the enclosing function (which returns cudaError_t)
#define CUDA_TRY(call)                    \
    do {                                  \
        const cudaError_t e_ = (call);    \
        if (e_ != cudaSuccess) return e_; \
    } while (0)

} // namespace
} // namespace b200
