// Ensemble histograms over the world axis: for every (sample, world group, spec) one record of integer counts over the
// group's worlds (include/b200_sixdof.h b200_sixdof_trajectory_histograms / _state_histograms, and the
// _group_histograms entries).  A world group is a contiguous world range; the ungrouped entries are the one-group case
// [0, n_worlds) of the same code.
//
// A value's cell is a pure function of the value and the spec's edges (numpy's own rules, below), so the table is a set
// of integer counts, and integer-valued f64 sums below 2^53 are exact in any order: the result does not depend on the
// launch shape or on the order of the atomics, and a group's record is the ungrouped table of a batch of its worlds.
// Shape of the reduction: the table is zeroed with one memset, then one launch; block task = (chunk of worlds of one
// group, sample, spec).  The chunks of all groups are numbered through the group table (WorldGroup::k0) and a block
// finds its group by binary search.  A block clears its spec's record (<= 4099 u32 cells) and copies its edges (<= 4099
// f64) into shared memory, walks the chunk with consecutive lanes on consecutive worlds (four loads in flight per
// thread), classifies each value, and adds one per world to its cell.  Lanes of a warp that hit the same cell are
// counted together (__match_any_sync) before one shared atomic, so a warp whose 32 worlds share a bin (early rows of a
// campaign) costs one atomic, not 32 serialised ones.  The block then adds its non-zero cells to its group's record of
// the f64 table with atomicAdd.  No scratch beyond the edges and the group table, no merge pass.
#include <algorithm>
#include <cfloat>

#include "sixdof_device.cuh"
#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kThreads = 256;
constexpr unsigned kUnroll = 4;                          // loads in flight per thread and axis
constexpr uint64_t kChunkTasks = 2ull * kNumSMs;         // block tasks of a call: 2 per SM
constexpr uint64_t kMinWorlds = kThreads * kUnroll;      // worlds per chunk at least: one pass of the block
constexpr uint32_t kNone = 0xffffffffu;                  // a lane without a world

// 1D cell of a finite value: numpy's _histogram, operation for operation (uncontracted, correctly rounded):
// keep lo <= x <= hi; f = ((x - lo) / (hi - lo)) * n; i = trunc(f); i == n -> n - 1; x < edge[i] -> i - 1; then
// x >= edge[i + 1] and i != n - 1 -> i + 1.  The division goes through ex::div_rcp with the divisor part computed once
// per task (ex::rcp_prep), which gives __ddiv_rn's bits; outside its window the quotient is redone with __ddiv_rn.
__device__ __forceinline__ uint32_t cell_1d(double x, const HistParams::Spec &sp, const ex::Rcp &r, const double *e)
{
    if (!(fabs(x) <= DBL_MAX)) return 0;
    if (x < sp.lo[0]) return 1;
    if (x > sp.hi[0]) return 2;
    const uint32_t n = sp.bins[0];
    const double d = __dsub_rn(x, sp.lo[0]);
    bool ok = true;
    double q = ex::div_rcp(d, r, ok);
    if (!ok) q = __ddiv_rn(d, ex::rare_path(r.d));
    const double f = __dmul_rn(q, (double)n);
    uint32_t i = (uint32_t)f;  // 0 <= f <= n: truncation
    if (i == n) i = n - 1;
    if (x < e[i]) i -= 1;
    if (x >= e[i + 1] && i != n - 1) i += 1;
    return 3 + i;
}

// numpy's histogramdd rule on one axis of a value in [lo, hi]: searchsorted(edges, v, side='right') - 1, with v == hi
// moved into the last bin -- the largest j < n with edge[j] <= v (edge[0] = lo <= v; the edges strictly increase)
__device__ __forceinline__ uint32_t bin_dd(double v, const double *e, uint32_t n)
{
    uint32_t j = 0;
    for (uint32_t step = 1u << (31 - __clz(n)); step; step >>= 1)
        if (j + step < n && e[j + step] <= v) j += step;
    return j;
}

__device__ __forceinline__ uint32_t cell_2d(double a, double b, const HistParams::Spec &sp, const double *ea, const double *eb)
{
    if (!(fabs(a) <= DBL_MAX && fabs(b) <= DBL_MAX)) return 0;
    if (!(a >= sp.lo[0] && a <= sp.hi[0] && b >= sp.lo[1] && b <= sp.hi[1])) return 1;
    return 2 + bin_dd(a, ea, sp.bins[0]) * sp.bins[1] + bin_dd(b, eb, sp.bins[1]);
}

// spec k of P with constant indices, so that the spec table stays in the parameter space
__device__ __forceinline__ HistParams::Spec spec_of(const HistParams &P, uint32_t k)
{
    HistParams::Spec sp = P.spec[0];
#pragma unroll
    for (uint32_t i = 1; i < B200_MAX_HISTOGRAMS; ++i)
        if (i == k) sp = P.spec[i];
    return sp;
}

// one world per lane: the lanes with the same cell add their count with one shared atomic
__device__ __forceinline__ void count(uint32_t *cells, uint32_t c)
{
    const unsigned same = __match_any_sync(0xffffffffu, c);
    if (c != kNone && (threadIdx.x & 31) == (unsigned)(__ffs(same) - 1)) atomicAdd(&cells[c], (unsigned)__popc(same));
}

__global__ void __launch_bounds__(kThreads) hist_kernel(HistParams P, const WorldGroup *groups, uint64_t G, uint64_t Q,
                                                        uint64_t n_samples)
{
    extern __shared__ double smem[];
    double *edges = smem;                                   // [P.smem_edges]
    uint32_t *cells = (uint32_t *)(smem + P.smem_edges);   // [record length]
    const uint64_t E = P.n_entities;
    const uint64_t n_tasks = Q * n_samples * P.n_specs;  // Q = the chunks of all groups
    for (uint64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
        const uint64_t k = task % Q, s = (task / Q) % n_samples;
        const HistParams::Spec sp = spec_of(P, (uint32_t)(task / (Q * n_samples)));
        const uint64_t g = group_of_chunk(groups, 0, G, k);
        const WorldGroup wg = groups[g];
        const bool two = sp.n_axes == 2;
        const uint32_t R = two ? 2 + sp.bins[0] * sp.bins[1] : 3 + sp.bins[0];
        const uint32_t ne = sp.bins[0] + 1 + (two ? sp.bins[1] + 1 : 0);
        __syncthreads();  // the previous task's cells are flushed
        for (uint32_t i = threadIdx.x; i < R; i += blockDim.x) cells[i] = 0;
        for (uint32_t i = threadIdx.x; i < ne; i += blockDim.x) edges[i] = P.edges[sp.edge_off + i];
        __syncthreads();
        const double *ea = edges, *eb = edges + sp.bins[0] + 1;
        const double *xa = sample_plane(P, s, sp.plane[0]) + sp.entity;
        const double *xb = two ? sample_plane(P, s, sp.plane[1]) + sp.entity : xa;
        const ex::Rcp r = ex::rcp_prep(sp.den);
        const uint64_t w0 = wg.o + (k - wg.k0) * wg.Wc, w1 = min(w0 + wg.Wc, wg.o + wg.n);
        for (uint64_t base = w0; base < w1; base += (uint64_t)kUnroll * blockDim.x) { // uniform trip count per warp
            double va[kUnroll], vb[kUnroll];
#pragma unroll
            for (unsigned u = 0; u < kUnroll; ++u) {
                const uint64_t w = base + u * blockDim.x + threadIdx.x;
                va[u] = w < w1 ? xa[w * E] : 0.0;  // cached loads: several specs often read one plane
                vb[u] = two && w < w1 ? xb[w * E] : 0.0;
            }
#pragma unroll
            for (unsigned u = 0; u < kUnroll; ++u) {
                const uint64_t w = base + u * blockDim.x + threadIdx.x;
                uint32_t cl = kNone;
                if (w < w1) cl = two ? cell_2d(va[u], vb[u], sp, ea, eb) : cell_1d(va[u], sp, r, ea);
                count(cells, cl);
            }
        }
        __syncthreads();
        double *o = P.out + (s * G + g) * P.record_len + sp.rec_off;
        for (uint32_t i = threadIdx.x; i < R; i += blockDim.x)
            if (cells[i]) atomicAdd(o + i, (double)cells[i]);
    }
}

} // namespace

std::vector<WorldGroup> hist_group_table(const uint64_t *sizes, uint64_t n_groups, uint64_t n_pairs)
{
    uint64_t n_worlds = 0;
    for (uint64_t g = 0; g < n_groups; ++g) n_worlds += sizes[g];
    std::vector<WorldGroup> t(n_groups);
    uint64_t o = 0, k0 = 0;
    for (uint64_t g = 0; g < n_groups; ++g) {
        const uint64_t n = sizes[g];
        uint64_t C = 0, Wc = 0;
        if (n) {  // the group's share of kChunkTasks over the call's pairs, rounded up: ceil(kChunkTasks / n_pairs) for one group
            const uint64_t pairs = std::max<uint64_t>(n_pairs, 1);
            const uint64_t want = std::max<uint64_t>(1, (kChunkTasks * n + n_worlds * pairs - 1) / (n_worlds * pairs));
            C = std::max<uint64_t>(1, std::min(want, n / kMinWorlds));
            Wc = (n + C - 1) / C;
            C = (n + Wc - 1) / Wc;
        }
        t[g] = {o, n, Wc, C, k0};
        o += n;
        k0 += C;
    }
    return t;
}

cudaError_t launch_histograms(const HistParams &P, const WorldGroup *groups, const std::vector<WorldGroup> &table,
                              int *launches, cudaStream_t s)
{
    *launches = 0;
    const uint64_t n_s = P.planes_per_sample ? P.n_planes / P.planes_per_sample : 0;
    const uint64_t G = table.size();
    if (n_s == 0 || G == 0 || P.n_entities == 0) return cudaSuccess;
    cudaError_t e = cudaMemsetAsync(P.out, 0, n_s * G * P.record_len * 8ull, s);
    if (e != cudaSuccess) return e;
    const uint64_t Q = table.back().k0 + table.back().C;
    if (Q == 0) return cudaSuccess;  // no worlds: the zeroed table
    uint32_t R = 0;
    for (uint32_t k = 0; k < P.n_specs; ++k)
        R = std::max(R, P.spec[k].n_axes == 2 ? 2 + P.spec[k].bins[0] * P.spec[k].bins[1] : 3 + P.spec[k].bins[0]);
    const size_t smem = P.smem_edges * 8ull + R * 4ull;
    e = cudaFuncSetAttribute(hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const uint64_t tasks = Q * n_s * P.n_specs;
    hist_kernel<<<(unsigned)std::min<uint64_t>(tasks, 64ull * kNumSMs * 8), kThreads, smem, s>>>(P, groups, G, Q, n_s);
    *launches = 1;
    return cudaGetLastError();
}

} // namespace b200
