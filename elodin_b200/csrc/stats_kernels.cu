// Ensemble statistics over the world axis: for every (plane, entity) one group (count, mean, m2, min, max) over the
// finite values of all worlds (include/b200_sixdof.h b200_sixdof_trajectory_stats / _state_stats).
//
// Shape of the reduction.  A block reduces one chunk of worlds of one plane for a tile of entities.  Thread t takes
// entity e = t % Et of the tile and the worlds w0 + j, w0 + j + J, ... of the chunk (j = t / Et): with Et = E <= 256
// entities per tile and J = 256 / E, lane t of world-step k reads body (w0 + j + kJ) E + e = w0 E + kJE + t, so a
// warp reads 32 consecutive doubles; worlds of more than 256 entities use tiles of 256 consecutive entities and J = 1.
// Inside a thread, shifted sums: K = the thread's first finite value, S1 = sum (x - K), S2 = sum (x - K)^2, which
// stays well conditioned because K is one of the values (|mean - K| is of the order of the spread, never of |mean|).
// The J partials of an entity are merged in a fixed binary tree in shared memory, the chunks of a plane left to right
// in a second launch.  The chunking depends on (n_worlds, n_entities) alone, so a group's bits do not depend on how
// many other planes share the launch, and there are no atomics: the same input gives the same bits on every call.
#include <algorithm>
#include <cfloat>

#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kStatsThreads = 256;
constexpr uint64_t kMaxChunks = 64;     // chunks per plane: the sequential length of the second pass
constexpr uint64_t kMinPerThread = 8;   // values per thread at least (fewer chunks, less scratch)

struct Shape {
    uint64_t Et, J, T;  // entities per tile, world lanes per entity, tiles
    uint64_t Wc, C;     // worlds per chunk, chunks
};

inline Shape stats_shape(uint64_t n_worlds, uint64_t E)
{
    Shape s;
    s.Et = E <= kStatsThreads ? E : kStatsThreads;
    s.J = E <= kStatsThreads ? kStatsThreads / E : 1;
    s.T = (E + s.Et - 1) / s.Et;
    const uint64_t lanes = kMaxChunks * s.J;
    uint64_t per = (n_worlds + lanes - 1) / lanes;
    if (per < kMinPerThread) per = kMinPerThread;
    s.Wc = per * s.J;
    s.C = (n_worlds + s.Wc - 1) / s.Wc;
    return s;
}

__device__ inline void write_final(const StatsParams &S, uint64_t i, uint64_t e, const StatsGroup &g)
{
    const uint64_t W = S.planes_per_sample;
    double *o = S.out + (((i / W) * S.n_entities + e) * W + i % W) * 5;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const bool any = g.n > 0.0;
    o[0] = g.n;
    o[1] = any ? g.mean : nan;
    o[2] = any ? g.m2 : nan;
    o[3] = any ? g.mn : nan;
    o[4] = any ? g.mx : nan;
}

struct Shifted {
    uint32_t n = 0;
    double K = 0.0, s1 = 0.0, s2 = 0.0;
    double mn = HUGE_VAL, mx = -HUGE_VAL;

    __device__ __forceinline__ void add(double x)
    {
        if (!(fabs(x) <= DBL_MAX)) return; // NaN / +-inf: not counted
        if (n == 0) K = x;
        const double y = x - K;
        s1 += y;
        s2 = fma(y, y, s2);
        mn = fmin(mn, x);
        mx = fmax(mx, x);
        ++n;
    }

    __device__ StatsGroup group() const
    {
        StatsGroup g{(double)n, 0.0, 0.0, mn, mx};
        if (n) {
            const double dn = (double)n;
            g.mean = K + s1 / dn;
            // s2 = m2 + n (mean - K)^2 <= (2n + 1) m2 (K is one of the values), so an overflowed s2 means m2 is at the
            // top of the range: +inf, never inf - inf = NaN clamped to 0.  s1 * (s1 / n) <= s2 does not overflow.
            g.m2 = s2 > DBL_MAX ? HUGE_VAL : fmax(s2 - s1 * (s1 / dn), 0.0);
        }
        return g;
    }
};

// pass 1: task = (plane i, chunk c, tile) -> the chunk's group per entity of the tile: finished when C = 1, else a
// partial in scratch, SoA [5][C][G] with G = n_planes * E (group g = i * E + e)
__global__ void __launch_bounds__(kStatsThreads, 4) world_stats_chunk_kernel(StatsParams S, Shape sp, double *scratch)
{
    __shared__ StatsGroup sh[kStatsThreads];
    const uint64_t E = S.n_entities, G = S.n_planes * E;
    const uint64_t n_tasks = S.n_planes * sp.C * sp.T;
    const unsigned t = threadIdx.x;
    const unsigned el = t % (unsigned)sp.Et, j = t / (unsigned)sp.Et;
    for (uint64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
        const uint64_t tile = task % sp.T, c = (task / sp.T) % sp.C, i = task / (sp.T * sp.C);
        const uint64_t e = tile * sp.Et + el;
        const uint64_t w0 = c * sp.Wc;
        const uint64_t w1 = min(w0 + sp.Wc, S.n_worlds);
        Shifted acc;
        if (j < sp.J && e < E) {
            const double *p = stats_plane(S, i) + e;
            const uint64_t step = sp.J * E;
            uint64_t w = w0 + j;
            for (; w + 3 * sp.J < w1; w += 4 * sp.J) { // four loads in flight before the first is used
                const double *q = p + w * E;
                const double x0 = __ldcs(q), x1 = __ldcs(q + step), x2 = __ldcs(q + 2 * step), x3 = __ldcs(q + 3 * step);
                acc.add(x0);
                acc.add(x1);
                acc.add(x2);
                acc.add(x3);
            }
            for (; w < w1; w += sp.J) acc.add(__ldcs(p + w * E));
        }
        StatsGroup g = acc.group();
        if (sp.J > 1) {
            sh[t] = g;
            __syncthreads();
            for (uint64_t s = 1; s < sp.J; s <<= 1) {
                if (j < sp.J && j % (2 * s) == 0 && j + s < sp.J) stats_merge(sh[t], sh[t + s * sp.Et]);
                __syncthreads();
            }
            g = sh[t];
            __syncthreads(); // the next task overwrites sh
        }
        if (j == 0 && e < E) {
            if (sp.C == 1) {
                write_final(S, i, e, g);
            } else {
                const uint64_t gi = i * E + e;
                scratch[(0 * sp.C + c) * G + gi] = g.n;
                scratch[(1 * sp.C + c) * G + gi] = g.mean;
                scratch[(2 * sp.C + c) * G + gi] = g.m2;
                scratch[(3 * sp.C + c) * G + gi] = g.mn;
                scratch[(4 * sp.C + c) * G + gi] = g.mx;
            }
        }
    }
}

// pass 2 (C > 1): one thread per group merges its C chunk partials in chunk order
__global__ void __launch_bounds__(kStatsThreads) world_stats_merge_kernel(StatsParams S, Shape sp, const double *scratch)
{
    const uint64_t E = S.n_entities, G = S.n_planes * E;
    for (uint64_t gi = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; gi < G; gi += (uint64_t)gridDim.x * blockDim.x) {
        StatsGroup acc{0.0, 0.0, 0.0, 0.0, 0.0};
        for (uint64_t c = 0; c < sp.C; ++c) {
            const StatsGroup b{scratch[(0 * sp.C + c) * G + gi], scratch[(1 * sp.C + c) * G + gi],
                               scratch[(2 * sp.C + c) * G + gi], scratch[(3 * sp.C + c) * G + gi],
                               scratch[(4 * sp.C + c) * G + gi]};
            stats_merge(acc, b);
        }
        write_final(S, gi / E, gi % E, acc);
    }
}

} // namespace

uint64_t world_stats_scratch_doubles(const StatsParams &S)
{
    if (S.n_worlds == 0 || S.n_entities == 0) return 0;
    const Shape sp = stats_shape(S.n_worlds, S.n_entities);
    return sp.C > 1 ? 5ull * sp.C * S.n_planes * S.n_entities : 0;
}

cudaError_t launch_world_stats(const StatsParams &S, double *scratch, int *launches, cudaStream_t s)
{
    *launches = 0;
    if (S.n_planes == 0 || S.n_worlds == 0 || S.n_entities == 0) return cudaSuccess;
    const Shape sp = stats_shape(S.n_worlds, S.n_entities);
    const uint64_t cap = 64ull * kNumSMs * 8;  // resident blocks x 64; larger launches stride over their tasks
    const uint64_t tasks = S.n_planes * sp.C * sp.T;
    world_stats_chunk_kernel<<<(unsigned)std::min(tasks, cap), kStatsThreads, 0, s>>>(S, sp, scratch);
    *launches = 1;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess || sp.C == 1) return e;
    const uint64_t G = S.n_planes * S.n_entities;
    world_stats_merge_kernel<<<(unsigned)std::min((G + kStatsThreads - 1) / kStatsThreads, cap), kStatsThreads, 0, s>>>(S, sp, scratch);
    *launches = 2;
    return cudaGetLastError();
}

} // namespace b200
