// Ensemble statistics over the world axis: for every (world group, plane, entity) one record (count, mean, m2, min,
// max) over the finite values of the group's worlds (include/b200_sixdof.h b200_sixdof_trajectory_stats / _state_stats,
// and the _group_stats entries).  A world group is a contiguous world range; the ungrouped entries are the one-group
// case [0, n_worlds) of the same code.
//
// Shape of the reduction.  A block reduces one chunk of worlds of one group of one plane for a tile of entities.  Thread
// t takes entity e = t % Et of the tile and the worlds w0 + j, w0 + j + J, ... of the chunk (j = t / Et): with Et = E <=
// 256 entities per tile and J = 256 / E, lane t of world-step k reads body (w0 + j + kJ) E + e = w0 E + kJE + t, so a
// warp reads 32 consecutive doubles; worlds of more than 256 entities use tiles of 256 consecutive entities and J = 1.
// Inside a thread, shifted sums: K = the thread's first finite value, S1 = sum (x - K), S2 = sum (x - K)^2, which
// stays well conditioned because K is one of the values (|mean - K| is of the order of the spread, never of |mean|).
// The J partials of an entity are merged in a fixed binary tree in shared memory, the chunks of a group left to right
// in a second launch.  A group's chunking depends on (its size, n_entities) alone (stats_shape), and chunk c of a group
// of size n starting at world o reads the worlds o + [c Wc, (c + 1) Wc) in the order a batch of exactly those n worlds
// reads [c Wc, (c + 1) Wc): a group's record has the bits of the ungrouped call on a batch of its worlds, whatever the
// other groups and planes of the launch.  There are no atomics: the same input gives the same bits on every call.
//
// Groups are found through the group table (WorldGroup): k0 = the chunks of the groups before it, so the chunks of all
// groups are numbered 0 .. sum C_g and a block finds the group of its chunk by binary search over k0.  An empty group has
// one chunk of no worlds, which writes count 0 and NaN.  Scratch: the partials of the chunks, [5][chunks][planes * E]
// f64, run in slices of groups and planes that keep it at most kScratchBytes (256 MiB), or one group-plane's
// 5 * 64 * 8 * E bytes when that alone is more (E > 104857).
#include <algorithm>
#include <cfloat>
#include <vector>

#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kStatsThreads = 256;
constexpr uint64_t kMaxChunks = 64;     // chunks per plane: the sequential length of the second pass
constexpr uint64_t kMinPerThread = 8;   // values per thread at least (fewer chunks, less scratch)
constexpr uint64_t kScratchBytes = 256ull << 20;  // chunk partials of one slice at most

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

// The groups [g0, g1) of a table of G groups and the planes [p0, p0 + np) of one slice; chunks k0 .. k1 of the table
// are the groups' chunks.
struct Slice {
    const WorldGroup *groups;
    uint64_t G, g0, g1, k0, k1, p0, np;
};

__device__ inline void write_final(const StatsParams &S, uint64_t G, uint64_t g, uint64_t i, uint64_t e, const StatsGroup &r)
{
    const uint64_t W = S.planes_per_sample;
    double *o = S.out + ((((i / W) * G + g) * S.n_entities + e) * W + i % W) * 5;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const bool any = r.n > 0.0;
    o[0] = r.n;
    o[1] = any ? r.mean : nan;
    o[2] = any ? r.m2 : nan;
    o[3] = any ? r.mn : nan;
    o[4] = any ? r.mx : nan;
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

// pass 1: task = (plane p0 + il, chunk k of the slice, tile) -> the chunk's record per entity of the tile: finished
// when its group has one chunk, else a partial in scratch, SoA [5][Q][PE] with Q = k1 - k0 chunks and PE = np * E
// (partial r = il * E + e).  sp gives the tiles (Et, J, T); each group's Wc and C come from the table.
__global__ void __launch_bounds__(kStatsThreads, 4) world_stats_chunk_kernel(StatsParams S, Shape sp, Slice L, double *scratch)
{
    __shared__ StatsGroup sh[kStatsThreads];
    const uint64_t E = S.n_entities, Q = L.k1 - L.k0, PE = L.np * E;
    const uint64_t n_tasks = L.np * Q * sp.T;
    const unsigned t = threadIdx.x;
    const unsigned el = t % (unsigned)sp.Et, j = t / (unsigned)sp.Et;
    for (uint64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
        const uint64_t tile = task % sp.T, qc = (task / sp.T) % Q, il = task / (sp.T * Q);
        const uint64_t i = L.p0 + il, k = L.k0 + qc;
        const uint64_t g = group_of_chunk(L.groups, L.g0, L.g1, k);
        const WorldGroup wg = L.groups[g];
        const uint64_t c = k - wg.k0;
        const uint64_t e = tile * sp.Et + el;
        const uint64_t w0 = wg.o + c * wg.Wc;
        const uint64_t w1 = wg.o + min((c + 1) * wg.Wc, wg.n);
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
        StatsGroup r = acc.group();
        if (sp.J > 1) {
            sh[t] = r;
            __syncthreads();
            for (uint64_t s = 1; s < sp.J; s <<= 1) {
                if (j < sp.J && j % (2 * s) == 0 && j + s < sp.J) stats_merge(sh[t], sh[t + s * sp.Et]);
                __syncthreads();
            }
            r = sh[t];
            __syncthreads(); // the next task overwrites sh
        }
        if (j == 0 && e < E) {
            if (wg.C == 1) {
                write_final(S, L.G, g, i, e, r);
            } else {
                const uint64_t ri = il * E + e;
                scratch[(0 * Q + qc) * PE + ri] = r.n;
                scratch[(1 * Q + qc) * PE + ri] = r.mean;
                scratch[(2 * Q + qc) * PE + ri] = r.m2;
                scratch[(3 * Q + qc) * PE + ri] = r.mn;
                scratch[(4 * Q + qc) * PE + ri] = r.mx;
            }
        }
    }
}

// pass 2: one thread per (group of the slice with C > 1, plane, entity) merges its C chunk partials in chunk order
__global__ void __launch_bounds__(kStatsThreads) world_stats_merge_kernel(StatsParams S, Slice L, const double *scratch)
{
    const uint64_t E = S.n_entities, Q = L.k1 - L.k0, PE = L.np * E;
    const uint64_t n = (L.g1 - L.g0) * PE;
    for (uint64_t x = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; x < n; x += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t g = L.g0 + x / PE, ri = x % PE;
        const WorldGroup wg = L.groups[g];
        if (wg.C == 1) continue;  // finished by pass 1
        const uint64_t q0 = wg.k0 - L.k0;
        StatsGroup acc{0.0, 0.0, 0.0, 0.0, 0.0};
        for (uint64_t c = 0; c < wg.C; ++c) {
            const uint64_t q = q0 + c;
            const StatsGroup b{scratch[(0 * Q + q) * PE + ri], scratch[(1 * Q + q) * PE + ri],
                               scratch[(2 * Q + q) * PE + ri], scratch[(3 * Q + q) * PE + ri],
                               scratch[(4 * Q + q) * PE + ri]};
            stats_merge(acc, b);
        }
        write_final(S, L.G, g, L.p0 + ri / E, ri % E, acc);
    }
}

// The slices of a launch over the planes of S and the groups of `table`: each slice's scratch (where any of its groups
// has more than one chunk) at most kScratchBytes, or one group-plane when that alone is more.  scratch = the largest
// slice's scratch in f64.
std::vector<Slice> stats_slices(const StatsParams &S, const std::vector<WorldGroup> &table, uint64_t *scratch)
{
    std::vector<Slice> out;
    *scratch = 0;
    const uint64_t G = table.size(), per_chunk = 5ull * S.n_entities;  // f64 per chunk and plane
    const uint64_t budget = kScratchBytes / 8;
    for (uint64_t g0 = 0; g0 < G;) {
        uint64_t g1 = g0 + 1, chunks = table[g0].C;
        bool merge = table[g0].C > 1;
        while (g1 < G && (chunks + table[g1].C) * per_chunk <= budget) {
            chunks += table[g1].C;
            merge = merge || table[g1].C > 1;
            ++g1;
        }
        const uint64_t np = merge ? std::max<uint64_t>(1, budget / (chunks * per_chunk)) : S.n_planes;
        for (uint64_t p0 = 0; p0 < S.n_planes; p0 += np) {
            Slice L{nullptr, G, g0, g1, table[g0].k0, table[g0].k0 + chunks, p0, std::min(np, S.n_planes - p0)};
            out.push_back(L);
            if (merge) *scratch = std::max(*scratch, chunks * per_chunk * L.np);
        }
        g0 = g1;
    }
    return out;
}

} // namespace

std::vector<WorldGroup> world_group_table(const uint64_t *sizes, uint64_t n_groups, uint64_t n_entities)
{
    std::vector<WorldGroup> t(n_groups);
    uint64_t o = 0, k0 = 0;
    for (uint64_t g = 0; g < n_groups; ++g) {
        // no entities: no planes to reduce, and stats_shape would divide by E; one chunk of the whole group stands in
        const Shape sp = n_entities ? stats_shape(sizes[g], n_entities) : Shape{0, 0, 0, sizes[g], 1};
        t[g] = {o, sizes[g], sp.Wc, std::max<uint64_t>(sp.C, 1), k0};
        o += sizes[g];
        k0 += t[g].C;
    }
    return t;
}

uint64_t world_stats_scratch_doubles(const StatsParams &S, const std::vector<WorldGroup> &table)
{
    uint64_t scratch = 0;
    if (S.n_planes && S.n_entities) stats_slices(S, table, &scratch);
    return scratch;
}

cudaError_t launch_world_stats(const StatsParams &S, const WorldGroup *groups, const std::vector<WorldGroup> &table,
                               double *scratch, int *launches, cudaStream_t s)
{
    *launches = 0;
    if (S.n_planes == 0 || S.n_entities == 0) return cudaSuccess;
    const Shape sp = stats_shape(0, S.n_entities);  // the tiles: Et, J, T depend on E alone
    const uint64_t cap = 64ull * kNumSMs * 8;  // resident blocks x 64; larger launches stride over their tasks
    uint64_t unused;
    for (Slice L : stats_slices(S, table, &unused)) {
        L.groups = groups;
        const uint64_t tasks = L.np * (L.k1 - L.k0) * sp.T;
        world_stats_chunk_kernel<<<(unsigned)std::min(tasks, cap), kStatsThreads, 0, s>>>(S, sp, L, scratch);
        ++*launches;
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
        bool merge = false;
        for (uint64_t g = L.g0; g < L.g1; ++g) merge = merge || table[g].C > 1;
        if (!merge) continue;
        const uint64_t n = (L.g1 - L.g0) * L.np * S.n_entities;
        world_stats_merge_kernel<<<(unsigned)std::min((n + kStatsThreads - 1) / kStatsThreads, cap), kStatsThreads, 0, s>>>(S, L, scratch);
        ++*launches;
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

} // namespace b200
