// Ensemble covariance over the world axis: for every (sample, world group, entity) one record (n, mean[p], M[p][p])
// over the group's worlds whose p selected values are all finite (include/b200_sixdof.h
// b200_sixdof_trajectory_covariance / _state_covariance and the _group_covariance entries).  A world group is a
// contiguous world range; the ungrouped entries are the one-group case [0, n_worlds) of the same code.
//
// Shape of the reduction.  A group's worlds are cut into C chunks of Wc consecutive worlds; Wc and C depend on (the
// group's size, n_entities) alone (cov_chunks), and chunk c of a group starting at world o reads o + [c Wc, (c + 1) Wc),
// so a group's record has the bits of the ungrouped call on a batch of exactly its worlds.  The chunks of all groups
// are numbered through the group table (WorldGroup, k0 = the chunks of the groups before it) and a block finds the
// group of its chunk by binary search, as the statistics do; an empty group is one chunk of no worlds, which writes
// n = 0 and NaN.  A block reduces one chunk of one sample for a tile of Et entities: it stages Wt worlds x p planes x
// Et entities at a time in shared memory (lanes read consecutive doubles of one plane: entities, then worlds when the
// tile is every entity), marks the complete worlds, then thread (entity, tile) accumulates a 4 x 4 register tile of the
// upper triangle of M over the chunk's complete worlds in world order.  Shift: K = the chunk's first complete world's
// row, y = x - K, sums S_a = sum y_a (diagonal tiles) and Q_ab = sum y_a y_b (fma); the chunk's record is
// mean_a = K_a + S_a / n, M_ab = Q_ab - lo (hi / n) with (lo, hi) = (min, max)(S_a, S_b), and M_aa = +inf where Q_aa overflowed.  Each entry is a sequential sum over the same worlds whatever the
// selection, the entity tile or the other planes, so an entry has the same bits in any selection with the same complete
// worlds.  Where a group has C > 1 a second launch merges its chunk records left to right with cov_merge, one thread per
// (group, sample, entity, upper entry).  The partials live in scratch; groups and samples run in slices that keep it
// under kScratchCap.  No atomics.
#include <algorithm>
#include <cfloat>

#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr uint64_t kChunkTasks = 4ull * kNumSMs; // chunk tasks of a one-sample call: 4 blocks per SM (the merge folds
                                                 // C chunks one after another, so C stays small)
constexpr uint64_t kEntTile = 32;                // entity tile the chunk count is sized by
constexpr uint64_t kMinWorlds = 64;              // worlds per chunk at least
constexpr unsigned kMaxThreads = 512;
constexpr unsigned kMinThreads = 128;            // loaders even where few threads accumulate
constexpr uint64_t kStageBytes = 40u << 10;      // staged worlds x planes x entities
constexpr uint64_t kScratchCap = 256ull << 20;
constexpr unsigned kMergeBatch = 8;              // chunk records a merge thread loads at once

struct Chunks {
    uint64_t Wc, C;  // worlds per chunk, chunks
};

inline Chunks cov_chunks(uint64_t n_worlds, uint64_t E)
{
    if (n_worlds == 0 || E == 0) return Chunks{n_worlds, 1};  // one chunk: of no worlds, or of no entities to reduce
    const uint64_t tiles = (E + kEntTile - 1) / kEntTile;
    uint64_t C = std::max<uint64_t>(1, (kChunkTasks + tiles - 1) / tiles);
    C = std::min(C, std::max<uint64_t>(1, (n_worlds + kMinWorlds - 1) / kMinWorlds));
    Chunks c;
    c.Wc = (n_worlds + C - 1) / C;
    c.C = (n_worlds + c.Wc - 1) / c.Wc;
    return c;
}

inline uint32_t nblk(uint32_t p) { return (p + 3) / 4; }
inline uint32_t tri_tiles(uint32_t p) { return nblk(p) * (nblk(p) + 1) / 2; }

// Launch geometry of the chunk kernel (free to depend on p: it decides which thread computes an entry, never how)
struct Geo {
    uint32_t Et, T, threads, Wt;
};

inline Geo cov_geo(const CovParams &S)
{
    Geo g;
    g.T = tri_tiles(S.n_p);
    uint32_t et = 32;
    while (et > 1 && et * g.T > kMaxThreads) et >>= 1;
    g.Et = (uint32_t)std::min<uint64_t>(et, S.n_entities);
    g.threads = std::max(kMinThreads, (g.Et * g.T + 31) / 32 * 32);
    g.Wt = (uint32_t)std::max<uint64_t>(1, kStageBytes / (8ull * S.n_p * g.Et + 1));
    return g;
}

// A slice: the groups [g0, g1) of a table of G groups, their chunks k0 .. k0 + K, and the samples [s0, s0 + ns)
struct Slice {
    const WorldGroup *groups;
    uint64_t G, g0, g1, k0, K, s0, ns;
};

// the final record of (sample s, group g, entity e), or, with scratch, the partial record of chunk q of the slice
__device__ inline double *record(const CovParams &S, const Slice &sl, double *scratch, uint64_t q, uint64_t g, uint64_t s,
                                 uint64_t e)
{
    const uint64_t R = 1 + S.n_p + (uint64_t)S.n_p * S.n_p;
    if (scratch) return scratch + ((q * sl.ns + (s - sl.s0)) * S.n_entities + e) * R;
    return S.out + ((s * sl.G + g) * S.n_entities + e) * R;
}

__device__ inline void tile_of(uint32_t t, uint32_t nb, uint32_t &ab, uint32_t &bb)
{
    ab = 0;
    while (t >= nb - ab) { t -= nb - ab; ++ab; }
    bb = ab + t;
}

// pass 1: task = (sample s of the slice, chunk q of the slice, entity tile) -> the chunk's record per entity: final
// (NaN where n = 0) when its group has C = 1, else a partial record in scratch
__global__ void __launch_bounds__(kMaxThreads) cov_chunk_kernel(CovParams S, Geo geo, Slice sl, double *scratch)
{
    extern __shared__ double smem[];
    __shared__ const double *src_plane[B200_MAX_COV_PLANES];  // the selected planes of the task's sample
    const uint32_t p = S.n_p, Et = geo.Et, Wt = geo.Wt;
    double *xs = smem;                                    // [Wt][p][Et]
    double *ss = xs + (uint64_t)Wt * p * Et;              // [p][Et]: the diagonal tiles' S_a
    unsigned char *ok = (unsigned char *)(ss + p * Et);   // [Wt][Et]
    const uint64_t E = S.n_entities;
    const uint64_t n_et = (E + Et - 1) / Et;
    const uint64_t n_tasks = sl.ns * sl.K * n_et;
    const unsigned t = threadIdx.x;
    const uint32_t el = t % Et, tile = t / Et, nb = (p + 3) / 4;
    const bool active = tile < geo.T;
    uint32_t ab = 0, bb = 0;
    if (active) tile_of(tile, nb, ab, bb);
    const bool diag = ab == bb;
    uint32_t ia[4], ib[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        ia[k] = min(4 * ab + k, p - 1);  // padded rows / columns read plane p - 1 and are never written
        ib[k] = min(4 * bb + k, p - 1);
    }
    for (uint64_t task = blockIdx.x; task < n_tasks; task += gridDim.x) {
        const uint64_t et = task % n_et, q = (task / n_et) % sl.K, s = sl.s0 + task / (n_et * sl.K);
        const uint64_t g = group_of_chunk(sl.groups, sl.g0, sl.g1, sl.k0 + q);
        const WorldGroup wg = sl.groups[g];
        const uint64_t c = sl.k0 + q - wg.k0;
        const uint64_t e0 = et * Et;
        const uint32_t ne = (uint32_t)min((uint64_t)Et, E - e0);
        const uint64_t w0 = wg.o + c * wg.Wc, w1 = wg.o + min((c + 1) * wg.Wc, wg.n);
        const bool fin = wg.C == 1;  // a final record holds NaN where n = 0; a partial leaves them (unread)
        // read after the barrier that opens each tile; the previous task's reads all precede its last tile's barrier
        if (t < p) src_plane[t] = sample_plane(S, s, S.planes[t]);
        double K[8], Q[16], Ssum[4];
#pragma unroll
        for (int k = 0; k < 8; ++k) K[k] = 0.0;
#pragma unroll
        for (int k = 0; k < 16; ++k) Q[k] = 0.0;
#pragma unroll
        for (int k = 0; k < 4; ++k) Ssum[k] = 0.0;
        uint32_t n = 0;
        for (uint64_t wa = w0; wa < w1; wa += Wt) {
            const uint32_t nw = (uint32_t)min((uint64_t)Wt, w1 - wa);
            const uint32_t per_plane = nw * ne, items = per_plane * p;
            __syncthreads();  // the previous tile is consumed
            for (uint32_t i0 = t; i0 < items; i0 += 4 * blockDim.x) { // four loads in flight before the first is stored
                double v[4];
                uint32_t dst[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const uint32_t i = i0 + u * blockDim.x;
                    if (i < items) {
                        const uint32_t q = i / per_plane, r = i % per_plane, w = r / ne, j = r % ne;
                        v[u] = __ldcs(src_plane[q] + (wa + w) * E + e0 + j);
                        dst[u] = (w * p + q) * Et + j;
                    }
                }
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (i0 + u * blockDim.x < items) xs[dst[u]] = v[u];
            }
            __syncthreads();
            for (uint32_t i = t; i < nw * ne; i += blockDim.x) {
                const uint32_t w = i / ne, j = i % ne;
                bool all = true;
                for (uint32_t q = 0; q < p; ++q) all &= fabs(xs[((uint64_t)w * p + q) * Et + j]) <= DBL_MAX;
                ok[w * Et + j] = all;
            }
            __syncthreads();
            if (active && el < ne) {
                for (uint32_t w = 0; w < nw; ++w) {
                    if (!ok[w * Et + el]) continue;
                    const double *x = xs + (uint64_t)w * p * Et + el;
                    double xa[4], xb[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        xa[k] = x[ia[k] * Et];
                        xb[k] = x[ib[k] * Et];
                    }
                    if (n == 0) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            K[k] = xa[k];
                            K[4 + k] = xb[k];
                        }
                    }
                    double ya[4], yb[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        ya[k] = xa[k] - K[k];
                        yb[k] = xb[k] - K[4 + k];
                        Ssum[k] += ya[k];
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) Q[i * 4 + j] = fma(ya[i], yb[j], Q[i * 4 + j]);
                    ++n;
                }
            }
        }
        // S_a of the column block comes from its diagonal tile
        __syncthreads();
        if (active && el < ne && diag)
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (4 * ab + k < p) ss[(4 * ab + k) * Et + el] = Ssum[k];
        __syncthreads();
        if (active && el < ne) {
            double *o = record(S, sl, fin ? nullptr : scratch, q, g, s, e0 + el);
            const double nan = __longlong_as_double(0x7ff8000000000000ll);
            const double dn = (double)n;
            if (tile == 0) o[0] = dn;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t a = 4 * ab + i;
                if (a >= p) continue;
                const double sa = Ssum[i];
                if (diag) o[1 + a] = n ? K[i] + sa / dn : (fin ? nan : 0.0);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t b = 4 * bb + j;
                    if (b >= p || (diag && j < i)) continue;
                    const double sb = diag ? Ssum[j] : ss[b * Et + el];
                    // as Shifted::group in stats_kernels.cu: one sum divided before the product (so it does not
                    // overflow where M is finite), the smaller first (so (a, b) and (b, a) get the same bits), and an
                    // overflowed Q_aa means M_aa at the top of the range
                    const double lo = fmin(sa, sb), hi = fmax(sa, sb);
                    double m = Q[i * 4 + j] - lo * (hi / dn);
                    if (a == b) m = Q[i * 4 + j] > DBL_MAX ? HUGE_VAL : fmax(m, 0.0);
                    if (!n) m = fin ? nan : 0.0;
                    o[1 + p + a * p + b] = m;
                    o[1 + p + b * p + a] = m;
                }
            }
        }
    }
}

// pass 2: thread = (group of the slice with C > 1, sample, entity, upper entry (a, b)) folds the group's C chunk
// records left to right
__global__ void __launch_bounds__(256) cov_merge_kernel(CovParams S, Slice sl, const double *scratch)
{
    const uint32_t p = S.n_p;
    const uint64_t U = (uint64_t)p * (p + 1) / 2, R = 1 + p + (uint64_t)p * p, SE = sl.ns * S.n_entities;
    const uint64_t n = (sl.g1 - sl.g0) * SE * U;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t g = sl.g0 + i / (SE * U), gl = i / U % SE;  // gl = (s - s0) * E + e
        const WorldGroup wg = sl.groups[g];
        if (wg.C == 1) continue;  // finished by pass 1
        uint32_t k = (uint32_t)(i % U), a = 0;
        while (k >= p - a) { k -= p - a; ++a; }
        const uint32_t b = a + k;
        CovEntry acc{0.0, 0.0, 0.0, 0.0};
        const double *r = scratch + ((wg.k0 - sl.k0) * SE + gl) * R;
        for (uint64_t c0 = 0; c0 < wg.C; c0 += kMergeBatch) { // the batch's loads are in flight before the first fold
            CovEntry v[kMergeBatch];
#pragma unroll
            for (unsigned u = 0; u < kMergeBatch; ++u) {
                v[u].n = 0.0;
                if (c0 + u < wg.C) {
                    const double *q = r + (c0 + u) * SE * R;
                    v[u] = CovEntry{q[0], q[1 + a], q[1 + b], q[1 + p + a * p + b]};
                }
            }
#pragma unroll
            for (unsigned u = 0; u < kMergeBatch; ++u) cov_merge(acc, v[u]);
        }
        const uint64_t s = sl.s0 + gl / S.n_entities, e = gl % S.n_entities;
        double *o = S.out + ((s * sl.G + g) * S.n_entities + e) * R;
        const bool any = acc.n > 0.0;
        if (a == 0 && b == 0) o[0] = acc.n;
        if (a == b) o[1 + a] = any ? acc.ma : nan;
        o[1 + p + a * p + b] = any ? acc.m : nan;
        o[1 + p + b * p + a] = any ? acc.m : nan;
    }
}

// Slices of groups and samples: consecutive groups while their chunks' partials for one sample fit in kScratchCap
// (counting every chunk of the slice's groups, as the scratch is indexed by chunk), then as many samples as fit; a
// slice whose groups all have one chunk needs no scratch and takes every sample.  With C > 1 (fewer than kChunkTasks
// entity tiles of kEntTile), one (group, sample)'s E * C partial records number at most kEntTile * 2 * kChunkTasks,
// which fit in kScratchCap at the largest record, so a slice always holds at least one group and one sample.  The
// one-group table gives the slices of whole samples the ungrouped call always had.
static_assert(kEntTile * 2 * kChunkTasks * (1 + B200_MAX_COV_PLANES + B200_MAX_COV_PLANES * B200_MAX_COV_PLANES) * 8 <= kScratchCap,
              "one sample's partials must fit in the scratch");
std::vector<Slice> cov_slices(const CovParams &S, const std::vector<WorldGroup> &table, uint64_t *scratch)
{
    std::vector<Slice> out;
    *scratch = 0;
    const uint64_t n_s = S.n_planes / S.planes_per_sample, G = table.size();
    const uint64_t per_chunk = S.n_entities * (1 + S.n_p + (uint64_t)S.n_p * S.n_p) * 8ull;  // bytes per chunk and sample
    for (uint64_t g0 = 0; g0 < G;) {
        uint64_t g1 = g0 + 1, chunks = table[g0].C;
        bool merge = table[g0].C > 1;
        while (g1 < G && (chunks + table[g1].C) * per_chunk <= kScratchCap) {
            chunks += table[g1].C;
            merge = merge || table[g1].C > 1;
            ++g1;
        }
        const uint64_t ns = merge ? std::max<uint64_t>(1, kScratchCap / (chunks * per_chunk)) : n_s;
        for (uint64_t s0 = 0; s0 < n_s; s0 += ns) {
            out.push_back(Slice{nullptr, G, g0, g1, table[g0].k0, chunks, s0, std::min(ns, n_s - s0)});
            if (merge) *scratch = std::max(*scratch, chunks * per_chunk * out.back().ns);
        }
        g0 = g1;
    }
    return out;
}

} // namespace

std::vector<WorldGroup> cov_group_table(const uint64_t *sizes, uint64_t n_groups, uint64_t n_entities)
{
    std::vector<WorldGroup> t(n_groups);
    uint64_t o = 0, k0 = 0;
    for (uint64_t g = 0; g < n_groups; ++g) {
        const Chunks ck = cov_chunks(sizes[g], n_entities);
        t[g] = {o, sizes[g], ck.Wc, ck.C, k0};
        o += sizes[g];
        k0 += ck.C;
    }
    return t;
}

uint64_t cov_scratch_bytes(const CovParams &S, const std::vector<WorldGroup> &table)
{
    uint64_t scratch = 0;
    if (S.n_planes && S.n_entities) cov_slices(S, table, &scratch);
    return scratch;
}

cudaError_t launch_covariance(const CovParams &S, const WorldGroup *groups, const std::vector<WorldGroup> &table,
                              void *scratch, int *launches, cudaStream_t s)
{
    *launches = 0;
    if (S.n_planes == 0 || S.n_entities == 0) return cudaSuccess;
    const Geo geo = cov_geo(S);
    const size_t smem = ((uint64_t)geo.Wt * S.n_p * geo.Et + (uint64_t)S.n_p * geo.Et) * 8 + (uint64_t)geo.Wt * geo.Et;
    cudaError_t e = cudaFuncSetAttribute(cov_chunk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const uint64_t cap = 64ull * kNumSMs * 8;
    uint64_t unused;
    for (Slice sl : cov_slices(S, table, &unused)) {
        sl.groups = groups;
        const uint64_t tasks = sl.ns * sl.K * ((S.n_entities + geo.Et - 1) / geo.Et);
        cov_chunk_kernel<<<(unsigned)std::min(tasks, cap), geo.threads, smem, s>>>(S, geo, sl, (double *)scratch);
        *launches += 1;
        bool merge = false;
        for (uint64_t g = sl.g0; g < sl.g1; ++g) merge = merge || table[g].C > 1;
        if (merge) {
            const uint64_t work = (sl.g1 - sl.g0) * sl.ns * S.n_entities * ((uint64_t)S.n_p * (S.n_p + 1) / 2);
            cov_merge_kernel<<<(unsigned)std::min((work + 255) / 256, cap), 256, 0, s>>>(S, sl, (const double *)scratch);
            *launches += 1;
        }
    }
    return cudaGetLastError();
}

} // namespace b200
