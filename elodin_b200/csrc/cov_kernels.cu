// Ensemble covariance over the world axis: for every (sample, entity) one record (n, mean[p], M[p][p]) over the worlds
// whose p selected values are all finite (include/b200_sixdof.h b200_sixdof_trajectory_covariance / _state_covariance).
//
// Shape of the reduction.  The worlds are cut into C chunks of Wc consecutive worlds; Wc and C depend on (n_worlds,
// n_entities) alone.  A block reduces one chunk of one sample for a tile of Et entities: it stages Wt worlds x p planes x
// Et entities at a time in shared memory (lanes read consecutive doubles of one plane: entities, then worlds when the
// tile is every entity), marks the complete worlds, then thread (entity, tile) accumulates a 4 x 4 register tile of the
// upper triangle of M over the chunk's complete worlds in world order.  Shift: K = the chunk's first complete world's
// row, y = x - K, sums S_a = sum y_a (diagonal tiles) and Q_ab = sum y_a y_b (fma); the chunk's record is
// mean_a = K_a + S_a / n, M_ab = Q_ab - lo (hi / n) with (lo, hi) = (min, max)(S_a, S_b), and M_aa = +inf where Q_aa overflowed.  Each entry is a sequential sum over the same worlds whatever the
// selection, the entity tile or the other planes, so an entry has the same bits in any selection with the same complete
// worlds.  With C > 1 a second launch merges the chunk records left to right with cov_merge, one thread per (group,
// upper entry).  The partials live in scratch; groups run in slices that keep it under kScratchCap.  No atomics.
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

// A slice of the groups: samples [s0, s0 + ns) x entities [e0, e0 + ne) (every entity, e0 = 0); local group
// gl = (s - s0) * ne + (e - e0)
struct Slice {
    uint64_t s0, ns, e0, ne;
};

__device__ inline double *record(const CovParams &S, const Slice &sl, double *scratch, uint64_t c, uint64_t s, uint64_t e)
{
    const uint64_t R = 1 + S.n_p + (uint64_t)S.n_p * S.n_p;
    if (scratch) return scratch + (c * sl.ns * sl.ne + (s - sl.s0) * sl.ne + (e - sl.e0)) * R;
    return S.out + (s * S.n_entities + e) * R;
}

__device__ inline void tile_of(uint32_t t, uint32_t nb, uint32_t &ab, uint32_t &bb)
{
    ab = 0;
    while (t >= nb - ab) { t -= nb - ab; ++ab; }
    bb = ab + t;
}

// pass 1: task = (sample s of the slice, chunk c, entity tile) -> the chunk's record per entity: final (NaN where
// n = 0) when C = 1, else a partial record in scratch
__global__ void __launch_bounds__(kMaxThreads) cov_chunk_kernel(CovParams S, Chunks ck, Geo geo, Slice sl, double *scratch)
{
    extern __shared__ double smem[];
    const uint32_t p = S.n_p, Et = geo.Et, Wt = geo.Wt;
    double *xs = smem;                                    // [Wt][p][Et]
    double *ss = xs + (uint64_t)Wt * p * Et;              // [p][Et]: the diagonal tiles' S_a
    unsigned char *ok = (unsigned char *)(ss + p * Et);   // [Wt][Et]
    const uint64_t E = S.n_entities;
    const uint64_t n_et = (sl.ne + Et - 1) / Et;
    const uint64_t n_tasks = sl.ns * ck.C * n_et;
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
        const uint64_t et = task % n_et, c = (task / n_et) % ck.C, s = sl.s0 + task / (n_et * ck.C);
        const uint64_t e0 = sl.e0 + et * Et;
        const uint32_t ne = (uint32_t)min((uint64_t)Et, sl.e0 + sl.ne - e0);
        const uint64_t w0 = c * ck.Wc, w1 = min(w0 + ck.Wc, S.n_worlds);
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
                        const double *src = stats_plane(S, s * S.planes_per_sample + S.planes[q]);
                        v[u] = __ldcs(src + (wa + w) * E + e0 + j);
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
            double *o = record(S, sl, ck.C > 1 ? scratch : nullptr, c, s, e0 + el);
            const double nan = __longlong_as_double(0x7ff8000000000000ll);
            const bool fin = ck.C == 1;  // a final record holds NaN where n = 0; a partial leaves them (unread)
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

// pass 2 (C > 1): thread = (group of the slice, upper entry (a, b)) folds the C chunk records left to right
__global__ void __launch_bounds__(256) cov_merge_kernel(CovParams S, Chunks ck, Slice sl, const double *scratch)
{
    const uint32_t p = S.n_p;
    const uint64_t U = (uint64_t)p * (p + 1) / 2, R = 1 + p + (uint64_t)p * p, Gs = sl.ns * sl.ne;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < Gs * U; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t gl = i / U;
        uint32_t k = (uint32_t)(i % U), a = 0;
        while (k >= p - a) { k -= p - a; ++a; }
        const uint32_t b = a + k;
        CovEntry acc{0.0, 0.0, 0.0, 0.0};
        const double *r = scratch + gl * R;
        for (uint64_t c0 = 0; c0 < ck.C; c0 += kMergeBatch) { // the batch's loads are in flight before the first fold
            CovEntry v[kMergeBatch];
#pragma unroll
            for (unsigned u = 0; u < kMergeBatch; ++u) {
                v[u].n = 0.0;
                if (c0 + u < ck.C) {
                    const double *q = r + (c0 + u) * Gs * R;
                    v[u] = CovEntry{q[0], q[1 + a], q[1 + b], q[1 + p + a * p + b]};
                }
            }
#pragma unroll
            for (unsigned u = 0; u < kMergeBatch; ++u) cov_merge(acc, v[u]);
        }
        const uint64_t s = sl.s0 + gl / sl.ne, e = sl.e0 + gl % sl.ne;
        double *o = S.out + (s * S.n_entities + e) * R;
        const bool any = acc.n > 0.0;
        if (a == 0 && b == 0) o[0] = acc.n;
        if (a == b) o[1 + a] = any ? acc.ma : nan;
        o[1 + p + a * p + b] = any ? acc.m : nan;
        o[1 + p + b * p + a] = any ? acc.m : nan;
    }
}

inline uint64_t partial_bytes(const CovParams &S, const Chunks &ck)
{
    return ck.C > 1 ? ck.C * (1 + S.n_p + (uint64_t)S.n_p * S.n_p) * 8ull : 0;
}

// Slices are whole samples: with C > 1 (fewer than kChunkTasks entity tiles of kEntTile), a sample's E * C partial
// records number at most kEntTile * 2 * kChunkTasks, which fit in kScratchCap at the largest record.
static_assert(kEntTile * 2 * kChunkTasks * (1 + B200_MAX_COV_PLANES + B200_MAX_COV_PLANES * B200_MAX_COV_PLANES) * 8 <= kScratchCap,
              "one sample's partials must fit in the scratch");
inline Slice slice_shape(const CovParams &S, const Chunks &ck)
{
    const uint64_t per = partial_bytes(S, ck);
    const uint64_t G = per ? kScratchCap / per : ~0ull;
    return Slice{0, std::max<uint64_t>(1, G / S.n_entities), 0, S.n_entities};
}

} // namespace

uint64_t cov_scratch_bytes(const CovParams &S)
{
    const uint64_t n_s = S.n_planes / S.planes_per_sample;
    if (n_s == 0 || S.n_worlds == 0 || S.n_entities == 0) return 0;
    const Chunks ck = cov_chunks(S.n_worlds, S.n_entities);
    const Slice sh = slice_shape(S, ck);
    return std::min(sh.ns, n_s) * sh.ne * partial_bytes(S, ck);
}

cudaError_t launch_covariance(const CovParams &S, void *scratch, int *launches, cudaStream_t s)
{
    *launches = 0;
    const uint64_t n_s = S.n_planes / S.planes_per_sample;
    if (n_s == 0 || S.n_worlds == 0 || S.n_entities == 0) return cudaSuccess;
    const Chunks ck = cov_chunks(S.n_worlds, S.n_entities);
    const Geo geo = cov_geo(S);
    const size_t smem = ((uint64_t)geo.Wt * S.n_p * geo.Et + (uint64_t)S.n_p * geo.Et) * 8 + (uint64_t)geo.Wt * geo.Et;
    cudaError_t e = cudaFuncSetAttribute(cov_chunk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const Slice sh = slice_shape(S, ck);
    const uint64_t cap = 64ull * kNumSMs * 8;
    for (uint64_t s0 = 0; s0 < n_s; s0 += sh.ns) {
        const Slice sl{s0, std::min(sh.ns, n_s - s0), 0, S.n_entities};
        const uint64_t tasks = sl.ns * ck.C * ((sl.ne + geo.Et - 1) / geo.Et);
        cov_chunk_kernel<<<(unsigned)std::min(tasks, cap), geo.threads, smem, s>>>(S, ck, geo, sl, (double *)scratch);
        *launches += 1;
        if (ck.C > 1) {
            const uint64_t work = sl.ns * sl.ne * ((uint64_t)S.n_p * (S.n_p + 1) / 2);
            cov_merge_kernel<<<(unsigned)std::min((work + 255) / 256, cap), 256, 0, s>>>(S, ck, sl, (const double *)scratch);
            *launches += 1;
        }
    }
    return cudaGetLastError();
}

} // namespace b200
