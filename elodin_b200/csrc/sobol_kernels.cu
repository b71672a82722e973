// Variance-based (Sobol) sensitivity of the outcomes of a Saltelli campaign (include/b200_sixdof.h
// b200_sixdof_outcome_sobol): the derived planes of every selected outcome, the complete-sample lists and the
// bootstrap of the first-order and total indices.  The point estimates come from the covariance kernels (cov_kernels.cu,
// unchanged) over the derived planes; this file only forms them and the bootstrap spread.
//
//  - Plane pass.  A block of kTile samples of one output stages the kTile (d + 2) consecutive worlds of the outcome
//    plane in shared memory (consecutive threads load consecutive worlds), then thread j forms sample j's planes
//    a = f(A), b = f(B), D_i = f(AB^(i)) - f(A) (__dsub_rn) and its completeness byte.
//  - Compaction.  One block per task (group, output) walks the group's completeness bytes in order and writes the
//    indices of its complete samples (relative to the group's first sample) into the output's list; the count goes to
//    scratch.  Ballots and a fixed warp scan: the list is in sample order whatever the launch.
//  - Bootstrap.  A block per item (task, resample r), items of a task adjacent in launch order, so a task's planes stay
//    in L2 while its resamples run.  Thread t of the block takes draws t, t + kBootThreads, ..; each draw's sample is
//    c[umulhi64(x, n)] with x the SplitMix64 output of the stream below.  The sums of the draws, shifted by the point
//    record's means, are reduced by a fixed shuffle tree and a fixed sum over the warps: no atomics, so the same bits on
//    every call.  The 4 + 3d sums are kept for kInChunk inputs at a time (the draws are replayed per chunk), so no
//    accumulator leaves the registers at d = 23.
//  - Finish.  A thread per (task, input) forms the point S1 and ST from the covariance record with correctly rounded
//    operations in the header's order (numpy's bits), and the standard deviation of the finite resample indices.
// Scratch (after the covariance table, which the caller puts first): per slice of tasks, a count per task and the
// resample records [V, S1[d], ST[d]]; slices keep it under kScratchCap and change no bits.
#include <algorithm>
#include <cfloat>

#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kTile = 128;          // samples per block of the plane pass
constexpr unsigned kScanThreads = 1024;  // compaction block
constexpr unsigned kBootThreads = 256;   // bootstrap block
constexpr unsigned kInChunk = 8;         // inputs whose sums a bootstrap pass keeps in registers
constexpr unsigned kFinThreads = 128;
constexpr uint64_t kScratchCap = 256ull << 20;
constexpr unsigned kSums = 4 + 3 * kInChunk;  // Sa, Saa, Sb, Sbb, then SD, SDD, SbD per input of the chunk

__device__ inline double nan_value() { return __longlong_as_double(0x7ff8000000000000ll); }

__device__ inline const double *sobol_plane(const SobolParams &S, uint32_t k, uint32_t j)
{
    return S.sp + ((uint64_t)k * (S.d + 2) + j) * S.ld;
}

// SplitMix64's output function
__device__ inline uint64_t mix64(uint64_t z)
{
    z ^= z >> 30;
    z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27;
    z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}

// grid (sample tile, output): the derived planes and completeness bytes of kTile samples of output k
__global__ void __launch_bounds__(kTile) sobol_plane_kernel(SobolParams S)
{
    __shared__ double ys[kTile * (B200_MAX_SOBOL_INPUTS + 2)];
    const uint32_t q = S.d + 2, k = blockIdx.y;
    const uint64_t s0 = (uint64_t)blockIdx.x * kTile;
    const uint32_t ns = (uint32_t)min((uint64_t)kTile, S.n_samples - s0);
    const double *src = S.planes + (uint64_t)S.plane[k] * S.ld_o + s0 * q;
    for (uint32_t i = threadIdx.x; i < ns * q; i += kTile) ys[i] = src[i];
    __syncthreads();
    const uint32_t j = threadIdx.x;
    if (j >= ns) return;
    const double *y = ys + j * q;
    const double a = y[0], b = y[q - 1];
    bool ok = fabs(a) <= DBL_MAX && fabs(b) <= DBL_MAX;
    for (uint32_t i = 0; i < S.d; ++i) ok &= fabs(__dsub_rn(y[1 + i], a)) <= DBL_MAX;
    const double nan = nan_value();
    const uint64_t s = s0 + j;
    double *out = S.sp + (uint64_t)k * q * S.ld + s;
    out[0] = ok ? a : nan;
    out[S.ld] = ok ? b : nan;
    for (uint32_t i = 0; i < S.d; ++i) out[(2 + i) * S.ld] = ok ? __dsub_rn(y[1 + i], a) : nan;
    S.mask[(uint64_t)k * S.ld + s] = ok;
}

// block = task t0 + blockIdx.x: the complete samples of its group in its output's list, their count in n_complete
__global__ void __launch_bounds__(kScanThreads) sobol_list_kernel(SobolParams S, const WorldGroup *groups, uint64_t t0,
                                                                  uint64_t *n_complete)
{
    __shared__ uint32_t warp_base[kScanThreads / 32 + 1];
    const uint64_t t = t0 + blockIdx.x, g = t / S.n_p;
    const uint32_t k = (uint32_t)(t % S.n_p), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const WorldGroup wg = groups[g];
    const uint8_t *m = S.mask + (uint64_t)k * S.ld + wg.o;
    uint32_t *list = S.list + (uint64_t)k * S.ld + wg.o;
    uint64_t running = 0;
    for (uint64_t base = 0; base < wg.n; base += kScanThreads) {
        const uint64_t i = base + threadIdx.x;
        const bool f = i < wg.n && m[i];
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (lane == 0) warp_base[warp] = __popc(bal);
        __syncthreads();
        if (warp == 0) {
            const uint32_t c = warp_base[lane];
            uint32_t x = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= (unsigned)o) x += y;
            }
            warp_base[lane] = x - c;  // exclusive
            if (lane == 31) warp_base[32] = x;
        }
        __syncthreads();
        if (f) list[running + warp_base[warp] + __popc(bal & ((1u << lane) - 1u))] = (uint32_t)i;
        running += warp_base[32];
        __syncthreads();  // warp_base is rewritten by the next chunk
    }
    if (threadIdx.x == 0) n_complete[blockIdx.x] = running;
}

__device__ inline double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// block per item (task t0 + item / B, resample item % B): the resample's V, S1[d] and ST[d] into its scratch record
__global__ void __launch_bounds__(kBootThreads) sobol_boot_kernel(SobolParams S, const double *cov, uint64_t G,
                                                                  const WorldGroup *groups, uint64_t t0, uint64_t n_tasks,
                                                                  uint32_t B, uint64_t seed, const uint64_t *n_complete,
                                                                  double *res)
{
    __shared__ double part[kSums][kBootThreads / 32];
    __shared__ double tot[kSums];
    const uint32_t d = S.d, q = d + 2, R = 1 + q + q * q;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double nan = nan_value();
    for (uint64_t item = blockIdx.x; item < n_tasks * B; item += gridDim.x) {
        const uint64_t tl = item / B, r = item % B, t = t0 + tl, g = t / S.n_p;
        const uint32_t k = (uint32_t)(t % S.n_p);
        const uint64_t n = n_complete[tl], o = groups[g].o;
        const double *rec = cov + ((uint64_t)k * G + g) * R;  // the point record: sample axis = output k
        const double ma = rec[1], mb = rec[2];
        const uint32_t *list = S.list + (uint64_t)k * S.ld + o;
        const double *pa = sobol_plane(S, k, 0) + o, *pb = sobol_plane(S, k, 1) + o;
        double *out = res + item * (1 + 2ull * d);
        const double fn = (double)n;
        for (uint32_t c0 = 0; c0 < d; c0 += kInChunk) {
            const uint32_t nc = min(kInChunk, d - c0);
            double acc[kSums], md[kInChunk];
            const double *pd[kInChunk];
#pragma unroll
            for (unsigned u = 0; u < kSums; ++u) acc[u] = 0.0;
#pragma unroll
            for (unsigned i = 0; i < kInChunk; ++i) {
                md[i] = i < nc ? rec[3 + c0 + i] : 0.0;
                pd[i] = sobol_plane(S, k, 2 + c0 + min(i, nc - 1)) + o;
            }
            for (uint64_t dr = threadIdx.x; dr < n; dr += kBootThreads) {
                const uint64_t x = mix64(seed + 0x9E3779B97F4A7C15ull * ((r << 32) + dr + 1));
                const uint32_t j = list[__umul64hi(x, n)];
                const double a = pa[j] - ma, b = pb[j] - mb;
                acc[0] += a;
                acc[1] = fma(a, a, acc[1]);
                acc[2] += b;
                acc[3] = fma(b, b, acc[3]);
#pragma unroll
                for (unsigned i = 0; i < kInChunk; ++i) {
                    if (i < nc) {
                        const double v = pd[i][j] - md[i];
                        acc[4 + 3 * i] += v;
                        acc[5 + 3 * i] = fma(v, v, acc[5 + 3 * i]);
                        acc[6 + 3 * i] = fma(b, v, acc[6 + 3 * i]);
                    }
                }
            }
#pragma unroll
            for (unsigned u = 0; u < kSums; ++u) {
                const double v = warp_sum(acc[u]);
                if (lane == 0) part[u][warp] = v;
            }
            __syncthreads();
            if (threadIdx.x < kSums) {
                double v = 0.0;
                for (unsigned w = 0; w < kBootThreads / 32; ++w) v += part[threadIdx.x][w];
                tot[threadIdx.x] = v;
            }
            __syncthreads();
            // the pooled variance of [a; b] and the estimators of the resample, from the shifted sums
            const double ea = tot[0] / fn, eb = tot[2] / fn;
            const double va = tot[1] / fn - ea * ea, vb = tot[3] / fn - eb * eb;
            const double dm = (ma + ea) - (mb + eb);
            const double V = (va + vb) * 0.5 + dm * dm * 0.25;
            const bool ok = n >= 2 && V > 0.0;
            if (threadIdx.x == 0 && c0 == 0) out[0] = n ? V : nan;
            if (threadIdx.x < nc) {
                const unsigned i = threadIdx.x;
                const double mD = rec[3 + c0 + i];
                const double eD = tot[4 + 3 * i] / fn;
                const double EbD = tot[6 + 3 * i] / fn + mb * eD + mD * eb + mb * mD;
                const double EDD = tot[5 + 3 * i] / fn + 2.0 * mD * eD + mD * mD;
                out[1 + c0 + i] = ok ? EbD / V : nan;
                out[1 + d + c0 + i] = ok ? EDD / (2.0 * V) : nan;
            }
            __syncthreads();  // part and tot are rewritten by the next chunk or item
        }
    }
}

// the sample standard deviation (ddof 1) of the finite x[0], x[stride], .. x[(B - 1) stride]; NaN below 2
__device__ inline double finite_sd(const double *x, uint32_t B, uint64_t stride)
{
    double s = 0.0;
    uint32_t c = 0;
    for (uint32_t r = 0; r < B; ++r) {
        const double v = x[r * stride];
        if (fabs(v) <= DBL_MAX) {
            s += v;
            ++c;
        }
    }
    if (c < 2) return nan_value();
    const double m = s / c;
    double ss = 0.0;
    for (uint32_t r = 0; r < B; ++r) {
        const double v = x[r * stride];
        if (fabs(v) <= DBL_MAX) ss += (v - m) * (v - m);
    }
    return sqrt(ss / (c - 1));
}

// thread per (task t0 + i / d, input i % d): the task's record [n, V, n_boot_ok, S1[d], ST[d], S1_sd[d], ST_sd[d]]
__global__ void __launch_bounds__(kFinThreads) sobol_finish_kernel(SobolParams S, const double *cov, uint64_t G,
                                                                   uint64_t t0, uint64_t n_tasks, uint32_t B,
                                                                   const double *res, double *out)
{
    const uint32_t d = S.d, q = d + 2, R = 1 + q + q * q;
    const uint64_t L = 1 + 2ull * d;
    const double nan = nan_value();
    for (uint64_t x = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; x < n_tasks * d;
         x += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t tl = x / d, t = t0 + tl, g = t / S.n_p;
        const uint32_t k = (uint32_t)(t % S.n_p), i = (uint32_t)(x % d);
        const double *rec = cov + ((uint64_t)k * G + g) * R;
        const double *m = rec + 1, *M = rec + 1 + q;
        const double n = rec[0];
        // include/b200_sixdof.h: V, EbD, EDD in this order, each operation correctly rounded
        const double dab = __dsub_rn(m[0], m[1]);
        const double V = __dadd_rn(__ddiv_rn(__dadd_rn(M[0], M[q + 1]), __dmul_rn(2.0, n)),
                                   __dmul_rn(__dmul_rn(dab, dab), 0.25));
        const uint32_t c = 2 + i;
        const double EbD = __dadd_rn(__ddiv_rn(M[1 * q + c], n), __dmul_rn(m[1], m[c]));
        const double EDD = __dadd_rn(__ddiv_rn(M[c * q + c], n), __dmul_rn(m[c], m[c]));
        const bool ok = n >= 2.0 && V > 0.0;
        double *o = out + t * (3 + 4ull * d);
        o[3 + i] = ok ? __ddiv_rn(EbD, V) : nan;
        o[3 + d + i] = ok ? __ddiv_rn(EDD, __dmul_rn(2.0, V)) : nan;
        const double *rr = res + tl * B * L;
        o[3 + 2 * d + i] = B ? finite_sd(rr + 1 + i, B, L) : nan;
        o[3 + 3 * d + i] = B ? finite_sd(rr + 1 + d + i, B, L) : nan;
        if (i == 0) {
            uint32_t good = 0;
            for (uint32_t r = 0; r < B; ++r) good += rr[r * L] > 0.0;
            o[0] = n;
            o[1] = n >= 2.0 ? V : nan;
            o[2] = (double)good;
        }
    }
}

// tasks per slice of the bootstrap's scratch: at least one
inline uint64_t slice_tasks(const SobolParams &S, uint64_t tasks, uint32_t B)
{
    const uint64_t per = 8 + (uint64_t)B * (1 + 2ull * S.d) * 8;
    return std::max<uint64_t>(1, std::min(tasks, kScratchCap / per));
}

} // namespace

uint64_t sobol_scratch_bytes(const SobolParams &S, uint64_t tasks, uint32_t n_boot)
{
    if (!tasks) return 0;
    const uint64_t nt = slice_tasks(S, tasks, n_boot);
    return nt * 8 + nt * (uint64_t)n_boot * (1 + 2ull * S.d) * 8;
}

cudaError_t launch_sobol_planes(const SobolParams &S, int *launches, cudaStream_t s)
{
    *launches = 0;
    if (S.n_samples == 0) return cudaSuccess;
    const dim3 grid((unsigned)((S.n_samples + kTile - 1) / kTile), S.n_p);
    sobol_plane_kernel<<<grid, kTile, 0, s>>>(S);
    *launches = 1;
    return cudaGetLastError();
}

cudaError_t launch_sobol_indices(const SobolParams &S, const double *cov, const WorldGroup *groups, uint64_t G,
                                 uint32_t n_boot, uint64_t seed, double *out, void *scratch, int *launches,
                                 cudaStream_t s)
{
    *launches = 0;
    const uint64_t tasks = G * S.n_p;
    if (!tasks) return cudaSuccess;
    const uint64_t nt = slice_tasks(S, tasks, n_boot);
    uint64_t *n_complete = (uint64_t *)scratch;
    double *res = (double *)scratch + nt;
    const uint64_t cap = 64ull * kNumSMs;
    for (uint64_t t0 = 0; t0 < tasks; t0 += nt) {
        const uint64_t n = std::min(nt, tasks - t0);
        if (n_boot) {
            sobol_list_kernel<<<(unsigned)n, kScanThreads, 0, s>>>(S, groups, t0, n_complete);
            const uint64_t items = n * n_boot;
            sobol_boot_kernel<<<(unsigned)std::min<uint64_t>(items, 64ull * kNumSMs), kBootThreads, 0, s>>>(
                S, cov, G, groups, t0, n, n_boot, seed, n_complete, res);
            *launches += 2;
        }
        const uint64_t work = n * S.d;
        sobol_finish_kernel<<<(unsigned)std::min((work + kFinThreads - 1) / kFinThreads, cap), kFinThreads, 0, s>>>(
            S, cov, G, t0, n, n_boot, res, out);
        *launches += 1;
    }
    return cudaGetLastError();
}

} // namespace b200
