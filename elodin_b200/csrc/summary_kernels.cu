// Run summaries over the time axis: per (world, entity, plane) extrema and per (world, threshold) first events
// (include/b200_sixdof.h b200_sixdof_summary_*).
//
// Shape of a fold.  Rows are SoA planes (the trajectory ring [samples][25][ld], or the state columns, then the channel
// planes of sixdof_abi.cu:ensemble_rows), so a thread owns
// one (body, plane): block (x, y) takes 256 consecutive bodies of plane planes[y], and every thread walks the fold's rows
// in order, one coalesced double per row, four loads in flight.  The thread's accumulators (5 extrema planes of ld,
// and the tick of each threshold on its (entity, plane)) are read once before the walk and written once after it; a
// threshold that fires inside the fold then has its 25 planes at that row copied by the same thread.  Each accumulator
// has exactly one owner, so there are no atomics, and the updates are order-free (strict comparisons, ties to the
// smaller tick): the result depends only on the set of rows folded.
#include <algorithm>
#include <cfloat>

#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kSumThreads = 256;
constexpr uint32_t kThrFields = 26;  // tick + 25 planes

__device__ __forceinline__ double nan_value() { return __longlong_as_double(0x7ff8000000000000ll); }

// 4 blocks per SM: 64 registers, no spills (without the bound ptxas also settles on 64, but spills the prologue)
__global__ void __launch_bounds__(kSumThreads, 4) summary_fold_kernel(const __grid_constant__ SummaryParams S)
{
    const uint64_t b = (uint64_t)blockIdx.x * kSumThreads + threadIdx.x;
    if (b >= S.n_bodies) return;
    const uint32_t p = S.planes[blockIdx.y];
    const uint32_t e = (uint32_t)(b % S.n_entities);
    const uint64_t w = b / S.n_entities;
    uint32_t mine = 0; // thresholds on this thread's (entity, plane)
#pragma unroll
    for (uint32_t i = 0; i < B200_MAX_THRESHOLDS; ++i)
        if (i < S.n_thr && S.t[i].entity == e && S.t[i].plane == p) mine |= 1u << i;
    const bool ext = S.ext != nullptr;
    if (!ext && !mine) return;

    double mn = 0.0, mx = 0.0, mn_t = -1.0, mx_t = -1.0, nf_t = -1.0;
    double *a = ext ? S.ext + (uint64_t)p * 5 * S.ld + b : nullptr;
    if (ext) {
        mn = a[0];
        mx = a[S.ld];
        mn_t = a[2 * S.ld];
        mx_t = a[3 * S.ld];
        nf_t = a[4 * S.ld];
    }
    double best[B200_MAX_THRESHOLDS]; // tick of the first firing row so far, -1 = none
    uint32_t at[B200_MAX_THRESHOLDS]; // its row in this fold, ~0 = not in this fold
#pragma unroll
    for (uint32_t i = 0; i < B200_MAX_THRESHOLDS; ++i) {
        best[i] = (mine >> i) & 1u ? S.thr[(w * S.n_thr + i) * kThrFields] : -1.0;
        at[i] = ~0u;
    }
    auto fold = [&](double x, uint64_t r) {
        const double t = (double)(S.tick0 + r * S.tick_step);
        if (ext) {
            if (fabs(x) <= DBL_MAX) {
                if (mn_t < 0.0 || x < mn || (x == mn && t < mn_t)) { mn = x; mn_t = t; }
                if (mx_t < 0.0 || x > mx || (x == mx && t < mx_t)) { mx = x; mx_t = t; }
            } else if (nf_t < 0.0 || t < nf_t) {
                nf_t = t;
            }
        }
#pragma unroll
        for (uint32_t i = 0; i < B200_MAX_THRESHOLDS; ++i) {
            if ((mine >> i) & 1u) {
                const bool fire = S.t[i].above ? x > S.t[i].value : x < S.t[i].value; // NaN never fires
                if (fire && (best[i] < 0.0 || t < best[i])) { best[i] = t; at[i] = (uint32_t)r; }
            }
        }
    };
    const double *src = S.row[p] + b;
    const uint64_t st = p < 25 ? S.row_stride : S.chan_stride;
    uint64_t r = 0;
    for (; r + 4 <= S.n_rows; r += 4) { // four loads in flight before the first is used
        const double x0 = __ldcs(src + r * st), x1 = __ldcs(src + (r + 1) * st), x2 = __ldcs(src + (r + 2) * st),
                     x3 = __ldcs(src + (r + 3) * st);
        fold(x0, r);
        fold(x1, r + 1);
        fold(x2, r + 2);
        fold(x3, r + 3);
    }
    for (; r < S.n_rows; ++r) fold(__ldcs(src + r * st), r);

    if (ext) {
        a[0] = mn;
        a[S.ld] = mx;
        a[2 * S.ld] = mn_t;
        a[3 * S.ld] = mx_t;
        a[4 * S.ld] = nf_t;
    }
#pragma unroll
    for (uint32_t i = 0; i < B200_MAX_THRESHOLDS; ++i) {
        if (at[i] != ~0u) { // fired inside this fold, earlier than anything folded before: capture the row
            double *o = S.thr + (w * S.n_thr + i) * kThrFields;
            const uint64_t off = (uint64_t)at[i] * S.row_stride + b;
            o[0] = best[i];
#pragma unroll
            for (uint32_t j = 0; j < 25; ++j) o[1 + j] = S.row[j][off];
        }
    }
}

// extrema planes: min, max = NaN, the three ticks = -1; threshold table: tick = -1, planes = NaN
__global__ void __launch_bounds__(kSumThreads) summary_clear_kernel(double *ext, uint64_t ld, uint32_t R, double *thr,
                                                                    uint64_t thr_len)
{
    const uint64_t ext_len = ext ? 5ull * R * ld : 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < ext_len + thr_len; i += (uint64_t)gridDim.x * blockDim.x) {
        if (i < ext_len) ext[i] = (i / ld) % 5 < 2 ? nan_value() : -1.0;
        else thr[i - ext_len] = (i - ext_len) % kThrFields == 0 ? -1.0 : nan_value();
    }
}

__global__ void __launch_bounds__(kSumThreads) extrema_table_kernel(const double *__restrict__ ext, uint64_t ld, uint32_t R,
                                                                    uint64_t b0, uint64_t nb, double *__restrict__ out)
{
    const uint64_t F = 5ull * R;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nb * F; i += (uint64_t)gridDim.x * blockDim.x)
        out[i] = ext[(i % F) * ld + b0 + i / F];
}

} // namespace

cudaError_t launch_summary_clear(const SummaryParams &S, int *launches, cudaStream_t s)
{
    *launches = 0;
    const uint64_t ext_len = S.ext ? 5ull * S.width * S.ld : 0;
    const uint64_t thr_len = (S.thr && S.n_entities) ? S.n_bodies / S.n_entities * S.n_thr * kThrFields : 0;
    if (ext_len + thr_len == 0) return cudaSuccess;
    const uint64_t blocks = std::min<uint64_t>((ext_len + thr_len + kSumThreads - 1) / kSumThreads, 64ull * kNumSMs * 8);
    summary_clear_kernel<<<(unsigned)blocks, kSumThreads, 0, s>>>(S.ext, S.ld, S.width, S.thr, thr_len);
    *launches = 1;
    return cudaGetLastError();
}

cudaError_t launch_summary_fold(const SummaryParams &S, int *launches, cudaStream_t s)
{
    *launches = 0;
    if (S.n_rows == 0 || S.n_bodies == 0 || S.n_planes == 0) return cudaSuccess;
    const dim3 grid((unsigned)((S.n_bodies + kSumThreads - 1) / kSumThreads), S.n_planes);
    summary_fold_kernel<<<grid, kSumThreads, 0, s>>>(S);
    *launches = 1;
    return cudaGetLastError();
}

cudaError_t launch_extrema_table(const double *ext, uint64_t ld, uint32_t R, uint64_t b0, uint64_t nb, double *out,
                                 cudaStream_t s)
{
    if (nb == 0) return cudaSuccess;
    const uint64_t blocks = std::min<uint64_t>((nb * 5 * R + kSumThreads - 1) / kSumThreads, 64ull * kNumSMs * 8);
    extrema_table_kernel<<<(unsigned)blocks, kSumThreads, 0, s>>>(ext, ld, R, b0, nb, out);
    return cudaGetLastError();
}

} // namespace b200
