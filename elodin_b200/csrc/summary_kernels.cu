// Run summaries over the time axis: per (world, entity, plane) extrema and moments, per (world, threshold) first events
// and per (world, dwell) counts of rows beyond a bound (include/b200_sixdof.h b200_sixdof_summary_*).
//
// Shape of a fold.  Rows are SoA planes (the trajectory ring [samples][25][ld], or the state columns, then the channel
// planes of sixdof_abi.cu:ensemble_rows), so a thread owns
// one (body, plane): block (x, y) takes 256 consecutive bodies of plane planes[y], and every thread walks the fold's rows
// in order, one coalesced double per row, four loads in flight.  The thread's accumulators (5 extrema planes of ld,
// and the tick of each threshold on its (entity, plane)) are read once before the walk and written once after it; a
// threshold that fires inside the fold then has its 25 planes at that row copied by the same thread.  Each accumulator
// has exactly one owner, so there are no atomics, and the updates are order-free (strict comparisons, ties to the
// smaller tick): the result depends only on the set of rows folded.
//
// Moments and dwells are the kScores instantiation of the same fold: the owner of (body, plane) also keeps the moment
// accumulator of that plane (read before the walk, written after it) and the dwells on its (entity, plane), counted in
// registers as rows of this fold and added to the record once after the walk.  The moment sums are sequential in the
// order the rows are folded, so their bits depend on that sequence (not on how it is cut into folds); the dwell counts
// are integers.  Without moments and dwells the launch takes the kScores = false instantiation, which is the extrema /
// threshold fold alone with its own register budget.
#include <algorithm>
#include <cfloat>

#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kSumThreads = 256;
constexpr uint32_t kThrFields = 26;  // tick + 25 planes

__device__ __forceinline__ double nan_value() { return __longlong_as_double(0x7ff8000000000000ll); }

// kScores = false, 4 blocks per SM: 64 registers, no spills (without the bound ptxas also settles on 64, but spills the
// prologue).  kScores = true, 2 blocks per SM: the 8 dwell counters and the moment sums need more than 64.
template <bool kScores>
__global__ void __launch_bounds__(kSumThreads, kScores ? 2 : 4) summary_fold_kernel(const __grid_constant__ SummaryParams S)
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
    uint32_t dmine = 0; // dwells on this thread's (entity, plane)
    const uint32_t slot = kScores ? S.mom_slot[blockIdx.y] : kNoMoment;
    if constexpr (kScores) {
#pragma unroll
        for (uint32_t i = 0; i < B200_MAX_DWELLS; ++i)
            if (i < S.n_dwell && S.d[i].entity == e && S.d[i].plane == p) dmine |= 1u << i;
    }
    if (!ext && !mine && !dmine && slot == kNoMoment) return;

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
    double n = 0.0, K = 0.0, S1 = 0.0, S2 = 0.0;
    double *m = slot != kNoMoment ? S.mom + (uint64_t)slot * 4 * S.ld + b : nullptr;
    if (m) {
        n = m[0];
        K = m[S.ld];
        S1 = m[2 * S.ld];
        S2 = m[3 * S.ld];
    }
    uint32_t cnt[B200_MAX_DWELLS], first[B200_MAX_DWELLS], last[B200_MAX_DWELLS]; // rows of this fold
#pragma unroll
    for (uint32_t i = 0; i < B200_MAX_DWELLS; ++i) cnt[i] = first[i] = last[i] = 0;
    auto fold = [&](double x, uint64_t r) {
        const double t = (double)(S.tick0 + r * S.tick_step);
        if constexpr (kScores) {
            if (m && fabs(x) <= DBL_MAX) {
                if (n == 0.0) K = x;
                const double y = __dsub_rn(x, K);
                S1 = __dadd_rn(S1, y);
                S2 = __dadd_rn(S2, __dmul_rn(y, y));
                n = n + 1.0;
            }
#pragma unroll
            for (uint32_t i = 0; i < B200_MAX_DWELLS; ++i) {
                if ((dmine >> i) & 1u) {
                    if (S.d[i].above ? x > S.d[i].value : x < S.d[i].value) { // NaN never counts
                        if (cnt[i] == 0) first[i] = (uint32_t)r;
                        last[i] = (uint32_t)r;
                        ++cnt[i];
                    }
                }
            }
        }
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
    if constexpr (kScores) {
        if (m) {
            m[0] = n;
            m[S.ld] = K;
            m[2 * S.ld] = S1;
            m[3 * S.ld] = S2;
        }
#pragma unroll
        for (uint32_t i = 0; i < B200_MAX_DWELLS; ++i) {
            if (cnt[i]) {
                double *o = S.dwell + (w * S.n_dwell + i) * 3;
                const double tf = (double)(S.tick0 + first[i] * S.tick_step);
                const double tl = (double)(S.tick0 + last[i] * S.tick_step);
                const double of = o[1], ol = o[2];
                o[0] = o[0] + (double)cnt[i];
                o[1] = of < 0.0 || tf < of ? tf : of;
                o[2] = tl > ol ? tl : ol;
            }
        }
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

// moment accumulators: n, K, S1, S2 = 0; dwell records: rows = 0, first_tick = last_tick = -1
__global__ void __launch_bounds__(kSumThreads) scores_clear_kernel(double *mom, uint64_t mom_len, double *dwell,
                                                                   uint64_t dwell_len)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < mom_len + dwell_len; i += (uint64_t)gridDim.x * blockDim.x) {
        if (i < mom_len) mom[i] = 0.0;
        else dwell[i - mom_len] = (i - mom_len) % 3 == 0 ? 0.0 : -1.0;
    }
}

// the public table's (n, mean, m2) records (moment_field)
__global__ void __launch_bounds__(kSumThreads) moment_table_kernel(const double *__restrict__ mom, uint64_t ld, uint32_t k,
                                                                   uint64_t b0, uint64_t nb, double *__restrict__ out)
{
    const uint64_t F = 3ull * k;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < nb * F; i += (uint64_t)gridDim.x * blockDim.x)
        out[i] = moment_field(mom + (i % F) / 3 * 4 * ld + b0 + i / F, ld, (uint32_t)(i % 3));
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
    const uint64_t n_worlds = S.n_entities ? S.n_bodies / S.n_entities : 0;
    const uint64_t ext_len = S.ext ? 5ull * S.width * S.ld : 0;
    const uint64_t thr_len = S.thr ? n_worlds * S.n_thr * kThrFields : 0;
    if (ext_len + thr_len) {
        const uint64_t blocks = std::min<uint64_t>((ext_len + thr_len + kSumThreads - 1) / kSumThreads, 64ull * kNumSMs * 8);
        summary_clear_kernel<<<(unsigned)blocks, kSumThreads, 0, s>>>(S.ext, S.ld, S.width, S.thr, thr_len);
        ++*launches;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    const uint64_t mom_len = S.mom ? 4ull * S.n_mom * S.ld : 0;
    const uint64_t dwell_len = S.dwell ? n_worlds * S.n_dwell * 3 : 0;
    if (mom_len + dwell_len) {
        const uint64_t blocks = std::min<uint64_t>((mom_len + dwell_len + kSumThreads - 1) / kSumThreads, 64ull * kNumSMs * 8);
        scores_clear_kernel<<<(unsigned)blocks, kSumThreads, 0, s>>>(S.mom, mom_len, S.dwell, dwell_len);
        ++*launches;
    }
    return cudaGetLastError();
}

cudaError_t launch_summary_fold(const SummaryParams &S, int *launches, cudaStream_t s)
{
    *launches = 0;
    if (S.n_rows == 0 || S.n_bodies == 0 || S.n_planes == 0) return cudaSuccess;
    const dim3 grid((unsigned)((S.n_bodies + kSumThreads - 1) / kSumThreads), S.n_planes);
    if (S.mom || S.dwell) summary_fold_kernel<true><<<grid, kSumThreads, 0, s>>>(S);
    else summary_fold_kernel<false><<<grid, kSumThreads, 0, s>>>(S);
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

cudaError_t launch_moment_table(const double *mom, uint64_t ld, uint32_t k, uint64_t b0, uint64_t nb, double *out,
                                cudaStream_t s)
{
    if (nb == 0 || k == 0) return cudaSuccess;
    const uint64_t blocks = std::min<uint64_t>((nb * 3 * k + kSumThreads - 1) / kSumThreads, 64ull * kNumSMs * 8);
    moment_table_kernel<<<(unsigned)blocks, kSumThreads, 0, s>>>(mom, ld, k, b0, nb, out);
    return cudaGetLastError();
}

} // namespace b200
