// sm_90a layout kernels (K6 of SURVEY §2.4): host column layout [body][width] <-> device SoA planes,
// and the FP64 throughput probe.
#include <algorithm>

#include "sixdof_device.cuh"
#include "sixdof_internal.h"
#include "sixdof_launch.h"

namespace b200 {

// ================================================================== layout kernels (K6)

static constexpr int kTile = 256;

__global__ void __launch_bounds__(kTile) aos_to_soa_kernel(const double *__restrict__ aos, double *__restrict__ soa,
                                                           uint64_t n_bodies, uint32_t width, uint64_t ld)
{
    extern __shared__ double tile[]; // kTile * (width | 1)
    const uint32_t pitch = width | 1u;
    const uint64_t base = (uint64_t)blockIdx.x * kTile;
    const uint32_t nb = (uint32_t)min((uint64_t)kTile, n_bodies - base);
    const double *src = aos + base * width;
    for (uint32_t i = threadIdx.x; i < nb * width; i += kTile) tile[(i / width) * pitch + (i % width)] = src[i];
    __syncthreads();
    if (threadIdx.x < nb)
        for (uint32_t k = 0; k < width; ++k) soa[(uint64_t)k * ld + base + threadIdx.x] = tile[threadIdx.x * pitch + k];
}

// gridDim.y = samples; a sample's planes start at soa + y*width*ld, its rows at aos + y*n_bodies*width
__global__ void __launch_bounds__(kTile) soa_to_aos_kernel(const double *__restrict__ soa, double *__restrict__ aos,
                                                           uint64_t n_bodies, uint32_t width, uint64_t ld)
{
    extern __shared__ double tile[];
    const uint32_t pitch = width | 1u;
    const uint64_t base = (uint64_t)blockIdx.x * kTile;
    const uint32_t nb = (uint32_t)min((uint64_t)kTile, n_bodies - base);
    const double *s = soa + (uint64_t)blockIdx.y * width * ld;
    double *dst = aos + (uint64_t)blockIdx.y * n_bodies * width + base * width;
    if (threadIdx.x < nb)
        for (uint32_t k = 0; k < width; ++k) tile[threadIdx.x * pitch + k] = s[(uint64_t)k * ld + base + threadIdx.x];
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < nb * width; i += kTile) dst[i] = tile[(i / width) * pitch + (i % width)];
}

// All columns of a small batch in one launch: blockIdx.y selects the column, the AoS side of every
// column lives in one packed staging buffer (one PCIe transfer per direction per invoke_batch).
__global__ void __launch_bounds__(kTile) multi_transpose_kernel(const __grid_constant__ MultiColumns mc, uint64_t n_bodies, uint64_t ld,
                                                                int to_soa)
{
    extern __shared__ double tile[];
    const MultiColumns::Col c = mc.col[blockIdx.y];
    const uint32_t width = c.width, pitch = width | 1u;
    const uint64_t base = (uint64_t)blockIdx.x * kTile;
    if (base >= n_bodies) return;
    const uint32_t nb = (uint32_t)min((uint64_t)kTile, n_bodies - base);
    double *aos = mc.packed + c.aos_offset + base * width;
    if (to_soa) {
        for (uint32_t i = threadIdx.x; i < nb * width; i += kTile) tile[(i / width) * pitch + (i % width)] = aos[i];
        __syncthreads();
        if (threadIdx.x < nb)
            for (uint32_t k = 0; k < width; ++k) c.soa[(uint64_t)k * ld + base + threadIdx.x] = tile[threadIdx.x * pitch + k];
    } else {
        if (threadIdx.x < nb)
            for (uint32_t k = 0; k < width; ++k) tile[threadIdx.x * pitch + k] = c.soa[(uint64_t)k * ld + base + threadIdx.x];
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < nb * width; i += kTile) aos[i] = tile[(i / width) * pitch + (i % width)];
    }
}

// FP64 FMA throughput probe: 8 independent chains per thread
__global__ void __launch_bounds__(256) probe_fp64_kernel(double *out, int iters)
{
    double a0 = threadIdx.x * 1e-9, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
    const double m = 1.0000001, c = 1e-9;
    for (int i = 0; i < iters; ++i) {
        a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
        a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
    }
    out[(uint64_t)blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

// ================================================================== launchers
//
// A tile holds kTile rows of (width | 1) doubles: a column wider than 23 (an 8-wheel torque column is 24, a full
// trajectory sample 25) needs more than the 48 KB of dynamic shared memory a kernel gets without opting in, so every
// launcher raises its kernel's limit first (once per kernel, device and size).

cudaError_t launch_aos_to_soa(const double *aos, double *soa, uint64_t n_bodies, uint32_t width, uint64_t ld, cudaStream_t s)
{
    if (n_bodies == 0) return cudaSuccess;
    const size_t smem = (size_t)kTile * (width | 1u) * sizeof(double);
    const cudaError_t e = ensure_dynamic_smem(aos_to_soa_kernel, smem);
    if (e != cudaSuccess) return e;
    const unsigned grid = (unsigned)((n_bodies + kTile - 1) / kTile);
    aos_to_soa_kernel<<<grid, kTile, smem, s>>>(aos, soa, n_bodies, width, ld);
    return cudaGetLastError();
}

cudaError_t launch_soa_to_aos(const double *soa, double *aos, uint64_t n_bodies, uint32_t width, uint64_t ld, cudaStream_t s)
{
    if (n_bodies == 0) return cudaSuccess;
    const size_t smem = (size_t)kTile * (width | 1u) * sizeof(double);
    const cudaError_t e = ensure_dynamic_smem(soa_to_aos_kernel, smem);
    if (e != cudaSuccess) return e;
    const dim3 grid((unsigned)((n_bodies + kTile - 1) / kTile), 1);
    soa_to_aos_kernel<<<grid, kTile, smem, s>>>(soa, aos, n_bodies, width, ld);
    return cudaGetLastError();
}

cudaError_t launch_traj_to_aos(const double *traj, double *aos, uint64_t n_samples, uint64_t n_bodies, uint64_t ld,
                               uint32_t width, cudaStream_t s)
{
    if (n_bodies == 0 || n_samples == 0) return cudaSuccess;
    const size_t smem = (size_t)kTile * (width | 1u) * sizeof(double); // 25 planes: 52 KB, above the 48 KB default
    cudaError_t e = ensure_dynamic_smem(soa_to_aos_kernel, smem);
    if (e != cudaSuccess) return e;
    for (uint64_t s0 = 0; s0 < n_samples; s0 += 32768) {
        const unsigned ny = (unsigned)min((uint64_t)32768, n_samples - s0);
        const dim3 grid((unsigned)((n_bodies + kTile - 1) / kTile), ny);
        soa_to_aos_kernel<<<grid, kTile, smem, s>>>(traj + s0 * width * ld, aos + s0 * n_bodies * width, n_bodies, width, ld);
    }
    return cudaGetLastError();
}

cudaError_t launch_multi_transpose(const MultiColumns &mc, uint64_t n_bodies, uint64_t ld, bool to_soa, cudaStream_t s)
{
    if (n_bodies == 0 || mc.n == 0) return cudaSuccess;
    uint32_t wmax = 1;
    for (uint32_t i = 0; i < mc.n; ++i) wmax = std::max(wmax, mc.col[i].width);
    const size_t smem = (size_t)kTile * (wmax | 1u) * sizeof(double);
    const cudaError_t e = ensure_dynamic_smem(multi_transpose_kernel, smem);
    if (e != cudaSuccess) return e;
    const dim3 grid((unsigned)((n_bodies + kTile - 1) / kTile), mc.n);
    multi_transpose_kernel<<<grid, kTile, smem, s>>>(mc, n_bodies, ld, to_soa ? 1 : 0);
    return cudaGetLastError();
}

cudaError_t launch_probe_fp64(double *out, int iters, int blocks, cudaStream_t s)
{
    probe_fp64_kernel<<<blocks, 256, 0, s>>>(out, iters);
    return cudaGetLastError();
}

// ================================================================== self-test of the shared-divisor divisions
//
// ex::rcp_prep / ex::div_rcp (sixdof_device.cuh) against div.rn.f64, operand for operand: groups of four dividends over
// one divisor, as the EXACT tick forms them (`ok` false -> the group is redone with __ddiv_rn), from a counter-based
// generator that covers the whole encoding space and the corners of the range test.
__device__ __forceinline__ uint64_t mix64(uint64_t z)
{
    z += 0x9e3779b97f4a7c15ull;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ double with_exponent(uint64_t bits, unsigned lo, unsigned span)
{
    const uint64_t e = lo + (unsigned)((bits >> 52) % span); // biased exponent in [lo, lo + span)
    return __longlong_as_double((long long)((bits & 0x800fffffffffffffull) | (e << 52)));
}

__global__ void __launch_bounds__(256) selftest_div_kernel(uint64_t seed, uint64_t n_groups, unsigned long long *counts)
{
    unsigned long long bad = 0, fast = 0;
    for (uint64_t g = (uint64_t)blockIdx.x * 256 + threadIdx.x; g < n_groups; g += (uint64_t)gridDim.x * 256) {
        const uint64_t h = mix64(seed + g * 5u);
        const unsigned mode = (unsigned)(g % 10u);
        double d, a[4];
        const uint64_t hd = mix64(h);
        uint64_t ha[4];
        for (int i = 0; i < 4; ++i) ha[i] = mix64(h + 1 + i);
        switch (mode) {
        case 0: d = __longlong_as_double((long long)hd); for (int i = 0; i < 4; ++i) a[i] = __longlong_as_double((long long)ha[i]); break; // any encoding
        case 1: d = with_exponent(hd, 993, 60); for (int i = 0; i < 4; ++i) a[i] = with_exponent(ha[i], 993, 60); break;                   // ordinary magnitudes
        case 2: d = with_exponent(hd, 1000, 40); for (int i = 0; i < 4; ++i) a[i] = with_exponent(ha[i], 30, 50); break;                    // dividends around the tiny-exponent threshold
        case 3: d = with_exponent(hd, 1, 80); for (int i = 0; i < 4; ++i) a[i] = with_exponent(ha[i], 1960, 86); break;                      // quotients at the overflow edge
        case 4: d = with_exponent(hd, 1900, 146); for (int i = 0; i < 4; ++i) a[i] = with_exponent(ha[i], 0, 120); break;                    // quotients in the denormals, denormal dividends
        case 5: d = with_exponent(hd, 0, 2047);                                                                                              // zero / denormal dividends over anything
                for (int i = 0; i < 4; ++i) a[i] = (ha[i] & 1) ? __longlong_as_double((long long)(ha[i] & 0x8000000000000000ull)) : with_exponent(ha[i], 0, 1);
                break;
        case 6: d = __longlong_as_double((long long)((hd & 0xfff0000000000000ull) | ((hd & 1) ? 0x000fffffffffffffull : 0ull)));            // power of two / all-ones significand
                d = with_exponent((uint64_t)__double_as_longlong(d), 900, 240);
                for (int i = 0; i < 4; ++i) a[i] = with_exponent(ha[i], 900, 240);
                break;
        case 7: d = with_exponent(hd, 1000, 46); for (int i = 0; i < 4; ++i) a[i] = __dmul_rn(d, (double)(int)(ha[i] % 2001u) - 1000.0); break; // exact quotients
        case 8: {                                                                                                                           // the workload: a unit quaternion over its norm
            double q[4], n2 = 0.0;
            for (int i = 0; i < 4; ++i) { q[i] = (double)(long long)(ha[i] >> 11) * 0x1p-52 - 1.0; n2 += q[i] * q[i]; }
            const double n = sqrt(n2) * (1.0 + ((double)(hd & 0xff) - 128.0) * 0x1p-52);
            d = (hd & 0x100) ? n : n * n;
            for (int i = 0; i < 4; ++i) a[i] = q[i];
            break;
        }
        default: d = with_exponent(hd, 1013, 20); for (int i = 0; i < 4; ++i) a[i] = (ha[i] & 3) ? with_exponent(ha[i], 1000, 46) : 0.0; break; // forces with zero components over a mass
        }
        const ex::Rcp r = ex::rcp_prep(d);
        bool ok = true;
        double got[4];
        for (int i = 0; i < 4; ++i) got[i] = ex::div_rcp(a[i], r, ok);
        if (!ok) { const double dd = ex::rare_path(d); for (int i = 0; i < 4; ++i) got[i] = __ddiv_rn(a[i], dd); }
        fast += ok ? 1u : 0u;
        for (int i = 0; i < 4; ++i) {
            const double want = __ddiv_rn(a[i], d);
            const bool same = __double_as_longlong(got[i]) == __double_as_longlong(want) || (got[i] != got[i] && want != want);
            bad += same ? 0u : 1u;
        }
    }
    if (bad) atomicAdd(counts, bad);
    if (fast) atomicAdd(counts + 1, fast);
}

cudaError_t launch_selftest_div(uint64_t seed, uint64_t n_groups, unsigned long long *counts, cudaStream_t s)
{
    const unsigned blocks = (unsigned)std::min<uint64_t>((n_groups + 255) / 256, kNumSMs * 16u);
    if (blocks) selftest_div_kernel<<<blocks, 256, 0, s>>>(seed, n_groups, counts);
    return cudaGetLastError();
}


} // namespace b200
