// Derived channels (include/b200_sixdof.h b200_channel): n_c values per body per row, computed from the body's 25-plane
// row and written as extra planes that every ensemble reduction and run summary reads like the state components.
//
// A streaming pass: one thread per body per sample, each reading the planes its channels need (coalesced, one double
// per plane) and writing n_c doubles; the channel table stays in the parameter space.  The arithmetic is the contract
// of the header: NORM in correctly rounded, uncontracted operations, AXIS_ANGLE through the EXACT rotation of the tick
// (sixdof_device.cuh ex::qrot) in both math modes, then CUDA's double atan2.
#include <algorithm>

#include "sixdof_device.cuh"
#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kChanThreads = 256;

__global__ void __launch_bounds__(kChanThreads) channel_kernel(const __grid_constant__ ChannelParams P)
{
    const uint64_t b = (uint64_t)blockIdx.x * kChanThreads + threadIdx.x;
    if (b >= P.n_bodies) return;
    for (uint64_t s = blockIdx.y; s < P.n_samples; s += gridDim.y) {
        const uint64_t off = s * P.row_stride + b;
        double *o = P.out + s * P.n_c * P.ld + b;
        for (uint32_t k = 0; k < P.n_c; ++k) {
            const b200_channel &c = P.c[k];
            double v;
            if (c.kind == B200_CHANNEL_NORM) {
                double acc = 0.0;
                for (uint32_t i = 0; i < c.n; ++i) {
                    const double d = __dsub_rn(P.row[c.plane[i]][off], c.c[i]);
                    const double sq = __dmul_rn(d, d);
                    acc = i == 0 ? sq : __dadd_rn(acc, sq);
                }
                v = __dsub_rn(__dsqrt_rn(acc), c.r0);
            } else { // B200_CHANNEL_AXIS_ANGLE
                const Quat q = {P.row[0][off], P.row[1][off], P.row[2][off], P.row[3][off]};
                const Vec3 u = ex::qrot(q, Vec3{c.c[0], c.c[1], c.c[2]});
                Vec3 w = {c.d[0], c.d[1], c.d[2]};
                if (c.n == 3) w = Vec3{P.row[c.plane[0]][off], P.row[c.plane[0] + 1][off], P.row[c.plane[0] + 2][off]};
                using namespace ex;
                const double x = sub(mul(u.y, w.z), mul(u.z, w.y));
                const double y = sub(mul(u.z, w.x), mul(u.x, w.z));
                const double z = sub(mul(u.x, w.y), mul(u.y, w.x));
                const double sn = sqr(add(add(mul(x, x), mul(y, y)), mul(z, z)));
                const double cs = add(add(mul(u.x, w.x), mul(u.y, w.y)), mul(u.z, w.z));
                v = atan2(sn, cs);
            }
            o[(uint64_t)k * P.ld] = v;
        }
    }
}

} // namespace

cudaError_t launch_channels(const ChannelParams &P, int *launches, cudaStream_t s)
{
    *launches = 0;
    if (P.n_samples == 0 || P.n_bodies == 0 || P.n_c == 0) return cudaSuccess;
    const uint64_t bx = (P.n_bodies + kChanThreads - 1) / kChanThreads;
    // enough blocks in flight to stream at full bandwidth; further samples loop inside the grid
    const uint64_t by = std::min<uint64_t>(P.n_samples, std::max<uint64_t>(1, std::min<uint64_t>(65535, 64ull * kNumSMs * 8 / bx)));
    channel_kernel<<<dim3((unsigned)bx, (unsigned)by), kChanThreads, 0, s>>>(P);
    *launches = 1;
    return cudaGetLastError();
}

} // namespace b200
