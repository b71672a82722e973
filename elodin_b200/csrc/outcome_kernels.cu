// Outcome values (include/b200_sixdof.h b200_outcome): one f64 per world per outcome, taken from the run summaries'
// accumulators or a device column and written as planes of ld_o values, which the ensemble reductions then read like a
// state of one entity.
//
// A streaming pass: one thread per world, each reading one record per outcome (a strided gather from the world-major
// threshold and dwell tables, coalesced loads from the SoA extrema, moment and column planes) and writing one
// coalesced double per outcome; the source table stays in the parameter space.
#include <algorithm>

#include "sixdof_internal.h"

namespace b200 {
namespace {

constexpr unsigned kOutThreads = 256;

__global__ void __launch_bounds__(kOutThreads) outcome_kernel(const __grid_constant__ OutcomeParams P)
{
    const uint64_t w = (uint64_t)blockIdx.x * kOutThreads + threadIdx.x;
    if (w >= P.n_worlds) return;
    for (uint32_t k = 0; k < P.n_src; ++k) {
        const OutcomeParams::Src &o = P.o[k];
        const double *a = o.src + w * o.stride;
        double v;
        if (o.op == kOutCopy) {
            v = a[0];
        } else if (o.op == kOutTick) {
            v = a[0] == -1.0 ? __longlong_as_double(0x7ff8000000000000ll) : a[0];
        } else if (o.op == kOutCount) {
            v = moment_field(a, P.ld, 0);
        } else if (o.op == kOutMean) {
            v = moment_field(a, P.ld, 1);
        } else { // kOutStd, kOutRms: numpy's sqrt(m2 / n) and sqrt(mean * mean + m2 / n)
            const double var = __ddiv_rn(moment_field(a, P.ld, 2), a[0]);
            if (o.op == kOutStd) {
                v = __dsqrt_rn(var);
            } else {
                const double mean = moment_field(a, P.ld, 1);
                v = __dsqrt_rn(__dadd_rn(__dmul_rn(mean, mean), var));
            }
        }
        P.out[(uint64_t)o.plane * P.ld_o + w] = v;
    }
}

} // namespace

cudaError_t launch_outcomes(const OutcomeParams &P, int *launches, cudaStream_t s)
{
    *launches = 0;
    if (P.n_src == 0 || P.n_worlds == 0) return cudaSuccess;
    outcome_kernel<<<(unsigned)((P.n_worlds + kOutThreads - 1) / kOutThreads), kOutThreads, 0, s>>>(P);
    *launches = 1;
    return cudaGetLastError();
}

} // namespace b200
