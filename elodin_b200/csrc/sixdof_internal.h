// Host<->kernel parameter blocks of libb200_sixdof (internal; the public surface
// is include/b200_sixdof.h).
#pragma once
#include <cfloat>
#include <cstdint>
#include <cuda_runtime.h>
#include <vector>

#include "../../include/b200_sixdof.h"

namespace b200 {

// SMs of the target GPU (H100 SXM): launch-shape thresholds that are fixed at compile time size themselves by it;
// grids that depend on occupancy query the device instead.
constexpr unsigned kNumSMs = 132;

// One built-in effector as the kernels see it.  `col` points at the SoA planes
// of its per-body input column (plane p at col + p*ld), nullptr if none.
struct EffDev {
    uint32_t kind;
    uint32_t flags;
    double p[8];
    const double *col;
    uint32_t col_width;
    uint32_t pad;
    const uint8_t *mask; // [n_entities] or nullptr (query-join membership)
    const double *table; // GRAVITY_EGM08: the term stream sixdof_abi.cu:egm08_tables builds (device)
};

// Launch parameters of the per-body integrator kernels.  All columns are SoA:
// plane k of a column lives at base + k*ld, body b at [.. + b].
struct StepParams {
    double *pos;        // 7 planes: q.i q.j q.k q.w x y z
    double *vel;        // 6 planes: omega(3) v(3)
    double *acc;        // 6 planes (WorldAccel; stage-4 value on output)
    double *frc;        // 6 planes (Force; stage-4 value on output)
    const double *ine;  // 7 planes: diag(3) momentum(3) mass
    const double *gforce; // 9 planes: edge_fold gravity at the 3 distinct stage positions (or nullptr)
    const uint8_t *has_edge; // [n_entities]: body owns >= 1 out-edge (or nullptr)
    const double *aforce;    // 9 planes: additive stage forces (GRAVITY_EGM08) at the 3 distinct stage positions (or nullptr)
    uint64_t ld;        // plane stride in doubles
    uint64_t n_bodies;  // n_worlds * n_entities
    uint32_t n_entities;
    uint32_t n_eff;
    double dt_stage;    // SimulationTimeStep (rk4.rs:90)
    double dt_final;    // six_dof(time_step=) or dt_stage (rk4.rs:83,119)
    uint32_t n_ticks;   // ticks integrated by this launch (state stays in registers)
    uint32_t write_fa;  // materialise Force / WorldAccel at the end of the launch
    // trajectory ring: sample s, plane p at traj + (s*traj_planes + p)*ld
    double *traj;
    uint64_t traj_capacity;
    uint32_t traj_every;  // 0 = off
    uint32_t traj_planes; // 13 (pos, vel) or 25 (+ accel, force)
    uint64_t tick0;     // global tick count before this launch
    uint32_t ent0;      // entity row of body 0 of this launch (row-sharded single worlds start inside a world)
    uint32_t reverse;   // walk the tiles from the last one down (alternating launches: L2 reuse of the previous launch's tail)
    // mass-class summary of this launch's bodies (one byte per 64-body segment, segment 0 starting at body 0 of the
    // launch; see body_fast_spec_kernel), or nullptr where the launch must read every mass
    uint8_t *mass_class;
    // compile-time-specialised FAST kernels (sixdof_tick.cuh SIG_*): what body_kernels.cu:spec_signature
    // distilled from eff[] — uniform constants and the plane bases of the per-body input columns
    struct Spec {
        double g[3];        // sum of the GRAVITY_CONST vectors
        double axis[3];     // THRUST_BODY body axis
        double kd;          // 0.5 * Cd*rho * area of a DRAG_QUADRATIC without per-body parameters
        double mu, om[3];   // GRAVITY_FRAME
        double j2_mu, j2_k; // GRAVITY_J2: mu, J2 * r_ref^2
        const double *wheels;        // 9 planes: three body-frame wheel torques
        const double *wworld;        // 6 planes: world-frame wrench [tau, f]
        const double *thrust;        // 1 plane
        const double *wr_t, *wr_f;   // 3 planes each: body-frame torque / force of the wrench column
        const double *drag;          // wind(3) [+ Cd*rho, area]
    } spec;
    EffDev eff[B200_MAX_EFFECTORS];
};

// Launch parameters of the edge_fold gravity kernels.
struct GraphParams {
    const double *pos, *vel, *ine;
    double *gforce;          // 9 planes out
    uint64_t ld;
    uint32_t n_entities;
    uint32_t n_worlds;
    double dt_stage;
    uint32_t kind;           // B200_EFF_GRAVITY_EDGES_*
    uint32_t integrator;     // B200_INTEGRATOR_*: RK4 evaluates 3 stage positions, semi-implicit 1
    double p0, p1;           // G | K^2, softening
    const uint32_t *row_ptr; // CSR over sources (n_entities+1), spawn order kept inside a row
    const uint32_t *col_idx;
    uint32_t max_deg;        // largest out-degree (uniform trip count of small_world_kernel's shuffle loop)
    uint32_t src0;           // dense kernels: fold only the source rows [src0, src0 + src_n) of every world (row-sharded
    uint32_t src_n;          // single worlds); src_n = 0 means every source
    uint32_t pad;
};

// Column table of the one-launch layout kernel used by small batches
struct MultiColumns {
    struct Col {
        uint64_t aos_offset; // doubles from `packed`
        double *soa;         // plane 0 of the device column
        uint32_t width;
        uint32_t pad;
    };
    double *packed;          // packed AoS staging (device)
    uint32_t n;
    uint32_t pad;
    Col col[16];
};

// kernel launchers (sixdof_kernels.cu); every one returns the launch status
cudaError_t launch_body_step(const StepParams &P, int integrator, int math_mode, cudaStream_t s);
cudaError_t launch_graph_force(const GraphParams &G, int math_mode, bool dense, cudaStream_t s);
// one-launch n-body tick (gravity + integration) for small grids; new pose / velocity go to *_out
bool nbody_fused_applicable(const GraphParams &G, int math_mode, bool dense);
cudaError_t launch_nbody_tick_fused(const GraphParams &G, const StepParams &P, double *pos_out, double *vel_out, cudaStream_t s);
// worlds of <= 32 bodies: gravity + integration of n_ticks ticks in one launch, one warp per floor(32/N) worlds
bool small_world_applicable(const GraphParams &G, int math_mode);
cudaError_t launch_small_world(const GraphParams &G, const StepParams &P, int math_mode, cudaStream_t s);
// GRAVITY_EGM08: the field at the three stage positions of every body -> 9 planes (one launch per tick)
struct EgmParams {
    const double *pos, *vel, *ine;
    double *aforce;
    const double *table;     // term stream of sixdof_abi.cu:egm08_tables (device)
    const uint8_t *mask;     // entity mask of the effector or nullptr
    uint64_t ld, n_bodies;
    uint32_t n_entities, ent0;
    uint32_t L, integrator;
    double mu, r_ref, dt_stage;
};
cudaError_t launch_egm08_force(const EgmParams &E, int math_mode, cudaStream_t s);
cudaError_t launch_aos_to_soa(const double *aos, double *soa, uint64_t n_bodies, uint32_t width, uint64_t ld,
                              cudaStream_t s);
cudaError_t launch_soa_to_aos(const double *soa, double *aos, uint64_t n_bodies, uint32_t width, uint64_t ld,
                              cudaStream_t s);
cudaError_t launch_traj_to_aos(const double *traj, double *aos, uint64_t n_samples, uint64_t n_bodies, uint64_t ld,
                               uint32_t width, cudaStream_t s);
cudaError_t launch_multi_transpose(const MultiColumns &mc, uint64_t n_bodies, uint64_t ld, bool to_soa, cudaStream_t s);
cudaError_t launch_probe_fp64(double *out, int iters, int blocks, cudaStream_t s);
cudaError_t launch_selftest_div(uint64_t seed, uint64_t n_groups, unsigned long long *counts, cudaStream_t s);

// Ensemble statistics over the world axis (stats_kernels.cu).  One group = (count, mean, m2 = sum (x - mean)^2, min,
// max) over the finite values of a set of worlds; while count = 0 the other fields are mean = m2 = 0, min = +inf,
// max = -inf (a finished table writes NaN there instead).
struct StatsGroup {
    double n, mean, m2, mn, mx;
};

// a := a (+) b, Chan et al.'s pairwise update.  Every merge of partial groups, on the device and in b200_stats_merge,
// goes through this function.  A group with count 0 is the identity, whatever its other fields hold.
__host__ __device__ inline void stats_merge(StatsGroup &a, const StatsGroup &b)
{
    if (b.n == 0.0) return;
    if (a.n == 0.0) { a = b; return; }
    const double n = a.n + b.n;
    const double d = b.mean - a.mean;
    a.mean = a.mean + d * b.n / n;
    a.m2 = a.m2 + b.m2 + d * d * a.n * b.n / n;
    a.mn = fmin(a.mn, b.mn);
    a.mx = fmax(a.mx, b.mx);
    a.n = n;
}

// Planes to reduce: the planes of a sample are the concatenated segments' planes, segment k holding n_planes planes per
// sample, plane j of sample s at base + s * stride + j * ld; plane i of the launch is plane i % W of sample i / W,
// W = planes_per_sample = the sum of the segments' n_planes.  Group (plane i, entity e) goes to
// out[((i / W) * n_entities + e) * W + i % W][5].  Only bodies b = w * n_entities + e with w < n_worlds are read (never
// the padding to ld).  A ring of W planes per sample is one segment of stride W * ld, so plane i is at base + i * ld.
constexpr uint32_t kMaxSegs = 5; // the state's four columns, then the channel planes (sixdof_abi.cu:ensemble_rows)
struct StatsParams {
    struct Seg {
        const double *base;
        uint64_t n_planes;
        uint64_t stride;
    } seg[kMaxSegs];
    uint32_t n_segs;
    uint32_t planes_per_sample;
    uint64_t n_planes;
    uint64_t ld;
    uint64_t n_worlds;
    uint64_t n_entities;
    double *out;
};
// plane j (< planes_per_sample) of sample s
__device__ inline const double *sample_plane(const StatsParams &S, uint64_t s, uint64_t j)
{
    const double *p = nullptr;
#pragma unroll
    for (uint32_t k = 0; k < kMaxSegs; ++k) { // constant indices: the segment table stays in the parameter space
        if (!p && k < S.n_segs) {
            if (j < S.seg[k].n_planes) p = S.seg[k].base + s * S.seg[k].stride + j * S.ld;
            else j -= S.seg[k].n_planes;
        }
    }
    return p; // j < planes_per_sample: always set
}
// plane i (< n_planes) of the concatenated samples
__device__ inline const double *stats_plane(const StatsParams &S, uint64_t i)
{
    const uint64_t s = i / S.planes_per_sample;
    return sample_plane(S, s, i - s * S.planes_per_sample);
}
// Rows of chosen worlds (layout_kernels.cu:gather_worlds_kernel): samples [s0, s0 + n_samples) of S's planes for the
// worlds worlds[0 .. n_worlds) (device memory, each < S.n_worlds, repeats allowed) into S.out =
// [n_samples][n_worlds][n_entities][planes_per_sample], the layout of b200_sixdof_trajectory_download restricted to
// those worlds.  One launch per 32768 samples on s (*launches); none without rows.
cudaError_t launch_gather_worlds(const StatsParams &S, const uint64_t *worlds, uint64_t n_worlds, uint64_t s0,
                                 uint64_t n_samples, int *launches, cudaStream_t s);
// A world group of a grouped reduction: the worlds [o, o + n), reduced in C chunks of Wc worlds; k0 = the chunks of the
// groups before it, which numbers the block tasks of a launch and places the group's partials.
struct WorldGroup {
    uint64_t o, n, Wc, C, k0;
};
// the group of chunk k among the groups [g0, g1) of t: the last one whose first chunk is at most k (empty groups of the
// histogram table share their successor's k0 and are never chosen)
__device__ inline uint64_t group_of_chunk(const WorldGroup *t, uint64_t g0, uint64_t g1, uint64_t k)
{
    uint64_t lo = g0, hi = g1 - 1;
    while (lo < hi) {
        const uint64_t mid = (lo + hi + 1) / 2;
        if (t[mid].k0 <= k) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}
// The statistics table of consecutive groups of sizes[0 .. n_groups) (stats_shape per group; an empty group has one
// chunk of no worlds).  The ungrouped statistics are the one-group table {n_worlds}.
std::vector<WorldGroup> world_group_table(const uint64_t *sizes, uint64_t n_groups, uint64_t n_entities);
// f64 of device scratch the reduction over the groups of `table` needs (0: one pass, no scratch); at most 256 MiB
// unless one group-plane alone needs more
uint64_t world_stats_scratch_doubles(const StatsParams &S, const std::vector<WorldGroup> &table);
// One or two launches per slice of groups and planes on s (written to *launches); `groups` is `table` in device memory
// and `scratch` holds world_stats_scratch_doubles(S, table) f64.  Group g of G = table.size() goes to
// out[(((i / W) * G + g) * n_entities + e) * W + i % W][5].
cudaError_t launch_world_stats(const StatsParams &S, const WorldGroup *groups, const std::vector<WorldGroup> &table,
                               double *scratch, int *launches, cudaStream_t s);

// Ensemble quantiles over the world axis (quantile_kernels.cu): the planes of a StatsParams, n_q levels and the world
// groups of a group table (only o and n are read).  Triple (group g of G = n_groups, plane i, entity e) goes to
// out[(((i / W) * G + g) * n_entities + e) * W + i % W][n_q].
struct QuantileParams : StatsParams {
    uint32_t n_q;
    double q[B200_MAX_QUANTILES];
    const WorldGroup *groups;  // the group table, in device memory
    const uint32_t *order;     // quantile_order(table), in device memory
    uint64_t n_groups;
};
// the groups of a table listed by route (route_of, order_stats.cuh), each route in table order: the warp route (empty
// groups included), then the block route, then the rest (the radix select)
std::vector<uint32_t> quantile_order(const std::vector<WorldGroup> &table);
// bytes of device scratch the call over the groups of `table` needs: 0 without a group above 8192 worlds (one pass,
// no scratch), else at most 256 MiB
uint64_t quantile_scratch_bytes(const QuantileParams &S, const std::vector<WorldGroup> &table);
// one launch per small route that has groups, and a fixed launch sequence per slice of the large groups' triples
// (written to *launches); `scratch` holds quantile_scratch_bytes(S, table), `order` is quantile_order(table).  With a
// large group *reads (host memory) receives, once the stream reaches it, the reads of the planes summed over every
// triple; it is left alone otherwise (one read per triple).
cudaError_t launch_quantiles(const QuantileParams &S, const std::vector<WorldGroup> &table,
                             const std::vector<uint32_t> &order, void *scratch, int *launches,
                             unsigned long long *reads, cudaStream_t s);
// A rank's part of a world-sharded quantile call between its rounds (b200_sixdof_sharded_quantiles_*): the radix select
// over every group of `table`, slice by slice, each pass's counters summed over the ranks before its plan runs.
struct QuantileShard {
    QuantileParams S;               // S.out: the whole table, in device memory
    std::vector<WorldGroup> table;  // the rank's part of every group (only o and n are read)
    void *scratch = nullptr;        // sharded_quantile_scratch_bytes(S, table.size())
    uint64_t slice = 0;             // the slice the rounds are in
    int level = -1;                 // the pass whose words the last round sent (0: the counts), -1: none
    unsigned long long reads = 0;   // reads of the planes summed over the triples, once the last round is made
};
// device scratch of a sharded call over n_groups groups (0 without a triple), and its largest round in bytes
uint64_t sharded_quantile_scratch_bytes(const QuantileParams &S, uint64_t n_groups);
uint64_t sharded_quantile_round_bytes(const QuantileParams &S, uint64_t n_groups);
// One round on s, returning once the round's words are in `partial` (host or device memory): the sums of the last
// round's words from `reduced` (nothing before the first round), then the launches up to the next round's words
// (*partial_bytes; 0 once S.out holds the table).  *launches: the kernels it launched.
cudaError_t sharded_quantile_round(QuantileShard &Q, const void *reduced, void *partial, uint64_t *partial_bytes,
                                   int *launches, cudaStream_t s);

// Ensemble covariance over the world axis (cov_kernels.cu).  One entry (a, b) of a group over a set of worlds: the
// count n, the means of planes a and b, and the co-moment m = sum (x_a - mean_a)(x_b - mean_b); while n = 0 the other
// fields are unread.
struct CovEntry {
    double n, ma, mb, m;
};

// x := x (+) y, the covariance form of Chan et al.'s pairwise update.  Every merge of partial records, on the device and
// in b200_covariance_merge, goes through this function.  Swapping a and b swaps ma / mb and leaves m's bits alone.
__host__ __device__ inline void cov_merge(CovEntry &x, const CovEntry &y)
{
    if (y.n == 0.0) return;
    if (x.n == 0.0) { x = y; return; }
    const double n = x.n + y.n;
    const double da = y.ma - x.ma, db = y.mb - x.mb;
    x.ma = x.ma + da * y.n / n;
    x.mb = x.mb + db * y.n / n;
    x.m = x.m + y.m + da * db * x.n * y.n / n;
    x.n = n;
}

// The samples of a StatsParams (n_planes / planes_per_sample of them) and a selection of n_p distinct planes of a
// sample.  A record is n, mean[n_p], M[n_p][n_p] over the worlds of one (sample, world group, entity).
struct CovParams : StatsParams {
    uint32_t n_p;
    uint32_t planes[B200_MAX_COV_PLANES];
};
// The covariance table of consecutive groups of sizes[0 .. n_groups): cov_chunks per group (an empty group has one chunk
// of no worlds), k0 = the chunks of the groups before it.  It depends on the sizes and n_entities alone; the ungrouped
// covariance is the one-group table {n_worlds}.
std::vector<WorldGroup> cov_group_table(const uint64_t *sizes, uint64_t n_groups, uint64_t n_entities);
// bytes of device scratch the call over the groups of `table` needs (0: one chunk per group, no scratch); at most
// 256 MiB
uint64_t cov_scratch_bytes(const CovParams &S, const std::vector<WorldGroup> &table);
// One chunk launch, and a merge launch where a group of the slice takes more than one chunk, per slice of groups and
// samples (*launches); `groups` is `table` in device memory.  Sample s, group g of G = table.size(), entity e goes to
// out[((s * G + g) * n_entities + e) * (1 + n_p + n_p^2)].
cudaError_t launch_covariance(const CovParams &S, const WorldGroup *groups, const std::vector<WorldGroup> &table,
                              void *scratch, int *launches, cudaStream_t s);

// Ensemble histograms over the world axis (hist_kernels.cu): the samples of a StatsParams and n_specs specs, each one
// entity and one or two planes of a sample.  Sample s, spec k goes to out[s * record_len + spec[k].rec_off ..]: a 1D
// record [nonfinite, below, above, c_0 .. c_{n-1}] or a 2D one [nonfinite, outside, c_00 .. c_{na-1,nb-1}].  The edges
// of axis a of spec k are edges[spec[k].edge_off + (a ? bins[0] + 1 : 0) ..] (device memory, np.linspace's values).
struct HistParams : StatsParams {
    struct Spec {
        uint64_t entity;
        uint32_t n_axes;
        uint32_t plane[2];
        uint32_t bins[2];
        double lo[2], hi[2];
        double den;        // hi[0] - lo[0]: the 1D rule's divisor
        uint64_t rec_off;  // f64 from the start of a sample's row
        uint64_t edge_off; // f64 from `edges`
    } spec[B200_MAX_HISTOGRAMS];
    uint32_t n_specs;
    uint32_t smem_edges;   // the most edges one spec has (both axes)
    uint64_t record_len;   // f64 per sample: every spec's record
    const double *edges;
};
// The histogram table of consecutive groups of sizes[0 .. n_groups) of a call over n_pairs (sample, spec) pairs: each
// group's chunks (none for an empty group), about 2 block tasks per SM over the whole call.
std::vector<WorldGroup> hist_group_table(const uint64_t *sizes, uint64_t n_groups, uint64_t n_pairs);
// Zeroes out (a memset) and counts every (sample, group, spec) in one launch on s (*launches = 1; 0 with nothing to
// count).  `groups` is `table` in device memory; sample s, group g of G = table.size() goes to
// out[(s * G + g) * record_len ..].
cudaError_t launch_histograms(const HistParams &P, const WorldGroup *groups, const std::vector<WorldGroup> &table,
                              int *launches, cudaStream_t s);

// Run summaries over the time axis (summary_kernels.cu).  A fold reads n_rows rows of R = 25 + n_channels planes:
// plane p of row r at row[p] + r * (p < 25 ? row_stride : chan_stride) + b for body b < n_bodies, at tick
// tick0 + r * tick_step.
//   ext: extrema accumulators, plane p * 5 + f of ld doubles (f = min, max, min_tick, max_tick, first_nonfinite_tick),
//        i.e. body b's 5 R values read in plane order are its row of the public table; nullptr = no extrema.
//   thr: the public threshold table itself, [n_worlds][n_thr][26] f64 (tick, the 25 raw planes); nullptr = no thresholds.
//   mom: moment accumulators (n, K, S1, S2) of selected plane j at plane j * 4 + f of ld doubles; mom_slot[y] = j when
//        planes[y] is selected plane j, kNoMoment otherwise; nullptr = no moments.
//   dwell: the public dwell table itself, [n_worlds][n_dwell][3] f64 (rows, first_tick, last_tick); nullptr = none.
// Ticks are stored as f64 (exact below 2^53), -1 = none; every accumulator has one owning thread per fold.
// A fold reads only the planes listed in planes[0 .. n_planes): all R with extrema, else the union of the thresholds',
// moments' and dwells' planes.  With mom and dwell null the fold is the extrema / threshold kernel alone.
constexpr uint32_t kMaxRow = 25 + B200_MAX_CHANNELS;
struct SummaryParams {
    const double *row[kMaxRow];
    uint64_t row_stride;
    uint64_t chan_stride;
    uint64_t n_rows;
    uint64_t tick0, tick_step;
    uint64_t ld, n_bodies;
    uint32_t n_entities;
    uint32_t n_thr;
    double *ext;
    double *thr;
    uint32_t n_planes;
    uint32_t width;    // R: the planes of a row, and of an extrema table row
    uint8_t planes[kMaxRow];
    struct Thr {
        uint32_t entity, plane;
        int32_t above;
        uint32_t pad;
        double value;
    } t[B200_MAX_THRESHOLDS];
    double *mom;
    double *dwell;
    uint32_t n_mom;
    uint32_t n_dwell;
    uint8_t mom_slot[kMaxRow];
    Thr d[B200_MAX_DWELLS];
};
constexpr uint8_t kNoMoment = 0xff;
// the accumulators of S (ext, thr, mom, dwell) set to "nothing seen yet"; launches written to *launches (0, 1 or 2:
// one for ext / thr, one for mom / dwell)
cudaError_t launch_summary_clear(const SummaryParams &S, int *launches, cudaStream_t s);
// fold S's rows into the accumulators; launches written to *launches (0 when there are no rows, else 1)
cudaError_t launch_summary_fold(const SummaryParams &S, int *launches, cudaStream_t s);
// extrema accumulators of rows of R planes, bodies [b0, b0 + nb) -> out[nb][5 R] (the public table's rows)
cudaError_t launch_extrema_table(const double *ext, uint64_t ld, uint32_t R, uint64_t b0, uint64_t nb, double *out,
                                 cudaStream_t s);
// Field f (0 = n, 1 = mean, 2 = m2) of the moment record of the accumulator at a (n, K, S1, S2 at a[0], a[ld],
// a[2 ld], a[3 ld]): mean = K + S1 / n, m2 = S2 - S1 * (S1 / n) clamped at 0, +inf where S2 overflowed, NaN mean and m2
// while n = 0; each operation correctly rounded in both math modes, so that the host can restate it bit for bit.  The
// public moment table (moment_table_kernel) and the moment outcomes (outcome_kernel) both take their values from here.
__device__ __forceinline__ double moment_field(const double *a, uint64_t ld, uint32_t f)
{
    const double n = a[0];
    if (f != 0 && n == 0.0) return __longlong_as_double(0x7ff8000000000000ll);
    if (f == 1) return __dadd_rn(a[ld], __ddiv_rn(a[2 * ld], n));
    if (f == 2) {
        const double S1 = a[2 * ld], S2 = a[3 * ld];
        const double d = __dsub_rn(S2, __dmul_rn(S1, __ddiv_rn(S1, n)));
        return S2 > DBL_MAX ? S2 : d < 0.0 ? 0.0 : d;
    }
    return n;
}
// moment accumulators of k selected planes, bodies [b0, b0 + nb) -> out[nb][k][3] (n, mean, m2: the public table's rows)
cudaError_t launch_moment_table(const double *mom, uint64_t ld, uint32_t k, uint64_t b0, uint64_t nb, double *out,
                                cudaStream_t s);

// Derived channels (channel_kernels.cu, include/b200_sixdof.h b200_channel): n_c values per body of samples
// [0, n_samples), from the 25 planes of each sample (plane p of sample s at row[p] + s * row_stride) into
// out + (s * n_c + k) * ld + b, for bodies b < n_bodies only.
struct ChannelParams {
    const double *row[25];
    uint64_t row_stride;
    double *out;
    uint64_t ld, n_bodies, n_samples;
    uint32_t n_c;
    uint32_t pad;
    b200_channel c[B200_MAX_CHANNELS];
};
// one launch on s (*launches = 1; 0 without samples, bodies or channels)
cudaError_t launch_channels(const ChannelParams &P, int *launches, cudaStream_t s);

// Outcome values (outcome_kernels.cu, include/b200_sixdof.h b200_outcome): source k gives world w < n_worlds the value
// out[plane * ld_o + w], read at src + w * stride (sixdof_abi.cu:outcome_params resolves every outcome to its record):
//   kCopy  the f64 at src, its bits;   kTick  the f64 at src, NaN where it is -1;
//   kCount, kMean, kStd, kRms  of the moment accumulator at src (planes of ld, moment_field).
// VALUES outcomes have no source: set_outcomes wrote their planes once.
enum : uint32_t { kOutCopy = 0, kOutTick = 1, kOutCount = 2, kOutMean = 3, kOutStd = 4, kOutRms = 5 };
struct OutcomeParams {
    struct Src {
        const double *src;
        uint64_t stride;
        uint32_t op;
        uint32_t plane;
    } o[B200_MAX_OUTCOMES];
    uint32_t n_src;
    uint32_t pad;
    double *out;
    uint64_t ld_o;   // f64 per outcome plane
    uint64_t ld;     // f64 per moment accumulator plane
    uint64_t n_worlds;
};
// one launch on s (*launches = 1; 0 without sources or worlds)
cudaError_t launch_outcomes(const OutcomeParams &P, int *launches, cudaStream_t s);

// Worst worlds of the outcome planes (topk_kernels.cu, include/b200_sixdof.h b200_sixdof_outcome_top_worlds): for
// group g of the table and selected plane j, the first min(k, count) finite worlds in totalOrder (descending when
// `largest`), ties by ascending world, into out[(g * n_p + j) * (1 + 2k) ..] = [count, values[k], worlds[k]].
struct TopkParams {
    const double *planes;  // outcome plane 0; plane p at planes + p * ld, world w at [w]
    uint64_t ld;
    uint32_t n_p, k;       // selected planes, 1 <= k <= B200_MAX_TOP_WORLDS
    int32_t largest;
    uint32_t plane[B200_MAX_OUTCOMES];
    const WorldGroup *groups;  // the group table, in device memory
    const uint32_t *order;     // quantile_order(table), in device memory
    double *out;
};
// bytes of device scratch the call over the groups of `table` needs: 0 without a group above 8192 worlds, else at most
// 256 MiB
uint64_t topk_scratch_bytes(const TopkParams &S, const std::vector<WorldGroup> &table);
// one launch per small route that has groups, and a fixed launch sequence per slice of the large groups' tasks
// (*launches); `scratch` holds topk_scratch_bytes(S, table).  With a large group *reads (host memory) receives, once the
// stream reaches it, the reads of the planes summed over every task; it is left alone otherwise (one read per task).
cudaError_t launch_top_worlds(const TopkParams &S, const std::vector<WorldGroup> &table,
                              const std::vector<uint32_t> &order, void *scratch, int *launches,
                              unsigned long long *reads, cudaStream_t s);

// Midranks of the outcome planes (rank_kernels.cu, include/b200_sixdof.h b200_sixdof_outcome_ranks): for group g of the
// table and selected plane j, every complete world's midrank within the group (scipy.stats.rankdata(method="average")
// over the worlds whose n_p selected values are all finite, -0 == +0) into rank plane j, NaN for the other worlds.
struct RankParams {
    const double *planes;  // outcome plane 0; plane p at planes + p * ld, world w at [w]
    uint64_t ld;
    uint32_t n_p;          // selected planes
    uint32_t plane[B200_MAX_OUTCOMES];
    const WorldGroup *groups;  // the group table, in device memory
    const uint32_t *order;     // quantile_order(table), in device memory
    double *ranks;             // rank plane j at ranks + j * ld
    uint8_t *mask;             // n_worlds bytes: world complete
};
// bytes of device scratch the call over the groups of `table` needs: 0 without a group above 8192 worlds, else at most
// 256 MiB unless one (group, plane) task alone needs more (about 42 bytes per world)
uint64_t rank_scratch_bytes(const RankParams &S, const std::vector<WorldGroup> &table, const std::vector<uint32_t> &order);
// the mask launch, one launch per small route that has groups, and a fixed launch sequence per slice of the large
// groups' tasks (*launches; none without worlds); `scratch` holds rank_scratch_bytes(S, table, order).  With a large
// group *reads (host memory) receives, once the stream reaches it, the reads of the planes summed over every task; it
// is left alone otherwise (one read per task).
cudaError_t launch_ranks(const RankParams &S, uint64_t n_worlds, const std::vector<WorldGroup> &table,
                         const std::vector<uint32_t> &order, void *scratch, int *launches, unsigned long long *reads,
                         cudaStream_t s);
// G covariance records [n, mean[n_p], M[n_p][n_p]] (cov, device) into G records [n, rho[n_p][n_p]] (out, device):
// rho = M[a][b] / sqrt(M[a][a] * M[b][b]), each operation correctly rounded, NaN where n < 2 or M[a][a] or M[b][b] is
// not > 0.  One launch (*launches = 1).
cudaError_t launch_rank_correlation(const double *cov, double *out, uint64_t G, uint32_t n_p, int *launches,
                                    cudaStream_t s);
// A rank's part of a world-sharded rank call between its rounds (b200_sixdof_sharded_ranks_*): the MSD bucket pass over
// every (group, plane) task, slice by slice, each exchange's u32 words summed over the ranks before the step that reads
// them.  The exchanges, in order: the group sizes (once per call), then per slice at most 5 histograms, then per window
// of the slice's buckets their local counts and their keys; none passes sharded_rank_round_bytes() but the sizes and the
// histograms, which are sent in rounds of at most that many bytes.
struct RankShard {
    // one per task of the slice, in device scratch, copied back after every plan
    struct TaskState {
        uint32_t N;              // complete worlds over every rank
        uint32_t lcn;            // complete worlds on this rank
        uint32_t level;          // the level whose codes name the worlds' bins
        uint32_t nr[7];          // ranges of each level
        uint32_t n_buckets;      // buckets, numbered in the same order on every rank
        uint32_t bucket_worlds;  // the buckets' worlds over every rank: the task's key words
        uint32_t local_worlds;   // the buckets' worlds on this rank
        uint32_t n_pieces;       // the pieces that hold worlds of this rank
        uint32_t pad[2];
    };
    RankParams S;                   // S.ranks, S.mask: the handle's rank planes
    std::vector<WorldGroup> table;  // the rank's part of every group (only o and n are read)
    uint32_t rank = 0, n_ranks = 1;
    // device buffers, grown during the call and freed by rank_shard_free: the slices' task areas, the two level pools
    // of histograms and the words of the exchange in flight
    void *area = nullptr;
    uint64_t area_bytes = 0;
    uint32_t *pool[2] = {nullptr, nullptr};
    uint64_t pool_bytes[2] = {0, 0};
    uint32_t *x = nullptr;
    uint64_t x_bytes = 0;
    int step = 0;                   // the exchange in flight (0: none yet)
    int level = 0;                  // the histogram level of a histogram exchange
    uint64_t xbytes = 0, xpos = 0;  // its size, and where the round last sent starts
    // per group: complete worlds over every rank and on this one, and the most complete worlds and worlds one rank holds
    std::vector<uint64_t> n_global, n_local, l_most, w_most;
    std::vector<uint64_t> tasks;    // group << 32 | plane
    std::vector<uint64_t> slices;   // the first task of every slice, then the task count
    uint64_t slice = 0;
    std::vector<TaskState> st;      // the slice's task states after the last plan
    uint64_t keys = 0, wkeys = 0, window = 0;  // the slice's key words, a window's, the window in flight
    uint64_t bad_group = ~0ull;     // a group of too many complete worlds over the ranks: the call fails
    unsigned long long reads = 0;   // reads of the planes summed over the tasks
};
// the largest round of a sharded rank call in bytes, and the most complete worlds a group may hold over the ranks
uint64_t sharded_rank_round_bytes();
uint64_t sharded_rank_max_worlds();
// One round on s, returning once the round's words are in `partial` (host or device memory): the sums of the last
// round's words from `reduced` (nothing before the first round), then the launches up to the next round's words
// (*partial_bytes; 0 once the rank planes hold the midranks of the rank's worlds, or once Q.bad_group is set).
cudaError_t sharded_rank_round(RankShard &Q, const void *reduced, void *partial, uint64_t *partial_bytes, int *launches,
                               cudaStream_t s);
void rank_shard_free(RankShard &Q);

// Sobol indices of the outcome planes of a Saltelli campaign (sobol_kernels.cu, include/b200_sixdof.h
// b200_sixdof_outcome_sobol): sample j is the worlds [j (d + 2), (j + 1) (d + 2)), [A, AB^(1) .. AB^(d), B].
struct SobolParams {
    const double *planes;  // outcome plane 0; plane p at planes + p * ld_o, world w at [w]
    uint64_t ld_o;
    uint32_t n_p;          // selected outputs
    uint32_t plane[B200_MAX_OUTCOMES];
    uint32_t d;            // inputs
    uint64_t n_samples;    // n_worlds / (d + 2)
    uint64_t ld;           // n_samples rounded up to 128
    double *sp;            // derived plane j (0: a, 1: b, 2 + i: D_i) of output k at sp + (k (d + 2) + j) ld
    uint32_t *list;        // output k's complete samples at list + k ld, group g's from its first sample o
    uint8_t *mask;         // output k's completeness bytes at mask + k ld
};
// The derived planes and completeness bytes of every selected output: one launch (*launches; none without samples).
cudaError_t launch_sobol_planes(const SobolParams &S, int *launches, cudaStream_t s);
// bytes of device scratch launch_sobol_indices needs over `tasks` (group, output) tasks: at most 256 MiB unless one
// task alone needs more
uint64_t sobol_scratch_bytes(const SobolParams &S, uint64_t tasks, uint32_t n_boot);
// The records [G][n_p][3 + 4d] into out (device) from the covariance table `cov` of the derived planes ([n_p][G]
// records of 1 + q + q^2, q = d + 2, sample axis = output) over the sample-axis group table `groups` (device, G groups;
// only o and n are read).  Per slice of tasks: with n_boot > 0 the list launch and the bootstrap launch, then the finish
// launch (*launches).
cudaError_t launch_sobol_indices(const SobolParams &S, const double *cov, const WorldGroup *groups, uint64_t G,
                                 uint32_t n_boot, uint64_t seed, double *out, void *scratch, int *launches,
                                 cudaStream_t s);

} // namespace b200
