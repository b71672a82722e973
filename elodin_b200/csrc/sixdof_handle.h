// Internals of a b200_sixdof handle, shared by the translation units that implement the C ABI
// (sixdof_abi.cu: executor; sixdof_comm.cu: NCCL gather, peer-memory row sharding).
#pragma once
#include <cstdarg>
#include <cstdio>
#include <string>
#include <vector>

#include "sixdof_internal.h"

namespace b200 {

int fail(int code, const char *fmt, ...);          // sets the thread-local message, returns code
const char *last_error_message();

struct Column {
    uint64_t id;
    uint32_t width;     // f64 per body (globals: 1)
    bool global;        // tick / simulation_time_step: one 8-byte scalar, host resident
    double *dev;        // width planes of ld doubles
};

inline uint64_t round_up(uint64_t x, uint64_t m) { return (x + m - 1) / m * m; }

} // namespace b200

struct b200_sixdof {
    uint64_t serial = 0;               // unique per created handle: what a peer window remembers of its owner besides the address
    b200_sixdof_desc desc{};
    std::vector<b200_effector> effectors;
    std::vector<uint8_t *> eff_masks; // device copies of the per-effector entity masks (nullptr = all)
    std::vector<double *> eff_tables; // device tables of GRAVITY_EGM08 effectors (nullptr = none)
    int egm_eff = -1;                  // index of the GRAVITY_EGM08 effector (at most one), -1 = none
    double *aforce = nullptr;          // 9 planes of additive stage forces it fills every tick
    int device = 0;
    uint64_t n_bodies = 0;
    uint64_t ld = 0;
    std::vector<b200::Column> cols;
    std::vector<uint64_t> input_ids, output_ids;
    double sim_time_step = 0.0;   // SimulationTimeStep column value
    uint64_t tick = 0;            // Tick column value
    uint64_t ticks_done = 0;      // ticks since create / trajectory reset (trajectory slot index base)
    // graph effector
    int graph_eff = -1;
    bool graph_dense = false;
    uint32_t *row_ptr = nullptr, *col_idx = nullptr;
    uint8_t *has_edge = nullptr;
    double *gforce = nullptr;
    double *pos_alt = nullptr, *vel_alt = nullptr; // ping-pong planes of the one-launch n-body tick
    bool nbody_fused = false;                       // decided once per handle (whole-batch grid size)
    bool small_world = false;                       // <= 32 bodies per world: whole ticks in one warp, n ticks per launch
    uint32_t max_deg = 0;
    // one byte per 64-body segment (absolute body index / 64): 1 = every mass of the segment is regular for the FAST
    // signature-0 tick (body_fast_spec_kernel), 0 = unknown.  Every write of the Inertia planes clears the bytes of the
    // segments it touches first (clear_mass_class); once a raw Inertia pointer is handed out, it is never used again.
    uint8_t *mass_class = nullptr;
    bool mass_class_off = false;
    // staging for AoS <-> SoA
    double *staging = nullptr;
    uint64_t staging_bytes = 0;
    double quantile_reads = 0.0;            // reads of the planes by the last quantile call, per group
    unsigned long long quantile_read_sum = 0;  // the same, summed over the groups (written by the stream)
    double topk_reads = 0.0;                // reads of the planes by the last top-worlds call, per task
    unsigned long long topk_read_sum = 0;   // the same, summed over the tasks (written by the stream)
    double rank_reads = 0.0;                // reads of the planes by the last rank call, per task
    unsigned long long rank_read_sum = 0;   // the same, summed over the tasks (written by the stream)
    // the rank planes of the last rank call (n_p x ld_o f64, then ld_o bytes of completeness mask): allocated by the
    // first rank call, freed by set_outcomes and destroy
    double *rank_planes = nullptr;
    uint64_t rank_bytes = 0;
    // the derived planes, complete-sample lists and completeness bytes of the last Sobol call (SobolParams): allocated
    // by the first Sobol call, freed by set_outcomes and destroy; apart from the rank planes, which a sharded rank call
    // owns between its rounds
    double *sobol_planes = nullptr;
    uint64_t sobol_bytes = 0;
    // a world-sharded quantile call (b200_sixdof_sharded_quantiles_*) between begin and end: its state, the write
    // generation of the rows at begin (rows_gen: bumped by every entry that changes what a reduction reads), and its own
    // device scratch (not the staging buffer, which the other reductions reuse between its rounds)
    struct ShardedQuantiles {
        bool active = false, ready = false, outcomes = false;
        uint64_t gen = 0, partial_bytes = 0, max_round = 0, table_bytes = 0, triples = 0;
        b200::QuantileShard Q;
    } sq;
    // a world-sharded rank call (b200_sixdof_sharded_ranks_*) between begin and end: its state (which owns its device
    // scratch), the write generation of the outcome planes at begin; it fills the rank planes above, so an unsharded
    // rank call discards it
    struct ShardedRanks {
        bool active = false, ready = false, grouped = false;
        uint64_t gen = 0, partial_bytes = 0, tasks = 0;
        b200::RankShard Q;
    } sr;
    uint64_t rows_gen = 0;
    uint64_t sum_gen = 0;  // bumped by every summary start and fold: what the outcome planes are computed from
    double *sq_scratch = nullptr;
    uint64_t sq_scratch_bytes = 0;
    // the group tables of one split of the worlds, each with its device copy: the statistics' (stats_kernels.cu), the
    // quantiles' route order over the same worlds (quantile_order, quantile_kernels.cu) and the covariance's own
    // chunking (cov_group_table, cov_kernels.cu)
    struct GroupTables {
        std::vector<b200::WorldGroup> stats, cov;
        std::vector<uint32_t> order;
        b200::WorldGroup *stats_dev = nullptr, *cov_dev = nullptr;
        uint32_t *order_dev = nullptr;
    };
    // indexed by `grouped`: all worlds as one group (built at creation), then the groups of b200_sixdof_set_world_groups
    // (sizes empty = none set)
    GroupTables tables[2];
    std::vector<uint64_t> group_sizes;
    // trajectory
    double *traj = nullptr;
    uint32_t traj_planes = 13;   // 25 with B200_TRAJ_FULL
    // derived channels (b200_sixdof_set_channels): the channel set and its planes, [capacity][n_c][ld] for the ring and
    // [n_c][ld] for the state, recomputed by every entry that reads them (channel_kernels.cu)
    std::vector<b200_channel> channels;
    double *chan_ring = nullptr, *chan_state = nullptr;
    // outcomes (b200_sixdof_set_outcomes): the set (values pointers cleared) and its planes, P of ld_o f64 (VALUES planes
    // written once by set_outcomes, the others by every outcome entry, outcome_kernels.cu); with n_entities != 1 the
    // outcome entries reduce over group tables of one entity of their own, indexed like `tables` and built only once
    // outcomes are set
    std::vector<b200_outcome> outcomes;
    double *out_planes = nullptr;
    uint64_t ld_o = 0;
    GroupTables out_tables[2];
    // run summaries (b200_sixdof_summary_*): device accumulators, allocated on first use, kept across begins
    bool sum_begun = false;
    bool sum_ever = false;           // summary_begin has been called: the channel set (the row width) is fixed
    bool sum_extrema = false;
    std::vector<b200_threshold> sum_thr_list;
    double *sum_ext = nullptr;       // 5 R planes of ld, R = 25 + channels (SummaryParams::ext)
    double *sum_thr = nullptr;       // [n_worlds][thresholds][26] (SummaryParams::thr)
    uint64_t sum_thr_bytes = 0;
    std::vector<uint32_t> sum_mom_planes;     // selected moment planes, in table order
    std::vector<b200_threshold> sum_dwell_list;
    double *sum_mom = nullptr;       // 4 planes of ld per selected plane (SummaryParams::mom)
    uint64_t sum_mom_bytes = 0;
    double *sum_dwell = nullptr;     // [n_worlds][dwells][3] (SummaryParams::dwell)
    uint64_t sum_dwell_bytes = 0;
    // plumbing
    cudaStream_t stream = nullptr;
    bool own_stream = true;
    // pipelined invoke_batch: copy engines on their own streams, whole-batch AoS staging
    cudaStream_t copy_in = nullptr, copy_out = nullptr;
    double *stage_in = nullptr, *stage_out = nullptr;
    uint64_t stage_in_bytes = 0, stage_out_bytes = 0;
    std::vector<cudaEvent_t> chunk_in, chunk_out;
    // small batches: packed pinned host staging (one PCIe transfer per direction)
    uint8_t *host_pack = nullptr;
    uint64_t host_pack_bytes = 0;
    cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}; // [0,1] H2D span, [2,3] compute span, [4,5] D2H span
    int status = B200_OK;
    b200_timings timings{};

    b200::Column *find(uint64_t id)
    {
        for (auto &c : cols) if (c.id == id) return &c;
        return nullptr;
    }
    const b200::Column *find(uint64_t id) const
    {
        for (auto &c : cols) if (c.id == id) return &c;
        return nullptr;
    }
};


namespace b200 {

int cuda_fail(b200_sixdof *h, cudaError_t e, const char *what);
int ensure_staging(b200_sixdof *h, uint64_t bytes);
// Every plane base, constant and effector of the handle, as the body kernels see bodies [b0, b0 + nb): each per-body
// plane base starts at body b0; rows inside a world keep their index.
StepParams range_step_params(b200_sixdof *h, uint64_t b0, uint64_t nb);
// The edge_fold gravity launch over the planes of P: the graph effector's kind and constants, the CSR arrays and the
// integrator, for n_worlds worlds starting where P starts.
GraphParams graph_params(const b200_sixdof *h, const StepParams &P, uint64_t n_worlds);

#define CU(h, call)                                                        \
    do {                                                                   \
        cudaError_t e_ = (call);                                           \
        if (e_ != cudaSuccess) return b200::cuda_fail((h), e_, #call);     \
    } while (0)

// Grow-only device buffer: *ptr holds at least need_bytes afterwards (its content is not kept).  need > have >= 0, so
// nothing is ever allocated with 0 bytes.
inline int grow_device(b200_sixdof *h, double **ptr, uint64_t *have_bytes, uint64_t need_bytes)
{
    if (*have_bytes >= need_bytes) return B200_OK;
    if (*ptr) CU(h, cudaFree(*ptr));
    *ptr = nullptr;
    *have_bytes = 0;
    CU(h, cudaMalloc(ptr, need_bytes));
    *have_bytes = need_bytes;
    return B200_OK;
}

// Is p device memory (of any GPU; *device receives which)?  Host pointers the runtime has never seen make the query
// fail: that error is cleared here, not left for the next call to find.
inline bool is_device_pointer(const void *p, int *device = nullptr)
{
    cudaPointerAttributes a{};
    const bool dev = cudaPointerGetAttributes(&a, p) == cudaSuccess && a.type == cudaMemoryTypeDevice;
    (void)cudaGetLastError();
    if (dev && device) *device = a.device;
    return dev;
}

// n ticks happened: the trajectory slot base, the Tick column and the tick counter of the timings.
inline void advance_ticks(b200_sixdof *h, uint64_t n)
{
    ++h->rows_gen;
    h->ticks_done += n;
    h->tick += n;
    h->timings.ticks += n;
}

} // namespace b200
