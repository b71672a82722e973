// Host runtime + C ABI of libb200_sixdof (include/b200_sixdof.h).
//
// Replaces CraneliftExec (libs/nox-py/src/cranelift_exec.rs:54-195) on the
// six_dof() path: owns device-resident SoA columns, maps the reference's host
// column buffers in and out, and drives the sm_90a kernels.  There is no CPU
// fallback anywhere in this file: without a CUDA device every entry point fails
// with B200_ERR_NO_DEVICE.
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cctype>
#include <chrono>
#include <map>
#include <mutex>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "sixdof_handle.h"

using namespace b200;

namespace b200 {

static thread_local std::string g_last_error = "";

int fail(int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

const char *last_error_message() { return g_last_error.c_str(); }

int cuda_fail(b200_sixdof *h, cudaError_t e, const char *what)
{
    if (h) h->status = B200_ERR_CUDA;
    return fail(e == cudaErrorMemoryAllocation ? B200_ERR_OUT_OF_MEMORY : B200_ERR_CUDA, "CUDA error in %s: %s", what,
                cudaGetErrorString(e));
}

int ensure_staging(b200_sixdof *h, uint64_t bytes) { return grow_device(h, &h->staging, &h->staging_bytes, bytes); }

} // namespace b200

namespace {

thread_local b200_sixdof *g_tick_handle = nullptr;

uint64_t column_bytes(const b200_sixdof *h, const Column &c)
{
    return c.global ? 8ull : h->n_bodies * c.width * 8ull;
}

// The reference's free six_dof() system has inputs (first-init order)
//   tick, force, inertia, world_pos, world_accel, simulation_time_step, world_vel
// (SURVEY §8a-7, cranelift-mlir/tests/three_body_e2e.rs:15-16); effector
// columns are inserted after `force` in effector order.  Outputs are every
// variable of the builder, ordered by ComponentId (BTreeMap, system.rs).
void build_id_tables(b200_sixdof *h)
{
    std::vector<uint64_t> in = {B200_ID_TICK, B200_ID_FORCE};
    for (auto &e : h->effectors)
        if (e.column_id && std::find(in.begin(), in.end(), e.column_id) == in.end()) in.push_back(e.column_id);
    for (uint64_t id : {B200_ID_INERTIA, B200_ID_WORLD_POS, B200_ID_WORLD_ACCEL, B200_ID_SIMULATION_TIME_STEP,
                        B200_ID_WORLD_VEL})
        if (std::find(in.begin(), in.end(), id) == in.end()) in.push_back(id);
    h->input_ids = in;
    h->output_ids = in;
    std::sort(h->output_ids.begin(), h->output_ids.end());
}

int add_column(b200_sixdof *h, uint64_t id, uint32_t width, bool global)
{
    if (h->find(id)) return B200_OK;
    Column c{id, width, global, nullptr};
    if (!global && h->n_bodies) {
        const uint64_t bytes = (uint64_t)width * h->ld * 8ull;
        CU(h, cudaMalloc(&c.dev, bytes));
        CU(h, cudaMemsetAsync(c.dev, 0, bytes, h->stream));
    }
    h->cols.push_back(c);
    return B200_OK;
}

// Derived tables of the EGM08 recursion (python/elodin/egm08.py:84-144) — the same formulas, operation for operation,
// as the test oracle's orc_egm08_tables, so both sides evaluate the series on bit-identical constants — emitted as ONE
// stream in the order egm08_field consumes it: column by column (m = 0..L), degree by degree (l = m..L), eight doubles
// per term:
//   [0] the A recursion's first constant: diag[m] (l = m), offc[l] (l = m+1), n1[l][m] otherwise      [1] n2[l][m] or 0
//   [2] the same for B at (l+1, m+1): diag[m+1], offc[l+1], n1[l+1][m+1], or 0 beyond degree L         [3] n2[l+1][m+1] or 0
//   [4] C[l][m]   [5] S[l][m]   [6] nq1[l][m]   [7] nq2[l][m]
// so a warp reads the 137 KB of a degree-64 field front to back, 64 contiguous bytes per term.
double kdelta(int d) { return d == 0 ? 1.0 : 2.0; }

std::vector<double> egm08_tables(int L, const double *c_bar, const double *s_bar)
{
    const int n = L + 1;
    std::vector<double> n1((size_t)n * n, 0.0), n2((size_t)n * n, 0.0), nq1((size_t)n * n, 0.0), nq2((size_t)n * n, 0.0), diag(n), offc(n);
    for (int l = 0; l <= L; ++l)
        for (int m = 0; m <= L; ++m) {
            double v1 = 0.0, v2 = 0.0;
            if (l >= m + 2) {
                v1 = std::sqrt((double)((2 * l + 1) * (2 * l - 1)) / (double)((l + m) * (l - m)));
                v2 = std::sqrt((double)((l + m - 1) * (l - m - 1) * (2 * l + 1)) / (double)((2 * l - 3) * (l + m) * (l - m)));
            }
            n1[l * n + m] = v1;
            n2[l * n + m] = v2;
            const double num1 = (double)(l - m) * kdelta(m) * (double)(l + m + 1);
            nq1[l * n + m] = num1 < 0.0 ? 0.0 : std::sqrt(num1 / kdelta(m + 1));
            const double num2 = (double)(l + m + 2) * (double)(l + m + 1) * (double)(2 * l + 1) * kdelta(m);
            nq2[l * n + m] = num2 < 0.0 ? 0.0 : std::sqrt(num2 / ((double)(2 * l + 3) * kdelta(m + 1)));
        }
    double cur = 1.0;
    for (int l = 0; l <= L; ++l) {
        if (l > 0) cur = cur * std::sqrt(((double)(2 * l + 1) * kdelta(l)) / ((double)(2 * l) * kdelta(l - 1)));
        diag[l] = cur;
        offc[l] = l == 0 ? 0.0 : diag[l] * std::sqrt(((double)(2 * l) * kdelta(l - 1)) / kdelta(l));
    }
    std::vector<double> t;
    t.reserve((size_t)4 * n * (n + 1));
    for (int m = 0; m <= L; ++m)
        for (int l = m; l <= L; ++l) {
            const int l1 = l + 1, m1 = m + 1;
            const bool b_live = m1 <= L && l1 <= L;
            t.push_back(l == m ? diag[m] : l == m + 1 ? offc[l] : n1[l * n + m]);
            t.push_back(l >= m + 2 ? n2[l * n + m] : 0.0);
            t.push_back(!b_live ? 0.0 : l1 == m1 ? diag[m1] : l1 == m1 + 1 ? offc[l1] : n1[l1 * n + m1]);
            t.push_back(b_live && l1 >= m1 + 2 ? n2[l1 * n + m1] : 0.0);
            t.push_back(c_bar[l * n + m]);
            t.push_back(s_bar[l * n + m]);
            t.push_back(nq1[l * n + m]);
            t.push_back(nq2[l * n + m]);
        }
    return t;
}

int build_graph(b200_sixdof *h, const b200_effector &e)
{
    const uint32_t N = (uint32_t)h->desc.n_entities;
    std::vector<uint32_t> row(N + 1, 0), col;
    std::vector<std::vector<uint32_t>> adj(N);
    for (uint64_t k = 0; k < e.n_edges; ++k) {
        const uint32_t a = e.edge_from[k], b = e.edge_to[k];
        if (a >= N || b >= N) return fail(B200_ERR_INVALID_ARGUMENT, "edge %llu (%u -> %u) out of range (n_entities=%u)",
                                          (unsigned long long)k, a, b, N);
        adj[a].push_back(b); // spawn order preserved per source (graph.rs:194-197)
    }
    std::vector<uint8_t> has(N ? N : 1, 0);
    bool dense = N > 1;
    for (uint32_t i = 0; i < N; ++i) {
        row[i + 1] = row[i] + (uint32_t)adj[i].size();
        col.insert(col.end(), adj[i].begin(), adj[i].end());
        has[i] = !adj[i].empty();
        if (adj[i].size() != N - 1) dense = false;
        else {
            uint32_t want = 0;
            for (uint32_t t : adj[i]) { if (want == i) ++want; if (t != want) { dense = false; break; } ++want; }
        }
    }
    h->graph_dense = dense;
    for (uint32_t i = 0; i < N; ++i) h->max_deg = std::max<uint32_t>(h->max_deg, (uint32_t)adj[i].size());
    CU(h, cudaMalloc(&h->row_ptr, (N + 1) * sizeof(uint32_t)));
    CU(h, cudaMalloc(&h->col_idx, std::max<size_t>(col.size(), 1) * sizeof(uint32_t)));
    CU(h, cudaMalloc(&h->has_edge, has.size()));
    CU(h, cudaMemcpy(h->row_ptr, row.data(), (N + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice));
    if (!col.empty()) CU(h, cudaMemcpy(h->col_idx, col.data(), col.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    CU(h, cudaMemcpy(h->has_edge, has.data(), has.size(), cudaMemcpyHostToDevice));
    CU(h, cudaMalloc(&h->gforce, 9ull * h->ld * 8ull));
    CU(h, cudaMemset(h->gforce, 0, 9ull * h->ld * 8ull));
    if (h->desc.math_mode == B200_MATH_FAST && dense) {
        CU(h, cudaMalloc(&h->pos_alt, 7ull * h->ld * 8ull));
        CU(h, cudaMalloc(&h->vel_alt, 6ull * h->ld * 8ull));
        CU(h, cudaMemset(h->pos_alt, 0, 7ull * h->ld * 8ull));
        CU(h, cudaMemset(h->vel_alt, 0, 6ull * h->ld * 8ull));
    }
    return B200_OK;
}

} // namespace

namespace b200 {

StepParams range_step_params(b200_sixdof *h, uint64_t b0, uint64_t nb)
{
    StepParams P;
    std::memset(&P, 0, sizeof P);
    P.pos = h->find(B200_ID_WORLD_POS)->dev;
    P.vel = h->find(B200_ID_WORLD_VEL)->dev;
    P.acc = h->find(B200_ID_WORLD_ACCEL)->dev;
    P.frc = h->find(B200_ID_FORCE)->dev;
    P.ine = h->find(B200_ID_INERTIA)->dev;
    P.gforce = h->gforce;
    P.has_edge = h->has_edge;
    P.aforce = h->aforce;
    P.ld = h->ld;
    P.n_bodies = nb;
    P.n_entities = (uint32_t)h->desc.n_entities;
    P.n_eff = (uint32_t)h->effectors.size();
    P.dt_stage = h->sim_time_step;
    P.dt_final = std::isnan(h->desc.time_step) ? h->sim_time_step : h->desc.time_step;
    P.traj = h->traj;
    P.traj_capacity = h->desc.trajectory_capacity;
    P.traj_every = h->traj ? h->desc.trajectory_every : 0;
    P.traj_planes = h->traj_planes;
    for (size_t i = 0; i < h->effectors.size(); ++i) {
        const b200_effector &e = h->effectors[i];
        P.eff[i].kind = e.kind;
        P.eff[i].flags = e.flags;
        std::memcpy(P.eff[i].p, e.p, sizeof e.p);
        const Column *c = e.column_id ? h->find(e.column_id) : nullptr;
        P.eff[i].col = c ? c->dev : nullptr;
        P.eff[i].col_width = c ? c->width : 0;
        P.eff[i].mask = i < h->eff_masks.size() ? h->eff_masks[i] : nullptr;
        P.eff[i].table = i < h->eff_tables.size() ? h->eff_tables[i] : nullptr;
    }
    P.pos += b0; P.vel += b0; P.acc += b0; P.frc += b0; P.ine += b0;
    if (P.gforce) P.gforce += b0;
    if (P.aforce) P.aforce += b0;
    if (P.traj) P.traj += b0;
    for (uint32_t i = 0; i < P.n_eff; ++i) if (P.eff[i].col) P.eff[i].col += b0;
    return P;
}

GraphParams graph_params(const b200_sixdof *h, const StepParams &P, uint64_t n_worlds)
{
    const b200_effector &e = h->effectors[h->graph_eff];
    GraphParams G{};
    G.pos = P.pos; G.vel = P.vel; G.ine = P.ine;
    G.gforce = const_cast<double *>(P.gforce); // the planes the fold writes are the ones the body step then reads
    G.ld = h->ld; G.n_entities = P.n_entities; G.n_worlds = (uint32_t)n_worlds;
    G.dt_stage = P.dt_stage; G.kind = e.kind; G.integrator = h->desc.integrator;
    G.p0 = e.p[0]; G.p1 = e.p[1]; G.row_ptr = h->row_ptr; G.col_idx = h->col_idx; G.max_deg = h->max_deg;
    return G;
}

} // namespace b200

namespace {

// The EGM08 stage-force launch over the planes of P (one per tick, before the body launch that adds its forces).
EgmParams egm_params(const b200_sixdof *h, const StepParams &P)
{
    const b200_effector &e = h->effectors[h->egm_eff];
    EgmParams E{};
    E.pos = P.pos; E.vel = P.vel; E.ine = P.ine;
    E.aforce = const_cast<double *>(P.aforce); // written here, read by the body step
    E.table = h->eff_tables[h->egm_eff]; E.mask = h->eff_masks[h->egm_eff];
    E.ld = h->ld; E.n_bodies = P.n_bodies; E.n_entities = P.n_entities; E.ent0 = P.ent0;
    E.L = (uint32_t)e.p[2]; E.integrator = h->desc.integrator; E.mu = e.p[0]; E.r_ref = e.p[1]; E.dt_stage = P.dt_stage;
    return E;
}

// Integrate n_ticks ticks of the worlds [w0, w0+nw) on `stream`.  Worlds are independent, so a
// world range can run to completion before the next one starts (used by the pipelined
// invoke_batch); counters are the caller's business.
int launch_ticks(b200_sixdof *h, uint64_t w0, uint64_t nw, uint64_t n_ticks, cudaStream_t stream)
{
    const uint64_t N = h->desc.n_entities;
    const uint64_t b0 = w0 * N, nb = nw * N;
    if (n_ticks == 0 || nb == 0) return B200_OK;
    StepParams P = range_step_params(h, b0, nb);
    // the summary's segments must be the launch's warps of pairs: only a range that starts on a segment boundary uses it
    P.mass_class = (!h->mass_class_off && b0 % 64 == 0) ? h->mass_class + b0 / 64 : nullptr;
    const bool exact = h->desc.math_mode == B200_MATH_EXACT;
    const bool graph = h->graph_eff >= 0;
    const bool egm = h->egm_eff >= 0; // its stage forces are a function of the tick's input state: one launch per tick
    const uint64_t fuse = ((graph && !h->small_world) || egm) ? 1 : std::max<uint32_t>(1u, h->desc.max_fused_ticks);
    uint64_t left = n_ticks, done = 0;
    double *pos_next = h->pos_alt ? h->pos_alt + b0 : nullptr, *vel_next = h->vel_alt ? h->vel_alt + b0 : nullptr;
    while (left) {
        const uint64_t n = std::min(left, fuse);
        if (egm) {
            CU(h, launch_egm08_force(egm_params(h, P), (int)h->desc.math_mode, stream));
            h->timings.kernel_launches++;
        }
        if (graph) {
            const GraphParams G = graph_params(h, P, nw); // of the planes live now: the fused route swaps them every tick
            if (h->small_world) {
                // gravity through warp shuffles + integration, n ticks in one launch, state in registers
                P.n_ticks = (uint32_t)n;
                P.tick0 = h->ticks_done + done;
                P.write_fa = (exact || left == n) ? 1u : 0u;
                CU(h, launch_small_world(G, P, (int)h->desc.math_mode, stream));
                h->timings.kernel_launches++;
                done += n;
                left -= n;
                continue;
            }
            if (h->nbody_fused) {
                // gravity + integration in one launch; the new state lands in the other plane set
                P.n_ticks = 1;
                P.tick0 = h->ticks_done + done;
                P.write_fa = (left == 1) ? 1u : 0u;
                CU(h, launch_nbody_tick_fused(G, P, pos_next, vel_next, stream));
                h->timings.kernel_launches++;
                std::swap(P.pos, pos_next);
                std::swap(P.vel, vel_next);
                done += 1;
                left -= 1;
                continue;
            }
            CU(h, launch_graph_force(G, h->desc.math_mode, h->graph_dense, stream));
            h->timings.kernel_launches++;
        }
        P.n_ticks = (uint32_t)n;
        P.tick0 = h->ticks_done + done;
        P.write_fa = (exact || left == n) ? 1u : 0u; // Force/WorldAccel are only host-visible after the batch
        P.reverse = (uint32_t)(h->timings.kernel_launches & 1u); // alternate the traversal direction launch to launch
        CU(h, launch_body_step(P, (int)h->desc.integrator, (int)h->desc.math_mode, stream));
        h->timings.kernel_launches++;
        done += n;
        left -= n;
    }
    return B200_OK;
}

// After every world range has advanced n_ticks through the one-launch n-body tick, the live pose /
// velocity planes are the "other" set when n_ticks is odd: make them the columns' planes.
void commit_ping_pong(b200_sixdof *h, uint64_t n_ticks)
{
    if (!h->nbody_fused || !(n_ticks & 1) || h->n_bodies == 0) return;
    std::swap(h->find(B200_ID_WORLD_POS)->dev, h->pos_alt);
    std::swap(h->find(B200_ID_WORLD_VEL)->dev, h->vel_alt);
}

int do_step(b200_sixdof *h, uint64_t n_ticks)
{
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    int rc = launch_ticks(h, 0, h->desc.n_worlds, n_ticks, h->stream);
    if (rc) return rc;
    commit_ping_pong(h, n_ticks);
    advance_ticks(h, n_ticks);
    return B200_OK;
}

// Forget what the mass-class summary knows about every segment that overlaps bodies [b0, b0 + n): their Inertia is
// about to be written.  Stream-ordered before that write and after every launch already queued.
int clear_mass_class(b200_sixdof *h, uint64_t b0, uint64_t n)
{
    if (n == 0) return B200_OK;
    const uint64_t s0 = b0 / 64, s1 = (b0 + n + 63) / 64;
    CU(h, cudaMemsetAsync(h->mass_class + s0, 0, s1 - s0, h->stream));
    return B200_OK;
}

int do_upload(b200_sixdof *h, uint64_t id, const void *src, uint64_t bytes)
{
    ++h->rows_gen;
    Column *c = h->find(id);
    if (!c) return fail(B200_ERR_COMPONENT_NOT_FOUND, "component not found: 0x%016llx", (unsigned long long)id);
    if (bytes != column_bytes(h, *c))
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "component value had wrong size: 0x%016llx has %llu bytes, got %llu",
                    (unsigned long long)id, (unsigned long long)column_bytes(h, *c), (unsigned long long)bytes);
    if (!src) return fail(B200_ERR_INVALID_ARGUMENT, "null source buffer");
    const bool device = is_device_pointer(src);
    if (c->global) {
        // the two globals are 8-byte scalars the handle keeps on the host (Globals entity, world.rs:174-191); a device
        // buffer is read on the handle's stream, after the work already queued there
        uint64_t raw;
        if (device) {
            CU(h, cudaMemcpyAsync(&raw, src, 8, cudaMemcpyDefault, h->stream));
            CU(h, cudaStreamSynchronize(h->stream));
        } else {
            std::memcpy(&raw, src, 8);
        }
        if (id == B200_ID_TICK) h->tick = raw;
        else std::memcpy(&h->sim_time_step, &raw, 8);
        return B200_OK;
    }
    if (bytes == 0) return B200_OK;
    int rc = ensure_staging(h, bytes);
    if (rc) return rc;
    if (id == B200_ID_INERTIA && (rc = clear_mass_class(h, 0, h->n_bodies))) return rc;
    CU(h, cudaMemcpyAsync(h->staging, src, bytes, cudaMemcpyDefault, h->stream));
    CU(h, launch_aos_to_soa(h->staging, c->dev, h->n_bodies, c->width, h->ld, h->stream));
    h->timings.kernel_launches++;
    // a host source is the caller's again when this returns: the copy out of it must have happened
    if (!device) CU(h, cudaStreamSynchronize(h->stream));
    return B200_OK;
}

int do_download(b200_sixdof *h, uint64_t id, void *dst, uint64_t bytes)
{
    Column *c = h->find(id);
    if (!c) return fail(B200_ERR_COMPONENT_NOT_FOUND, "component not found: 0x%016llx", (unsigned long long)id);
    if (bytes != column_bytes(h, *c))
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "component value had wrong size: 0x%016llx has %llu bytes, got %llu",
                    (unsigned long long)id, (unsigned long long)column_bytes(h, *c), (unsigned long long)bytes);
    if (!dst) return fail(B200_ERR_INVALID_ARGUMENT, "null destination buffer");
    if (c->global) {
        uint64_t raw;
        if (id == B200_ID_TICK) raw = h->tick;
        else std::memcpy(&raw, &h->sim_time_step, 8);
        if (is_device_pointer(dst)) { // written on the handle's stream, after the work already queued there
            CU(h, cudaMemcpyAsync(dst, &raw, 8, cudaMemcpyDefault, h->stream));
            CU(h, cudaStreamSynchronize(h->stream));
        } else {
            std::memcpy(dst, &raw, 8);
        }
        return B200_OK;
    }
    if (bytes == 0) return B200_OK;
    int rc = ensure_staging(h, bytes);
    if (rc) return rc;
    CU(h, launch_soa_to_aos(c->dev, h->staging, h->n_bodies, c->width, h->ld, h->stream));
    h->timings.kernel_launches++;
    CU(h, cudaMemcpyAsync(dst, h->staging, bytes, cudaMemcpyDefault, h->stream));
    // the staging buffer is reused by the next transfer; the copy must have left it first
    CU(h, cudaStreamSynchronize(h->stream));
    return B200_OK;
}

float ev_ms(cudaEvent_t a, cudaEvent_t b)
{
    float ms = 0.f;
    cudaEventElapsedTime(&ms, a, b);
    return ms;
}

} // namespace

// ===================================================================== C ABI

extern "C" {

uint64_t b200_component_id(const char *name)
{
    uint64_t h = 0xcbf29ce484222325ull; // FNV-1a 64 offset basis
    if (name)
        for (const unsigned char *p = (const unsigned char *)name; *p; ++p) { h ^= *p; h *= 0x100000001b3ull; }
    return h & ~(1ull << 63); // types.rs:43
}

const char *b200_last_error(void) { return last_error_message(); }

int b200_device_count(void)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) { (void)cudaGetLastError(); return -fail(B200_ERR_NO_DEVICE, "no CUDA device: %s", cudaGetErrorString(e)); }
    return n;
}

void *b200_host_alloc(uint64_t bytes)
{
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
        fail(B200_ERR_OUT_OF_MEMORY, "cudaHostAlloc(%llu) failed: %s", (unsigned long long)bytes,
             cudaGetErrorString(cudaGetLastError()));
        return nullptr;
    }
    return p;
}

// NUMA node of a GPU's PCIe root: /sys/bus/pci/devices/<domain:bus:dev.fn>/numa_node
int b200_device_numa_node(int device)
{
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { (void)cudaGetLastError(); return -1; }
    for (char *c = bus; *c; ++c) *c = (char)std::tolower((unsigned char)*c);
    char path[128];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE *f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

// NUMA node the first page of a host buffer lives on (move_pages query), -1 if unknown
int b200_host_node_of(const void *p)
{
#ifdef SYS_move_pages
    void *page = (void *)((uintptr_t)p & ~(uintptr_t)4095);
    int status = -1;
    if (syscall(SYS_move_pages, 0, 1ul, &page, nullptr, &status, 0) == 0) return status;
#endif
    return -1;
}

namespace {
std::mutex g_local_mu;
std::map<void *, size_t> g_local_allocs; // b200_host_alloc_local blocks: base -> mapped length
}

// Page-locked host memory on the NUMA node of `device`'s PCIe root: anonymous mapping, mbind(MPOL_BIND) to that
// node, first touch, cudaHostRegister.  With 4 GPUs per socket moving ~100 GB/s each way, buffers that sit on the
// other socket (or interleaved) make the inter-socket link the bottleneck.  Falls back to b200_host_alloc when the
// node is unknown or the policy cannot be applied.
void *b200_host_alloc_local(uint64_t bytes, int device)
{
    if (device < 0 && cudaGetDevice(&device) != cudaSuccess) { (void)cudaGetLastError(); return b200_host_alloc(bytes); }
    const int node = b200_device_numa_node(device);
    if (node < 0 || node >= 1024) return b200_host_alloc(bytes);
    const size_t len = (size_t)round_up(std::max<uint64_t>(bytes, 1), 2ull << 20);
    void *p = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (p == MAP_FAILED) return b200_host_alloc(bytes);
#ifdef SYS_mbind
    unsigned long mask[16] = {0};
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    if (syscall(SYS_mbind, p, len, 2 /* MPOL_BIND */, mask, sizeof mask * 8, 0u) != 0) {
        munmap(p, len); // the node is not in this process's allowed set: plain first-touch allocation instead
        return b200_host_alloc(bytes);
    }
#endif
    std::memset(p, 0, len); // first touch under the policy
    if (cudaHostRegister(p, len, cudaHostRegisterDefault) != cudaSuccess) {
        (void)cudaGetLastError();
        munmap(p, len);
        return b200_host_alloc(bytes);
    }
    std::lock_guard<std::mutex> lock(g_local_mu);
    g_local_allocs[p] = len;
    return p;
}

void b200_host_free(void *p)
{
    if (!p) return;
    {
        std::lock_guard<std::mutex> lock(g_local_mu);
        auto it = g_local_allocs.find(p);
        if (it != g_local_allocs.end()) {
            cudaHostUnregister(p);
            munmap(p, it->second);
            g_local_allocs.erase(it);
            return;
        }
    }
    cudaFreeHost(p);
}

// Everything of b200_sixdof_create that needs the handle: the stream and events, the effectors' validation, every
// device allocation.  On failure the caller destroys the handle, which frees whatever was allocated by then.
static int init_handle(b200_sixdof *h, const b200_sixdof_desc *d);

static int build_group_tables(b200_sixdof *h, const uint64_t *sizes, uint32_t n_groups, bool grouped);

int b200_sixdof_create(const b200_sixdof_desc *d, b200_sixdof **out)
{
    if (!d || !out) return fail(B200_ERR_INVALID_ARGUMENT, "null descriptor / out pointer");
    *out = nullptr;
    if (d->abi_version != B200_SIXDOF_ABI_VERSION)
        return fail(B200_ERR_INVALID_ARGUMENT, "ABI version mismatch: library %u, caller %u", B200_SIXDOF_ABI_VERSION,
                    d->abi_version);
    if (d->integrator > B200_INTEGRATOR_SEMI_IMPLICIT) return fail(B200_ERR_UNSUPPORTED, "unknown integrator %u", d->integrator);
    if (d->math_mode > B200_MATH_FAST) return fail(B200_ERR_UNSUPPORTED, "unknown math mode %u", d->math_mode);
    if (d->n_effectors > B200_MAX_EFFECTORS) return fail(B200_ERR_UNSUPPORTED, "too many effectors (%u > %u)", d->n_effectors, B200_MAX_EFFECTORS);
    if (d->n_effectors && !d->effectors) return fail(B200_ERR_INVALID_ARGUMENT, "n_effectors > 0 but effectors is null");
    if (d->n_worlds == 0) return fail(B200_ERR_INVALID_ARGUMENT, "n_worlds must be >= 1");
    if (d->n_entities > 0xffffffffull || d->n_worlds > 0xffffffffull) return fail(B200_ERR_UNSUPPORTED, "n_entities / n_worlds exceed 2^32-1");
    if ((d->trajectory_flags & ~(uint32_t)B200_TRAJ_FULL) || d->reserved0)
        return fail(B200_ERR_INVALID_ARGUMENT, "unknown trajectory_flags 0x%x / non-zero reserved field", d->trajectory_flags);
    if (!(d->sim_time_step > 0.0) || !std::isfinite(d->sim_time_step))
        return fail(B200_ERR_INVALID_ARGUMENT, "invalid time step: %g", d->sim_time_step); // Error::InvalidTimeStep

    int ndev = b200_device_count();
    if (ndev <= 0) return fail(B200_ERR_NO_DEVICE, "no CUDA device visible; this library has no CPU fallback");
    int dev = d->device;
    if (dev < 0) { if (cudaGetDevice(&dev) != cudaSuccess) dev = 0; }
    if (dev >= ndev) return fail(B200_ERR_INVALID_ARGUMENT, "device %d out of range (%d devices)", dev, ndev);

    b200_sixdof *h = new (std::nothrow) b200_sixdof();
    if (!h) return fail(B200_ERR_OUT_OF_MEMORY, "out of host memory");
    static std::atomic<uint64_t> next_serial{1};
    h->serial = next_serial.fetch_add(1);
    h->desc = *d;
    h->device = dev;
    h->effectors.assign(d->effectors, d->effectors + d->n_effectors);
    h->desc.effectors = nullptr;
    h->n_bodies = d->n_entities * d->n_worlds;
    h->ld = round_up(std::max<uint64_t>(h->n_bodies, 1), 128); // whole 128-body tiles inside every plane
    h->sim_time_step = d->sim_time_step;

    int rc = init_handle(h, d);
    if (!rc)  // the ungrouped reductions' one-group tables {n_worlds}, on the device for the handle's life
        rc = build_group_tables(h, &h->desc.n_worlds, 1, false);
    if (rc) { b200_sixdof_destroy(h); return rc; }
    *out = h;
    return B200_OK;
}

static int init_handle(b200_sixdof *h, const b200_sixdof_desc *d)
{
    int rc = B200_OK;
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (auto &e : h->ev) CU(h, cudaEventCreate(&e));

    // validate effectors
    int n_drag = 0, n_frame = 0;
    for (size_t i = 0; i < h->effectors.size(); ++i) {
        b200_effector &e = h->effectors[i];
        uint32_t want_w = 0;
        switch (e.kind) {
        case B200_EFF_GRAVITY_CONST: case B200_EFF_GRAVITY_FRAME: want_w = 0; break;
        case B200_EFF_DRAG_QUADRATIC: want_w = 3; ++n_drag; break;
        case B200_EFF_THRUST_BODY: want_w = 1; break;
        case B200_EFF_WRENCH_BODY: case B200_EFF_WRENCH_WORLD: want_w = 6; break;
        case B200_EFF_GRAVITY_J2: want_w = 0; break;
        case B200_EFF_GRAVITY_EGM08: {
            want_w = 0;
            const double Ld = e.p[2];
            if (!(Ld >= 0.0) || Ld > 128.0 || Ld != std::floor(Ld))
                return fail(B200_ERR_INVALID_ARGUMENT, "effector %zu: EGM08 max_degree must be an integer in 0..128 (got %g)", i, Ld);
            const uint64_t n = (uint64_t)Ld + 1;
            if (!e.table0 || !e.table1 || e.table_len != n * n)
                return fail(B200_ERR_VALUE_SIZE_MISMATCH, "effector %zu: EGM08 needs C and S tables of (L+1)^2 = %llu f64 (got %llu)", i,
                            (unsigned long long)(n * n), (unsigned long long)e.table_len);
            if (h->egm_eff >= 0) return fail(B200_ERR_UNSUPPORTED, "only one EGM08 gravity effector is supported");
            h->egm_eff = (int)i;
            break;
        }
        case B200_EFF_TORQUE_BODY_FOLD:
            want_w = e.column_width; // 3 per wheel
            if (e.column_width == 0 || e.column_width % 3 != 0 || e.column_width > 24)
                return fail(B200_ERR_VALUE_SIZE_MISMATCH, "effector %zu: a wheel-torque column holds 3 f64 per wheel, 1..8 wheels (got width %u)", i, e.column_width);
            break;
        case B200_EFF_GRAVITY_EDGES_NEWTON: case B200_EFF_GRAVITY_EDGES_SOFTENED:
            if (h->graph_eff >= 0) return fail(B200_ERR_UNSUPPORTED, "only one edge_fold gravity effector is supported");
            if (e.n_edges && (!e.edge_from || !e.edge_to)) return fail(B200_ERR_INVALID_ARGUMENT, "edge arrays are null");
            // the fold's members are the sources of its edges: a mask would define a membership the reference lacks
            if (e.entity_mask)
                return fail(B200_ERR_UNSUPPORTED, "effector %zu: an edge_fold gravity effector takes no entity mask", i);
            if (d->math_mode == B200_MATH_FAST && i != 0)
                return fail(B200_ERR_UNSUPPORTED, "FAST math: the edge_fold gravity effector must come first (it overwrites Force)");
            h->graph_eff = (int)i;
            break;
        default:
            return fail(B200_ERR_UNSUPPORTED, "effector kind %u is not built in (no CPU fallback, no JIT)", e.kind);
        }
        if (e.kind == B200_EFF_GRAVITY_FRAME) ++n_frame;
        if (e.column_id) {
            if (e.column_width != want_w && !(e.kind == B200_EFF_DRAG_QUADRATIC && e.column_width == 5))
                return fail(B200_ERR_VALUE_SIZE_MISMATCH, "effector %zu: column width %u, kind %u needs %u", i, e.column_width, e.kind, want_w);
        } else if (e.kind == B200_EFF_THRUST_BODY || e.kind == B200_EFF_WRENCH_BODY || e.kind == B200_EFF_WRENCH_WORLD ||
                   e.kind == B200_EFF_TORQUE_BODY_FOLD) {
            return fail(B200_ERR_INVALID_ARGUMENT, "effector %zu (kind %u) needs an input column", i, e.kind);
        }
    }
    if (d->math_mode == B200_MATH_FAST && (n_drag > 1 || n_frame > 1))
        return fail(B200_ERR_UNSUPPORTED, "FAST math supports at most one drag and one frame effector");

    // columns
    if ((rc = add_column(h, B200_ID_TICK, 1, true))) return rc;
    if ((rc = add_column(h, B200_ID_SIMULATION_TIME_STEP, 1, true))) return rc;
    if ((rc = add_column(h, B200_ID_WORLD_POS, 7, false))) return rc;
    if ((rc = add_column(h, B200_ID_WORLD_VEL, 6, false))) return rc;
    if ((rc = add_column(h, B200_ID_WORLD_ACCEL, 6, false))) return rc;
    if ((rc = add_column(h, B200_ID_FORCE, 6, false))) return rc;
    if ((rc = add_column(h, B200_ID_INERTIA, 7, false))) return rc;
    for (auto &e : h->effectors)
        if (e.column_id) {
            const Column *c = h->find(e.column_id);
            if (c && c->width != e.column_width)
                return fail(B200_ERR_VALUE_SIZE_MISMATCH, "column 0x%016llx declared with two widths", (unsigned long long)e.column_id);
            if ((rc = add_column(h, e.column_id, e.column_width, false))) return rc;
        }
    {
        const uint64_t bytes = (h->ld + 63) / 64;
        CU(h, cudaMalloc(&h->mass_class, bytes));
        CU(h, cudaMemsetAsync(h->mass_class, 0, bytes, h->stream));
    }
    build_id_tables(h);
    // per-effector entity masks: copy now, the caller's arrays are only valid for this call
    h->eff_masks.assign(h->effectors.size(), nullptr);
    for (size_t i = 0; i < h->effectors.size(); ++i) {
        b200_effector &e = h->effectors[i];
        if (e.entity_mask && d->n_entities) {
            CU(h, cudaMalloc(&h->eff_masks[i], d->n_entities));
            CU(h, cudaMemcpy(h->eff_masks[i], e.entity_mask, d->n_entities, cudaMemcpyHostToDevice));
        }
        e.entity_mask = nullptr;
    }

    // EGM08 coefficient tables: copied (with the derived recursion tables) now, the caller's arrays are only valid for this call
    h->eff_tables.assign(h->effectors.size(), nullptr);
    for (size_t i = 0; i < h->effectors.size(); ++i) {
        b200_effector &e = h->effectors[i];
        if (e.kind == B200_EFF_GRAVITY_EGM08) {
            const std::vector<double> t = egm08_tables((int)e.p[2], e.table0, e.table1);
            CU(h, cudaMalloc(&h->eff_tables[i], t.size() * sizeof(double)));
            CU(h, cudaMemcpy(h->eff_tables[i], t.data(), t.size() * sizeof(double), cudaMemcpyHostToDevice));
        }
        e.table0 = e.table1 = nullptr;
    }
    if (h->graph_eff >= 0) {
        // copy the edge arrays' content now: the caller's pointers are only valid for this call
        if ((rc = build_graph(h, h->effectors[h->graph_eff]))) return rc;
        const GraphParams G = graph_params(h, range_step_params(h, 0, h->n_bodies), d->n_worlds);
        // (an EGM08 effector needs its stage-force launch before every body launch: the generic two-launch route)
        h->small_world = h->egm_eff < 0 && small_world_applicable(G, (int)d->math_mode);
        h->nbody_fused = h->egm_eff < 0 && !h->small_world && h->pos_alt && nbody_fused_applicable(G, (int)d->math_mode, h->graph_dense);
        h->effectors[h->graph_eff].edge_from = h->effectors[h->graph_eff].edge_to = nullptr;
    }
    if (h->egm_eff >= 0) {
        CU(h, cudaMalloc(&h->aforce, 9ull * h->ld * 8ull));
        CU(h, cudaMemset(h->aforce, 0, 9ull * h->ld * 8ull));
    }
    if (d->trajectory_every && d->trajectory_capacity) {
        h->traj_planes = (d->trajectory_flags & B200_TRAJ_FULL) ? 25u : 13u;
        CU(h, cudaMalloc(&h->traj, d->trajectory_capacity * (uint64_t)h->traj_planes * h->ld * 8ull));
    }
    CU(h, cudaStreamSynchronize(h->stream));
    return B200_OK;
}

void b200_sixdof_destroy(b200_sixdof *h)
{
    if (!h) return;
    if (g_tick_handle == h) g_tick_handle = nullptr;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    for (auto &c : h->cols) if (c.dev) cudaFree(c.dev);
    if (h->mass_class) cudaFree(h->mass_class);
    for (auto m : h->eff_masks) if (m) cudaFree(m);
    for (auto t : h->eff_tables) if (t) cudaFree(t);
    if (h->row_ptr) cudaFree(h->row_ptr);
    if (h->col_idx) cudaFree(h->col_idx);
    if (h->has_edge) cudaFree(h->has_edge);
    if (h->gforce) cudaFree(h->gforce);
    if (h->aforce) cudaFree(h->aforce);
    if (h->pos_alt) cudaFree(h->pos_alt);
    if (h->vel_alt) cudaFree(h->vel_alt);
    if (h->staging) cudaFree(h->staging);
    if (h->sq_scratch) cudaFree(h->sq_scratch);
    if (h->stage_in) cudaFree(h->stage_in);
    if (h->stage_out) cudaFree(h->stage_out);
    if (h->traj) cudaFree(h->traj);
    if (h->sum_ext) cudaFree(h->sum_ext);
    if (h->chan_ring) cudaFree(h->chan_ring);
    if (h->chan_state) cudaFree(h->chan_state);
    if (h->sum_thr) cudaFree(h->sum_thr);
    if (h->sum_mom) cudaFree(h->sum_mom);
    if (h->sum_dwell) cudaFree(h->sum_dwell);
    if (h->out_planes) cudaFree(h->out_planes);
    if (h->rank_planes) cudaFree(h->rank_planes);
    if (h->sobol_planes) cudaFree(h->sobol_planes);
    rank_shard_free(h->sr.Q);
    for (const auto *ts : {h->tables, h->out_tables})
        for (int g = 0; g < 2; ++g)
            for (void *p : {(void *)ts[g].stats_dev, (void *)ts[g].cov_dev, (void *)ts[g].order_dev})
                if (p) cudaFree(p);
    for (auto &e : h->chunk_in) if (e) cudaEventDestroy(e);
    for (auto &e : h->chunk_out) if (e) cudaEventDestroy(e);
    if (h->host_pack) cudaFreeHost(h->host_pack);
    if (h->copy_in) cudaStreamDestroy(h->copy_in);
    if (h->copy_out) cudaStreamDestroy(h->copy_out);
    for (auto &e : h->ev) if (e) cudaEventDestroy(e);
    if (h->stream && h->own_stream) cudaStreamDestroy(h->stream);
    (void)cudaGetLastError();
    delete h;
}

uint32_t b200_sixdof_input_ids(const b200_sixdof *h, uint64_t *ids, uint32_t cap)
{
    if (!h) return 0;
    for (uint32_t i = 0; i < cap && i < h->input_ids.size(); ++i) ids[i] = h->input_ids[i];
    return (uint32_t)h->input_ids.size();
}

uint32_t b200_sixdof_output_ids(const b200_sixdof *h, uint64_t *ids, uint32_t cap)
{
    if (!h) return 0;
    for (uint32_t i = 0; i < cap && i < h->output_ids.size(); ++i) ids[i] = h->output_ids[i];
    return (uint32_t)h->output_ids.size();
}

uint64_t b200_sixdof_column_bytes(const b200_sixdof *h, uint64_t id)
{
    if (!h) return 0;
    const Column *c = h->find(id);
    return c ? column_bytes(h, *c) : 0;
}

int b200_sixdof_upload(b200_sixdof *h, uint64_t id, const void *src, uint64_t bytes)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    return do_upload(h, id, src, bytes);
}

int b200_sixdof_download(b200_sixdof *h, uint64_t id, void *dst, uint64_t bytes)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    return do_download(h, id, dst, bytes);
}

int b200_sixdof_step(b200_sixdof *h, uint64_t n_ticks)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    return do_step(h, n_ticks);
}

int b200_sixdof_sync(b200_sixdof *h)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaStreamSynchronize(h->stream));
    return B200_OK;
}

// Which input columns really have to cross PCIe: Force is cleared before any effector runs
// (clear_forces, six_dof.rs:148-150) so its input value is dead; WorldAccel only enters as
// `0 * a_prev` (rk4.rs:85-104), which FAST math does not evaluate.  EXACT keeps WorldAccel.
static bool input_is_live(const b200_sixdof *h, uint64_t id)
{
    if (id == B200_ID_FORCE) return false;
    if (id == B200_ID_WORLD_ACCEL) return h->desc.math_mode == B200_MATH_EXACT && h->desc.integrator == B200_INTEGRATOR_RK4;
    return true;
}

// Output columns the kernels never write (Inertia, effector input columns) are pass-through
// variables of the reference system (`builder.to_compiled_system()` returns every var): their
// output buffer is the input buffer's content, so it is filled host-to-host on worker threads
// while the PCIe link carries the columns that did change.
static bool output_is_pass_through(uint64_t id)
{
    return id != B200_ID_WORLD_POS && id != B200_ID_WORLD_VEL && id != B200_ID_WORLD_ACCEL && id != B200_ID_FORCE &&
           id != B200_ID_TICK && id != B200_ID_SIMULATION_TIME_STEP;
}

// What one b200_sixdof_invoke_batch call does with each caller column, decided once.  A NULL in_cols[i] means "not
// dirty" (World::dirty_components, world.rs:43,249-252): the device-resident copy of that column stands.  A NULL
// out_cols[j] means the caller does not read that column after this batch.
struct BatchPlan {
    enum Role {
        ABSENT = 0,   // NULL buffer
        GLOBAL,       // one of the two host-resident scalars
        DEAD,         // an input the ticks never read (input_is_live): present, not uploaded
        UPLOAD,       // an input that crosses PCIe
        DOWNLOAD,     // an output that crosses PCIe
        PASS_THROUGH  // an output the ticks never write (output_is_pass_through): filled from the input of the same column
    };
    struct Col {
        Role role;
        Column *col;
        const uint8_t *src; // inputs: the caller's buffer.  PASS_THROUGH: the caller's input buffer of the same column, NULL =
                            // that input is not dirty (the device column is the value: downloaded after the ticks)
        uint8_t *dst;       // outputs: the caller's buffer
        uint64_t offset;    // UPLOAD / DOWNLOAD: doubles from the start of the packed / staged block of its direction
        bool device;        // non-global columns: the caller's buffer (PASS_THROUGH: either of the two) is device memory
    };
    // in input_ids / output_ids order; entries past the handle's columns stay ABSENT
    Col in[B200_MAX_EFFECTORS + 7], out[B200_MAX_EFFECTORS + 7];
    uint64_t in_total, out_total; // doubles of the UPLOAD / DOWNLOAD columns
    bool device_buffers;          // some present non-global caller buffer is device memory
};

static BatchPlan plan_batch(b200_sixdof *h, const uint8_t *const *in_cols, uint8_t *const *out_cols)
{
    BatchPlan p{};
    for (size_t i = 0; i < h->input_ids.size(); ++i) {
        BatchPlan::Col &c = p.in[i];
        c.col = h->find(h->input_ids[i]);
        c.src = in_cols[i];
        if (!c.src) continue;
        if (c.col->global) { c.role = BatchPlan::GLOBAL; continue; }
        c.device = is_device_pointer(c.src);
        c.role = input_is_live(h, c.col->id) ? BatchPlan::UPLOAD : BatchPlan::DEAD;
        if (c.role == BatchPlan::UPLOAD) { c.offset = p.in_total; p.in_total += h->n_bodies * c.col->width; }
        p.device_buffers = p.device_buffers || c.device;
    }
    for (size_t i = 0; i < h->output_ids.size(); ++i) {
        BatchPlan::Col &c = p.out[i];
        c.col = h->find(h->output_ids[i]);
        c.dst = out_cols[i];
        if (!c.dst) continue;
        if (c.col->global) { c.role = BatchPlan::GLOBAL; continue; }
        c.device = is_device_pointer(c.dst);
        p.device_buffers = p.device_buffers || c.device;
        if (!output_is_pass_through(c.col->id)) {
            c.role = BatchPlan::DOWNLOAD;
            c.offset = p.out_total;
            p.out_total += h->n_bodies * c.col->width;
            continue;
        }
        c.role = BatchPlan::PASS_THROUGH;
        for (const BatchPlan::Col &in : p.in)
            if (in.col == c.col && in.src) { c.src = in.src; c.device = c.device || in.device; }
    }
    return p;
}

// Small batches (interactive single-vehicle sims: the reference's everyday case) are bound by the
// number of driver calls, not by bytes: pack every live input column into one pinned block, ONE
// host->device copy, ONE layout launch for all columns, the ticks, ONE layout launch, ONE copy back.
static int invoke_small(b200_sixdof *h, const BatchPlan &plan, uint64_t n_ticks)
{
    MultiColumns mi{}, mo{};
    int rc;
    for (const BatchPlan::Col &c : plan.in) {
        if (c.role == BatchPlan::GLOBAL && (rc = do_upload(h, c.col->id, c.src, 8))) return rc;
        if (c.role != BatchPlan::UPLOAD) continue;
        if (c.col->id == B200_ID_INERTIA && (rc = clear_mass_class(h, 0, h->n_bodies))) return rc;
        mi.col[mi.n++] = {c.offset, c.col->dev, c.col->width, 0};
    }
    const uint64_t need = std::max(plan.in_total, plan.out_total) * 8;
    if (h->host_pack_bytes < need) {
        if (h->host_pack) cudaFreeHost(h->host_pack);
        h->host_pack = nullptr; h->host_pack_bytes = 0;
        CU(h, cudaHostAlloc((void **)&h->host_pack, std::max<uint64_t>(need, 4096), cudaHostAllocDefault));
        h->host_pack_bytes = std::max<uint64_t>(need, 4096);
    }
    if ((rc = ensure_staging(h, std::max<uint64_t>(need, 8)))) return rc;
    for (const BatchPlan::Col &c : plan.in)
        if (c.role == BatchPlan::UPLOAD) std::memcpy(h->host_pack + c.offset * 8, c.src, column_bytes(h, *c.col));
    mi.packed = mo.packed = h->staging;
    if (plan.in_total) {
        CU(h, cudaMemcpyAsync(h->staging, h->host_pack, plan.in_total * 8, cudaMemcpyHostToDevice, h->stream));
        CU(h, launch_multi_transpose(mi, h->n_bodies, h->ld, true, h->stream));
        h->timings.kernel_launches++;
    }
    if ((rc = launch_ticks(h, 0, h->desc.n_worlds, n_ticks, h->stream))) return rc;
    commit_ping_pong(h, n_ticks);
    advance_ticks(h, n_ticks);
    for (const BatchPlan::Col &c : plan.out) // after a ping-pong swap: the columns' planes are the live ones
        if (c.role == BatchPlan::DOWNLOAD) mo.col[mo.n++] = {c.offset, c.col->dev, c.col->width, 0};
    if (plan.out_total) {
        CU(h, launch_multi_transpose(mo, h->n_bodies, h->ld, false, h->stream));
        h->timings.kernel_launches++;
        CU(h, cudaMemcpyAsync(h->host_pack, h->staging, plan.out_total * 8, cudaMemcpyDeviceToHost, h->stream));
    }
    CU(h, cudaStreamSynchronize(h->stream));
    for (const BatchPlan::Col &c : plan.out)
        if (c.role == BatchPlan::DOWNLOAD) std::memcpy(c.dst, h->host_pack + c.offset * 8, column_bytes(h, *c.col));
    for (const BatchPlan::Col &c : plan.out) {
        if (c.role == BatchPlan::GLOBAL && (rc = do_download(h, c.col->id, c.dst, 8))) return rc;
        if (c.role != BatchPlan::PASS_THROUGH) continue;
        if (!c.src) { // input was not dirty: the device copy is the value
            if ((rc = do_download(h, c.col->id, c.dst, column_bytes(h, *c.col)))) return rc;
        } else if (c.src != c.dst) {
            std::memcpy(c.dst, c.src, column_bytes(h, *c.col));
        }
    }
    h->timings.h2d_upload_ms = h->timings.kernel_invoke_ms = h->timings.d2h_download_ms = 0.0; // not separable here
    return B200_OK;
}

static int invoke_pipelined(b200_sixdof *h, const BatchPlan &plan, uint64_t n_ticks, uint64_t worlds_per_chunk)
{
    const uint64_t N = h->desc.n_entities, M = h->desc.n_worlds;
    const uint64_t n_chunks = (M + worlds_per_chunk - 1) / worlds_per_chunk;
    if (!h->copy_in) {
        CU(h, cudaStreamCreateWithFlags(&h->copy_in, cudaStreamNonBlocking));
        CU(h, cudaStreamCreateWithFlags(&h->copy_out, cudaStreamNonBlocking));
    }
    // B200_PIPE_TRACE=1: per-range completion times of the three engines on stderr (diagnostic; timing events)
    static const bool trace = [] { const char *e = getenv("B200_PIPE_TRACE"); return e && atoi(e) != 0; }();
    std::vector<cudaEvent_t> trace_d2h;
    const auto host_t0 = std::chrono::steady_clock::now();
    auto host_ms = [&] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count(); };
    double host_loop0 = 0.0, host_loop1 = 0.0;
    while (h->chunk_in.size() < n_chunks) {
        cudaEvent_t a, b;
        CU(h, cudaEventCreateWithFlags(&a, trace ? cudaEventDefault : cudaEventDisableTiming));
        CU(h, cudaEventCreateWithFlags(&b, trace ? cudaEventDefault : cudaEventDisableTiming));
        h->chunk_in.push_back(a);
        h->chunk_out.push_back(b);
    }
    int rc;
    // whole-batch AoS staging: an UPLOAD / DOWNLOAD column lives at its plan offset (doubles)
    if ((rc = grow_device(h, &h->stage_in, &h->stage_in_bytes, plan.in_total * 8))) return rc;
    if ((rc = grow_device(h, &h->stage_out, &h->stage_out_bytes, plan.out_total * 8))) return rc;
    // globals first (scalars the handle keeps on the host)
    for (const BatchPlan::Col &c : plan.in)
        if (c.role == BatchPlan::GLOBAL && (rc = do_upload(h, c.col->id, c.src, 8))) return rc;
    // the copy streams must not run ahead of work already queued on the compute stream (a caller's stream may still
    // write an input or read an output the copies below touch)
    CU(h, cudaEventRecord(h->ev[2], h->stream));
    CU(h, cudaStreamWaitEvent(h->copy_in, h->ev[2], 0));
    CU(h, cudaStreamWaitEvent(h->copy_out, h->ev[2], 0));
    // the pass-through outputs whose input is here: by the copy engine when either side is device memory, else
    // host-to-host on a few worker threads, while the PCIe link carries the columns that did change
    std::vector<std::thread> fillers;
    struct Joiner { std::vector<std::thread> &v; ~Joiner() { for (auto &t : v) if (t.joinable()) t.join(); } } joiner{fillers};
    for (const BatchPlan::Col &c : plan.out) {
        if (c.role != BatchPlan::PASS_THROUGH || !c.src || c.src == c.dst) continue;
        const uint64_t bytes = column_bytes(h, *c.col);
        if (c.device) {
            CU(h, cudaMemcpyAsync(c.dst, c.src, bytes, cudaMemcpyDefault, h->copy_out));
            continue;
        }
        const unsigned parts = bytes >= (8u << 20) ? 4u : 1u;
        for (unsigned t = 0; t < parts; ++t) {
            const uint64_t o0 = bytes * t / parts, o1 = bytes * (t + 1) / parts;
            fillers.emplace_back([dst = c.dst, src = c.src, o0, o1] { std::memcpy(dst + o0, src + o0, o1 - o0); });
        }
    }
    CU(h, cudaEventRecord(h->ev[0], h->copy_in));

    host_loop0 = host_ms();
    for (uint64_t k = 0; k < n_chunks; ++k) {
        const uint64_t w0 = k * worlds_per_chunk, nw = std::min(worlds_per_chunk, M - w0);
        const uint64_t b0 = w0 * N, nb = nw * N;
        // H2D of this world range, every live input column (copy engine 1)
        for (const BatchPlan::Col &c : plan.in) {
            if (c.role != BatchPlan::UPLOAD) continue;
            const uint32_t w = c.col->width;
            CU(h, cudaMemcpyAsync(h->stage_in + c.offset + b0 * w, (const double *)c.src + b0 * w, nb * w * 8, cudaMemcpyDefault,
                                  h->copy_in));
        }
        CU(h, cudaEventRecord(h->chunk_in[k], h->copy_in));
        if (k + 1 == n_chunks) CU(h, cudaEventRecord(h->ev[1], h->copy_in));
        // compute stream: AoS -> SoA, n ticks, SoA -> AoS
        CU(h, cudaStreamWaitEvent(h->stream, h->chunk_in[k], 0));
        for (const BatchPlan::Col &c : plan.in) {
            if (c.role != BatchPlan::UPLOAD) continue;
            if (c.col->id == B200_ID_INERTIA && (rc = clear_mass_class(h, b0, nb))) return rc;
            CU(h, launch_aos_to_soa(h->stage_in + c.offset + b0 * c.col->width, c.col->dev + b0, nb, c.col->width, h->ld, h->stream));
            h->timings.kernel_launches++;
        }
        if ((rc = launch_ticks(h, w0, nw, n_ticks, h->stream))) return rc;
        const bool flipped = h->nbody_fused && (n_ticks & 1); // live pose / velocity sit in the other plane set
        for (const BatchPlan::Col &c : plan.out) {
            if (c.role != BatchPlan::DOWNLOAD) continue;
            const double *live = c.col->dev;
            if (flipped && c.col->id == B200_ID_WORLD_POS) live = h->pos_alt;
            if (flipped && c.col->id == B200_ID_WORLD_VEL) live = h->vel_alt;
            CU(h, launch_soa_to_aos(live + b0, h->stage_out + c.offset + b0 * c.col->width, nb, c.col->width, h->ld, h->stream));
            h->timings.kernel_launches++;
        }
        CU(h, cudaEventRecord(h->chunk_out[k], h->stream));
        if (k + 1 == n_chunks) CU(h, cudaEventRecord(h->ev[3], h->stream));
        // D2H of this world range (copy engine 2) overlaps the next range's H2D and ticks
        CU(h, cudaStreamWaitEvent(h->copy_out, h->chunk_out[k], 0));
        if (k == 0) CU(h, cudaEventRecord(h->ev[4], h->copy_out));
        for (const BatchPlan::Col &c : plan.out) {
            if (c.role != BatchPlan::DOWNLOAD) continue;
            const uint32_t w = c.col->width;
            CU(h, cudaMemcpyAsync((double *)c.dst + b0 * w, h->stage_out + c.offset + b0 * w, nb * w * 8, cudaMemcpyDefault,
                                  h->copy_out));
        }
        if (trace) {
            cudaEvent_t e;
            CU(h, cudaEventCreate(&e));
            CU(h, cudaEventRecord(e, h->copy_out));
            trace_d2h.push_back(e);
        }
    }
    host_loop1 = host_ms();
    commit_ping_pong(h, n_ticks);
    advance_ticks(h, n_ticks);
    for (const BatchPlan::Col &c : plan.out)
        if (c.role == BatchPlan::GLOBAL && (rc = do_download(h, c.col->id, c.dst, 8))) return rc;
    CU(h, cudaEventRecord(h->ev[5], h->copy_out));
    CU(h, cudaStreamSynchronize(h->copy_out));
    CU(h, cudaStreamSynchronize(h->stream));
    CU(h, cudaStreamSynchronize(h->copy_in));
    for (const BatchPlan::Col &c : plan.out) // input not dirty: its value is the device-resident column
        if (c.role == BatchPlan::PASS_THROUGH && !c.src && (rc = do_download(h, c.col->id, c.dst, column_bytes(h, *c.col))))
            return rc;
    if (trace) {
        fprintf(stderr, "[b200 pipe] host: enqueue loop %.3f..%.3f ms, synced at %.3f ms; device times from the first upload's start:\n",
                host_loop0, host_loop1, host_ms());
        for (uint64_t k = 0; k < n_chunks; ++k) {
            fprintf(stderr, "[b200 pipe]  range %2llu: upload done %.3f  ticks done %.3f  download done %.3f ms\n", (unsigned long long)k,
                    ev_ms(h->ev[0], h->chunk_in[k]), ev_ms(h->ev[0], h->chunk_out[k]), ev_ms(h->ev[0], trace_d2h[k]));
            cudaEventDestroy(trace_d2h[k]);
        }
    }
    // busy spans of the three engines; they overlap, so they do not add up to the call time
    h->timings.h2d_upload_ms = ev_ms(h->ev[0], h->ev[1]);
    h->timings.kernel_invoke_ms = ev_ms(h->ev[2], h->ev[3]);
    h->timings.d2h_download_ms = ev_ms(h->ev[4], h->ev[5]);
    return B200_OK;
}

int b200_sixdof_invoke_batch(b200_sixdof *h, const uint8_t *const *in_cols, uint8_t *const *out_cols, uint64_t n_ticks)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    ++h->rows_gen;
    if (!in_cols || !out_cols) return fail(B200_ERR_INVALID_ARGUMENT, "null column tables");
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    CU(h, cudaSetDevice(h->device));
    n_ticks = std::max<uint64_t>(n_ticks, 1); // `n.max(1)`, cranelift_exec.rs:135

    // World ranges of ~kChunkBodies bodies: range k's PCIe download overlaps range k+1's upload
    // and ticks (two copy engines + the compute stream).  Small batches run as one range.
    static const uint64_t kEnvChunk = [] { const char *e = getenv("B200_CHUNK_BODIES"); return e ? (uint64_t)atoll(e) : (uint64_t)0; }();
    const uint64_t chunk_bodies = h->desc.invoke_chunk_bodies ? h->desc.invoke_chunk_bodies : (kEnvChunk ? kEnvChunk : 131072);
    const uint64_t N = std::max<uint64_t>(h->desc.n_entities, 1);
    uint64_t wpc = std::max<uint64_t>(1, chunk_bodies / N);
    if (N == 1 && wpc >= 128) wpc = wpc / 128 * 128;
    if (h->n_bodies == 0) wpc = std::max<uint64_t>(h->desc.n_worlds, 1);

    auto t0 = std::chrono::steady_clock::now();
    const BatchPlan plan = plan_batch(h, in_cols, out_cols);
    // the packed path memcpy()s: only for host-resident caller buffers; device-resident callers use the pipeline
    const bool small = h->n_bodies > 0 && h->n_bodies * 32ull * 8ull <= (256ull << 10) && h->input_ids.size() <= 16 &&
                       !h->desc.invoke_chunk_bodies && !plan.device_buffers;
    int rc = small ? invoke_small(h, plan, n_ticks) : invoke_pipelined(h, plan, n_ticks, wpc);
    if (rc) {
        // copies into the caller's buffers may still be queued: they must not outlive this call
        (void)cudaStreamSynchronize(h->stream);
        if (h->copy_in) (void)cudaStreamSynchronize(h->copy_in);
        if (h->copy_out) (void)cudaStreamSynchronize(h->copy_out);
        (void)cudaGetLastError();
        return rc;
    }
    h->timings.invoke_wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return B200_OK;
}

int b200_sixdof_bind_tick(b200_sixdof *h)
{
    g_tick_handle = h;
    return B200_OK;
}

void b200_sixdof_tick(const uint8_t *const *in_cols, uint8_t **out_cols)
{
    b200_sixdof *h = g_tick_handle;
    if (!h) { fail(B200_ERR_INVALID_ARGUMENT, "b200_sixdof_tick: no handle bound on this thread"); return; }
    (void)b200_sixdof_invoke_batch(h, in_cols, out_cols, 1); // errors stay sticky on the handle / last_error
}

uint64_t b200_sixdof_trajectory_len(const b200_sixdof *h)
{
    if (!h || !h->traj || !h->desc.trajectory_every) return 0;
    return std::min<uint64_t>(h->ticks_done / h->desc.trajectory_every, h->desc.trajectory_capacity);
}

int b200_sixdof_trajectory_download(b200_sixdof *h, void *dst, uint64_t bytes)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    const uint64_t n = b200_sixdof_trajectory_len(h);
    const uint64_t W = h->traj_planes;
    const uint64_t want = n * h->n_bodies * W * 8ull;
    if (bytes != want) return fail(B200_ERR_VALUE_SIZE_MISMATCH, "trajectory is %llu bytes, got %llu", (unsigned long long)want, (unsigned long long)bytes);
    if (want == 0) return B200_OK;
    // convert in chunks through the staging buffer
    const uint64_t per_sample = h->n_bodies * W * 8ull;
    const uint64_t chunk = std::max<uint64_t>(1, std::min<uint64_t>(n, (256ull << 20) / per_sample));
    int rc = ensure_staging(h, chunk * per_sample);
    if (rc) return rc;
    for (uint64_t s0 = 0; s0 < n; s0 += chunk) {
        const uint64_t ns = std::min(chunk, n - s0);
        CU(h, launch_traj_to_aos(h->traj + s0 * W * h->ld, h->staging, ns, h->n_bodies, h->ld, (uint32_t)W, h->stream));
        h->timings.kernel_launches++;
        CU(h, cudaMemcpyAsync((char *)dst + s0 * per_sample, h->staging, ns * per_sample, cudaMemcpyDefault, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
    }
    return B200_OK;
}

uint32_t b200_sixdof_trajectory_width(const b200_sixdof *h) { return (h && h->traj) ? h->traj_planes : 0; }

// dst is device memory on the handle's GPU, which a kernel can write directly; any other destination goes through the
// staging buffer.
static bool device_destination(const b200_sixdof *h, const void *dst)
{
    int device = -1;
    return is_device_pointer(dst, &device) && device == h->device;
}

static int refresh_channels(b200_sixdof *h, bool ring);
static int write_outcomes(b200_sixdof *h);

// What a reduction over the world axis reads: the rows of the state or of the ring's samples (ensemble_rows), or the
// outcome planes (b200_sixdof_set_outcomes), reduced as the state of a handle with one entity.
enum class Rows { state, ring, outcomes };

// A reduction over the world axis (stats_kernels.cu, quantile_kernels.cu, cov_kernels.cu, hist_kernels.cu) of `src` into
// dst, `bytes` already checked.  When it reads a channel plane (`channels`), the channel planes are recomputed first, on
// the handle's stream; the outcome planes are always rewritten first.  A device destination takes the table straight
// from the kernel; any other gets it through the staging buffer, after the `scratch` bytes the reduction needs.
// launch(out, scratch, &launches) enqueues the reduction on the handle's stream.
extern "C++" {
template <class Launch>
static int run_world_reduction(b200_sixdof *h, Rows src, bool channels, uint64_t scratch, void *dst, uint64_t bytes,
                               Launch launch)
{
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (bytes == 0) return B200_OK;
    if (!dst) return fail(B200_ERR_INVALID_ARGUMENT, "null destination buffer");
    int rc = src == Rows::outcomes ? write_outcomes(h) : channels ? refresh_channels(h, src == Rows::ring) : B200_OK;
    if (rc) return rc;
    const bool direct = device_destination(h, dst);
    scratch = (scratch + 7) / 8 * 8;
    rc = ensure_staging(h, std::max<uint64_t>(scratch + (direct ? 0 : bytes), 8));
    if (rc) return rc;
    double *out = direct ? (double *)dst : (double *)((char *)h->staging + scratch);
    int launches = 0;
    CU(h, launch(out, (void *)h->staging, &launches));
    h->timings.kernel_launches += (uint64_t)launches;
    if (!direct) CU(h, cudaMemcpyAsync(dst, out, bytes, cudaMemcpyDefault, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return B200_OK;
}
}

// The sampled planes (the B200_TRAJ_FULL layout: world_pos 0-6, world_vel 7-12, world_accel 13-18, force 19-24) of the
// samples now in the trajectory ring, and of the current state.  Every reduction and run summary reads them from here.
static StatsParams trajectory_planes(const b200_sixdof *h)
{
    const uint64_t n = b200_sixdof_trajectory_len(h);
    const uint64_t W = h->traj_planes;
    StatsParams S{};
    S.seg[0] = {h->traj, W, W * h->ld};
    S.n_segs = 1;
    S.planes_per_sample = (uint32_t)W;
    S.n_planes = n * W;
    S.ld = h->ld;
    S.n_worlds = h->desc.n_worlds;
    S.n_entities = h->desc.n_entities;
    return S;
}

static StatsParams state_planes(const b200_sixdof *h)
{
    StatsParams S{};
    const uint64_t ids[4] = {B200_ID_WORLD_POS, B200_ID_WORLD_VEL, B200_ID_WORLD_ACCEL, B200_ID_FORCE};
    for (int k = 0; k < 4; ++k) {
        const Column *c = h->find(ids[k]);
        S.seg[k] = {c->dev, c->width, 0};
    }
    S.n_segs = 4;
    S.planes_per_sample = 25;
    S.n_planes = 25;
    S.ld = h->ld;
    S.n_worlds = h->desc.n_worlds;
    S.n_entities = h->desc.n_entities;
    return S;
}

// download_worlds runs over one of these; `what` names it in error messages.
using PlaneSource = StatsParams (*)(const b200_sixdof *);

// The rows every ensemble reduction and run summary reads, R = 25 + n_c planes per sample: the sampled planes of the
// ring's samples (ring) or of the state, then the channel planes (b200_sixdof_set_channels) as a segment of its own.
static StatsParams ensemble_rows(const b200_sixdof *h, bool ring)
{
    StatsParams S = ring ? trajectory_planes(h) : state_planes(h);
    const uint64_t n_c = h->channels.size();
    if (n_c) {
        const uint64_t n_s = S.n_planes / S.planes_per_sample;
        S.seg[S.n_segs++] = {ring ? h->chan_ring : h->chan_state, n_c, n_c * h->ld};
        S.planes_per_sample += (uint32_t)n_c;
        S.n_planes = n_s * S.planes_per_sample;
    }
    return S;
}

// The planes of a row of the ring (0 without a ring) or of the state: what a plane index is checked against.
static uint32_t row_width(const b200_sixdof *h, bool ring)
{
    const uint32_t n_c = (uint32_t)h->channels.size();
    return ring ? (h->traj ? h->traj_planes + n_c : 0) : 25 + n_c;
}

// Recompute the channel planes of every sample now in the ring (ring) or of the state, on the handle's stream (one
// launch, none without channels or samples).  Always recomputed, never cached: b200_sixdof_device_plane hands out
// writable planes.
static int refresh_channels(b200_sixdof *h, bool ring)
{
    if (h->channels.empty()) return B200_OK;
    const StatsParams S = ring ? trajectory_planes(h) : state_planes(h);
    ChannelParams P{};
    uint32_t p = 0;
    for (uint32_t k = 0; k < S.n_segs; ++k)
        for (uint64_t j = 0; j < S.seg[k].n_planes && p < 25; ++j) P.row[p++] = S.seg[k].base + j * S.ld;
    P.row_stride = S.seg[0].stride;
    P.out = ring ? h->chan_ring : h->chan_state;
    P.ld = h->ld;
    P.n_bodies = h->n_bodies;
    P.n_samples = S.n_planes / S.planes_per_sample;
    P.n_c = (uint32_t)h->channels.size();
    for (uint32_t k = 0; k < P.n_c; ++k) P.c[k] = h->channels[k];
    int launches = 0;
    CU(h, launch_channels(P, &launches, h->stream));
    h->timings.kernel_launches += (uint64_t)launches;
    return B200_OK;
}

// The rows of worlds[0 .. n) of the planes of `source` into dst (gather_worlds_kernel): the arguments checked, then
// `bytes`, then the handle's status.  The index list goes to the device once, at the front of the staging buffer.  A
// device destination on the handle's GPU takes the rows straight from the kernel; any other gets them through the
// staging buffer in slices of at most 256 MiB of samples (one sample at least).
static int download_worlds(b200_sixdof *h, PlaneSource source, const uint64_t *worlds, uint32_t n, void *dst,
                           uint64_t bytes, const char *what)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (n == 0) return fail(B200_ERR_INVALID_ARGUMENT, "%s rows of 0 worlds: list at least one", what);
    if (!worlds) return fail(B200_ERR_INVALID_ARGUMENT, "null world list");
    for (uint32_t j = 0; j < n; ++j)
        if (worlds[j] >= h->desc.n_worlds)
            return fail(B200_ERR_INVALID_ARGUMENT, "world index %llu (entry %u) is not below the %llu worlds",
                        (unsigned long long)worlds[j], j, (unsigned long long)h->desc.n_worlds);
    CU(h, cudaSetDevice(h->device));
    StatsParams S = source(h);
    const uint64_t W = S.planes_per_sample, n_samples = S.n_planes / W;
    const uint64_t per_sample = (uint64_t)n * S.n_entities * W * 8ull, want = n_samples * per_sample;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "%s rows of %u worlds are %llu bytes, got %llu", what, n,
                    (unsigned long long)want, (unsigned long long)bytes);
    if (want == 0) return B200_OK;
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (!dst) return fail(B200_ERR_INVALID_ARGUMENT, "null destination buffer");
    const bool direct = device_destination(h, dst);
    const uint64_t list = (uint64_t)n * 8ull;
    const uint64_t chunk = direct ? n_samples : std::max<uint64_t>(1, std::min<uint64_t>(n_samples, (256ull << 20) / per_sample));
    int rc = ensure_staging(h, list + (direct ? 0 : chunk * per_sample));
    if (rc) return rc;
    const uint64_t *dev_worlds = (const uint64_t *)h->staging;
    CU(h, cudaMemcpyAsync(h->staging, worlds, list, cudaMemcpyHostToDevice, h->stream));
    for (uint64_t s0 = 0; s0 < n_samples; s0 += chunk) {
        const uint64_t ns = std::min(chunk, n_samples - s0);
        S.out = direct ? (double *)((char *)dst + s0 * per_sample) : (double *)((char *)h->staging + list);
        int launches = 0;
        CU(h, launch_gather_worlds(S, dev_worlds, n, s0, ns, &launches, h->stream));
        h->timings.kernel_launches += (uint64_t)launches;
        if (!direct) CU(h, cudaMemcpyAsync((char *)dst + s0 * per_sample, S.out, ns * per_sample, cudaMemcpyDefault, h->stream));
    }
    CU(h, cudaStreamSynchronize(h->stream));
    return B200_OK;
}

int b200_sixdof_trajectory_download_worlds(b200_sixdof *h, const uint64_t *worlds, uint32_t n, void *dst, uint64_t bytes)
{
    return download_worlds(h, trajectory_planes, worlds, n, dst, bytes, "trajectory");
}

int b200_sixdof_state_download_worlds(b200_sixdof *h, const uint64_t *worlds, uint32_t n, void *dst, uint64_t bytes)
{
    return download_worlds(h, state_planes, worlds, n, dst, bytes, "state");
}

// A group table of `bytes` into device memory (*dev, replaced): the stream is drained first, so that no reduction still
// in flight reads the table it replaces.
static int upload_group_table(b200_sixdof *h, const void *t, uint64_t bytes, void **dev)
{
    CU(h, cudaStreamSynchronize(h->stream));
    if (*dev) CU(h, cudaFree(*dev));
    *dev = nullptr;
    if (bytes == 0) return B200_OK;
    CU(h, cudaMalloc(dev, bytes));
    CU(h, cudaMemcpy(*dev, t, bytes, cudaMemcpyHostToDevice));
    return B200_OK;
}

// The tables of consecutive groups of sizes[0 .. n_groups) of worlds of n_entities entities into t, each with its
// device copy: the statistics' group table, the quantiles' route order over it and the covariance's group table.
static int fill_group_tables(b200_sixdof *h, b200_sixdof::GroupTables &t, const uint64_t *sizes, uint32_t n_groups,
                             uint64_t n_entities)
{
    t.stats = world_group_table(sizes, n_groups, n_entities);
    t.cov = cov_group_table(sizes, n_groups, n_entities);
    t.order = quantile_order(t.stats);
    int rc = upload_group_table(h, t.stats.data(), t.stats.size() * sizeof(WorldGroup), (void **)&t.stats_dev);
    if (!rc) rc = upload_group_table(h, t.cov.data(), t.cov.size() * sizeof(WorldGroup), (void **)&t.cov_dev);
    if (!rc) rc = upload_group_table(h, t.order.data(), t.order.size() * sizeof(uint32_t), (void **)&t.order_dev);
    return rc;
}

// The outcome entries' tables of one entity over the same worlds as h->tables[grouped], where n_entities != 1 (with one
// entity they share `tables`).  Built only once outcomes are set (set_outcomes builds both), so that a handle without
// outcomes allocates and uploads exactly what it did before outcomes existed.
static int build_outcome_tables(b200_sixdof *h, const uint64_t *sizes, uint32_t n_groups, bool grouped)
{
    if (h->desc.n_entities == 1 || h->outcomes.empty()) return B200_OK;
    return fill_group_tables(h, h->out_tables[grouped], sizes, n_groups, 1);
}

// The grouped entries' tables, else the all-worlds ones, and the outcome entries' over the same worlds.
static int build_group_tables(b200_sixdof *h, const uint64_t *sizes, uint32_t n_groups, bool grouped)
{
    const int rc = fill_group_tables(h, h->tables[grouped], sizes, n_groups, h->desc.n_entities);
    return rc ? rc : build_outcome_tables(h, sizes, n_groups, grouped);
}

int b200_sixdof_set_world_groups(b200_sixdof *h, const uint64_t *sizes, uint32_t n_groups)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (n_groups > B200_MAX_WORLD_GROUPS)
        return fail(B200_ERR_INVALID_ARGUMENT, "%u world groups: at most %u", n_groups, B200_MAX_WORLD_GROUPS);
    if (n_groups && !sizes) return fail(B200_ERR_INVALID_ARGUMENT, "null world group sizes");
    uint64_t sum = 0;
    for (uint32_t g = 0; g < n_groups; ++g) {
        if (sizes[g] > h->desc.n_worlds - sum)
            return fail(B200_ERR_INVALID_ARGUMENT, "world group sizes exceed the %llu worlds at group %u",
                        (unsigned long long)h->desc.n_worlds, g);
        sum += sizes[g];
    }
    if (n_groups && sum != h->desc.n_worlds)
        return fail(B200_ERR_INVALID_ARGUMENT, "world group sizes sum to %llu, not to the %llu worlds", (unsigned long long)sum,
                    (unsigned long long)h->desc.n_worlds);
    CU(h, cudaSetDevice(h->device));
    ++h->rows_gen;
    h->group_sizes.assign(sizes, sizes + n_groups);
    return build_group_tables(h, sizes, n_groups, true);
}

uint32_t b200_sixdof_world_groups(const b200_sixdof *h) { return h ? (uint32_t)h->group_sizes.size() : 0; }

// The world sizes a reduction runs over: the groups set (grouped), else all worlds as one group.
static std::vector<uint64_t> reduction_groups(const b200_sixdof *h, bool grouped)
{
    return grouped ? h->group_sizes : std::vector<uint64_t>{h->desc.n_worlds};
}

static int no_groups(const char *what)
{
    return fail(B200_ERR_INVALID_ARGUMENT, "grouped %s: call b200_sixdof_set_world_groups first", what);
}

static int check_outcomes(const b200_sixdof *h);

// The planes a reduction reads (Rows), their width (what a plane index is checked against) and its group tables.
static StatsParams reduction_rows(const b200_sixdof *h, Rows src)
{
    if (src != Rows::outcomes) return ensemble_rows(h, src == Rows::ring);
    const uint64_t P = h->outcomes.size();
    StatsParams S{};
    S.seg[0] = {h->out_planes, P, P * h->ld_o};
    S.n_segs = 1;
    S.planes_per_sample = (uint32_t)P;
    S.n_planes = P;
    S.ld = h->ld_o;
    S.n_worlds = h->desc.n_worlds;
    S.n_entities = 1;
    return S;
}

static uint32_t reduction_width(const b200_sixdof *h, Rows src)
{
    return src == Rows::outcomes ? (uint32_t)h->outcomes.size() : row_width(h, src == Rows::ring);
}

static const b200_sixdof::GroupTables &reduction_tables(const b200_sixdof *h, Rows src, bool grouped)
{
    return src == Rows::outcomes && h->desc.n_entities != 1 ? h->out_tables[grouped] : h->tables[grouped];
}

// The checks every reduction makes first: a null handle, groups for a grouped one, and for the outcome entries an
// outcome set that the summary in force still has.
static int reduction_ready(const b200_sixdof *h, Rows src, bool grouped, const char *what)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (grouped && h->group_sizes.empty()) return no_groups(what);
    return src == Rows::outcomes ? check_outcomes(h) : B200_OK;
}

// Statistics of the planes over the worlds, per group when `grouped` (stats_kernels.cu), into dst: the groups checked,
// then `bytes`, then the handle's status.
static int run_world_stats(b200_sixdof *h, Rows src, bool grouped, void *dst, uint64_t bytes, const char *what)
{
    int rc = reduction_ready(h, src, grouped, what);
    if (rc) return rc;
    CU(h, cudaSetDevice(h->device));
    StatsParams S = reduction_rows(h, src);
    const uint64_t G = grouped ? h->group_sizes.size() : 1;
    const uint64_t want = S.n_planes * G * S.n_entities * 5ull * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "%s statistics are %llu bytes, got %llu", what, (unsigned long long)want,
                    (unsigned long long)bytes);
    const b200_sixdof::GroupTables &t = reduction_tables(h, src, grouped);
    const uint64_t scratch = bytes && h->status == B200_OK ? world_stats_scratch_doubles(S, t.stats) * 8ull : 0;
    return run_world_reduction(h, src, true, scratch, dst, bytes, [&](double *out, void *scr, int *n) {
        S.out = out;
        return launch_world_stats(S, t.stats_dev, t.stats, (double *)scr, n, h->stream);
    });
}

int b200_sixdof_trajectory_stats(b200_sixdof *h, void *dst, uint64_t bytes)
{
    return run_world_stats(h, Rows::ring, false, dst, bytes, "trajectory");
}

int b200_sixdof_state_stats(b200_sixdof *h, void *dst, uint64_t bytes)
{
    return run_world_stats(h, Rows::state, false, dst, bytes, "state");
}

int b200_sixdof_trajectory_group_stats(b200_sixdof *h, void *dst, uint64_t bytes)
{
    return run_world_stats(h, Rows::ring, true, dst, bytes, "trajectory");
}

int b200_sixdof_state_group_stats(b200_sixdof *h, void *dst, uint64_t bytes)
{
    return run_world_stats(h, Rows::state, true, dst, bytes, "state");
}

// The checks of a quantile call, in order: the groups, then the handle's status, then the levels.  Fills S with the
// rows, the levels and the group table of the call.
static int quantile_params(b200_sixdof *h, Rows src, bool grouped, const double *q, uint32_t n_q, const char *what,
                           QuantileParams &S)
{
    int rc = reduction_ready(h, src, grouped, what);
    if (rc) return rc;
    CU(h, cudaSetDevice(h->device));
    static_cast<StatsParams &>(S) = reduction_rows(h, src);
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (n_q == 0 || n_q > B200_MAX_QUANTILES)
        return fail(B200_ERR_INVALID_ARGUMENT, "%u quantile levels: 1 to %u", n_q, B200_MAX_QUANTILES);
    if (!q) return fail(B200_ERR_INVALID_ARGUMENT, "null quantile levels");
    for (uint32_t l = 0; l < n_q; ++l)
        if (!(q[l] >= 0.0 && q[l] <= 1.0)) return fail(B200_ERR_INVALID_ARGUMENT, "quantile level %u is %g, not in [0, 1]", l, q[l]);
    const b200_sixdof::GroupTables &t = reduction_tables(h, src, grouped);
    S.n_q = n_q;
    for (uint32_t l = 0; l < n_q; ++l) S.q[l] = q[l];
    S.groups = t.stats_dev;
    S.order = t.order_dev;
    S.n_groups = reduction_groups(h, grouped).size();
    return B200_OK;
}

// Quantiles of the planes over the worlds, per group when `grouped` (quantile_kernels.cu), into dst: the groups checked,
// then the handle's status, then the levels, then `bytes`.
static int run_quantiles(b200_sixdof *h, Rows src, bool grouped, const double *q, uint32_t n_q, void *dst,
                         uint64_t bytes, const char *what)
{
    QuantileParams S{};
    int rc = quantile_params(h, src, grouped, q, n_q, what, S);
    if (rc) return rc;
    const b200_sixdof::GroupTables &t = reduction_tables(h, src, grouped);
    const uint64_t G = S.n_groups;
    const uint64_t want = S.n_planes * G * S.n_entities * n_q * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "%s quantiles are %llu bytes, got %llu", what, (unsigned long long)want,
                    (unsigned long long)bytes);
    const uint64_t triples = S.n_planes * G * S.n_entities;
    h->quantile_read_sum = triples;  // the small-group routes read every triple once
    const uint64_t scratch = quantile_scratch_bytes(S, t.stats);
    rc = run_world_reduction(h, src, true, scratch, dst, bytes, [&](double *out, void *scr, int *n) {
        S.out = out;
        return launch_quantiles(S, t.stats, t.order, scr, n, &h->quantile_read_sum, h->stream);
    });
    h->quantile_reads = rc == B200_OK && bytes && triples ? (double)h->quantile_read_sum / (double)triples : 0.0;
    return rc;
}

int b200_sixdof_trajectory_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes)
{
    return run_quantiles(h, Rows::ring, false, q, n_q, dst, bytes, "trajectory");
}

int b200_sixdof_state_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes)
{
    return run_quantiles(h, Rows::state, false, q, n_q, dst, bytes, "state");
}

int b200_sixdof_trajectory_group_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes)
{
    return run_quantiles(h, Rows::ring, true, q, n_q, dst, bytes, "trajectory");
}

int b200_sixdof_state_group_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes)
{
    return run_quantiles(h, Rows::state, true, q, n_q, dst, bytes, "state");
}

double b200_sixdof_quantile_reads(const b200_sixdof *h) { return h ? h->quantile_reads : 0.0; }

// ---- world-sharded quantiles (quantile_kernels.cu: sharded_quantile_round) ----

// The write generation of what a sharded call over `outcomes` (else the ring or state rows) reads: the outcome planes
// are rewritten from the run summaries by every outcome entry, so a summary start or fold changes them too.
static uint64_t rows_generation(const b200_sixdof *h, bool outcomes)
{
    return h->rows_gen + (outcomes ? h->sum_gen : 0);
}

int b200_sixdof_sharded_quantiles_begin(b200_sixdof *h, uint32_t source, int grouped, const double *q, uint32_t n_q,
                                        uint64_t *max_round_bytes)
{
    static const char *const names[3] = {"trajectory", "state", "outcome"};
    static const Rows rows[3] = {Rows::ring, Rows::state, Rows::outcomes};
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (source > B200_QUANTILE_OUTCOMES)
        return fail(B200_ERR_INVALID_ARGUMENT, "quantile source %u: B200_QUANTILE_RING, _STATE or _OUTCOMES", source);
    if (!max_round_bytes) return fail(B200_ERR_INVALID_ARGUMENT, "null max_round_bytes");
    h->sq.active = false;  // a call still pending is discarded
    const Rows src = rows[source];
    QuantileParams S{};
    int rc = quantile_params(h, src, grouped != 0, q, n_q, names[source], S);
    if (rc) return rc;
    const b200_sixdof::GroupTables &t = reduction_tables(h, src, grouped != 0);
    const uint64_t table_bytes = S.n_planes * S.n_groups * S.n_entities * n_q * 8ull;
    const uint64_t scratch = sharded_quantile_scratch_bytes(S, S.n_groups);
    rc = src == Rows::outcomes ? write_outcomes(h) : refresh_channels(h, src == Rows::ring);
    if (!rc) rc = grow_device(h, &h->sq_scratch, &h->sq_scratch_bytes, std::max<uint64_t>(scratch + table_bytes, 8));
    if (rc) return rc;
    b200_sixdof::ShardedQuantiles &c = h->sq;
    c.Q.S = S;
    c.Q.S.out = (double *)((char *)h->sq_scratch + scratch);
    c.Q.table = t.stats;
    c.Q.scratch = h->sq_scratch;
    c.Q.slice = 0;
    c.Q.level = -1;
    c.Q.reads = 0;
    c.outcomes = src == Rows::outcomes;
    c.gen = rows_generation(h, c.outcomes);
    c.partial_bytes = 0;
    c.max_round = sharded_quantile_round_bytes(S, S.n_groups);
    c.table_bytes = table_bytes;
    c.triples = S.n_planes * S.n_groups * S.n_entities;
    c.ready = false;
    c.active = true;
    *max_round_bytes = c.max_round;
    return B200_OK;
}

// the checks every round and end make first: a call begun, on the rows it began on
static int sharded_quantiles_pending(b200_sixdof *h, const char *what)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (!h->sq.active) return fail(B200_ERR_INVALID_ARGUMENT, "sharded quantiles %s without a begin", what);
    if (h->sq.gen != rows_generation(h, h->sq.outcomes)) {
        h->sq.active = false;
        return fail(B200_ERR_INVALID_ARGUMENT, "sharded quantiles %s: the handle's rows changed since the begin", what);
    }
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    return B200_OK;
}

int b200_sixdof_sharded_quantiles_round(b200_sixdof *h, const void *reduced, uint64_t reduced_bytes, void *partial,
                                        uint64_t partial_cap, uint64_t *partial_bytes)
{
    int rc = sharded_quantiles_pending(h, "round");
    if (rc) return rc;
    b200_sixdof::ShardedQuantiles &c = h->sq;
    if (c.ready) return fail(B200_ERR_INVALID_ARGUMENT, "sharded quantiles: the table is ready, call the end");
    if (reduced_bytes != c.partial_bytes)
        return fail(B200_ERR_INVALID_ARGUMENT, "sharded quantiles: %llu reduced bytes, the last round sent %llu",
                    (unsigned long long)reduced_bytes, (unsigned long long)c.partial_bytes);
    if (reduced_bytes && !reduced) return fail(B200_ERR_INVALID_ARGUMENT, "null reduced words");
    if (!partial_bytes) return fail(B200_ERR_INVALID_ARGUMENT, "null partial_bytes");
    if (partial_cap < c.max_round || (c.max_round && !partial))
        return fail(B200_ERR_INVALID_ARGUMENT, "sharded quantiles: a partial of %llu bytes, the begin asked for %llu",
                    (unsigned long long)partial_cap, (unsigned long long)c.max_round);
    CU(h, cudaSetDevice(h->device));
    int launches = 0;
    uint64_t out = 0;
    const cudaError_t e = sharded_quantile_round(c.Q, reduced, partial, &out, &launches, h->stream);
    h->timings.kernel_launches += (uint64_t)launches;
    if (e != cudaSuccess) {
        c.active = false;
        return cuda_fail(h, e, "sharded_quantile_round");
    }
    c.partial_bytes = *partial_bytes = out;
    c.ready = out == 0;
    return B200_OK;
}

int b200_sixdof_sharded_quantiles_end(b200_sixdof *h, void *dst, uint64_t bytes)
{
    int rc = sharded_quantiles_pending(h, "end");
    if (rc) return rc;
    b200_sixdof::ShardedQuantiles &c = h->sq;
    if (!c.ready) return fail(B200_ERR_INVALID_ARGUMENT, "sharded quantiles: end before the last round");
    if (bytes != c.table_bytes)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "sharded quantiles are %llu bytes, got %llu",
                    (unsigned long long)c.table_bytes, (unsigned long long)bytes);
    if (bytes && !dst) return fail(B200_ERR_INVALID_ARGUMENT, "null destination buffer");
    CU(h, cudaSetDevice(h->device));
    if (bytes) {
        CU(h, cudaMemcpyAsync(dst, c.Q.S.out, bytes, cudaMemcpyDefault, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
    }
    h->quantile_reads = bytes && c.triples ? (double)c.Q.reads / (double)c.triples : 0.0;
    c.active = false;
    return B200_OK;
}

// Covariance of the selection `planes` (each < width) of every sample over the worlds, per group when `grouped`
// (cov_kernels.cu), into dst: the groups checked, then the handle's status, then the selection, then `bytes`.
static int run_covariance(b200_sixdof *h, Rows src, bool grouped, const uint32_t *planes, uint32_t n_p, void *dst,
                          uint64_t bytes, const char *what)
{
    int rc = reduction_ready(h, src, grouped, what);
    if (rc) return rc;
    CU(h, cudaSetDevice(h->device));
    CovParams S{};
    static_cast<StatsParams &>(S) = reduction_rows(h, src);
    const uint32_t width = reduction_width(h, src);
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (n_p == 0 || n_p > B200_MAX_COV_PLANES)
        return fail(B200_ERR_INVALID_ARGUMENT, "%u covariance planes: 1 to %u", n_p, B200_MAX_COV_PLANES);
    if (!planes) return fail(B200_ERR_INVALID_ARGUMENT, "null covariance planes");
    uint64_t seen = 0;
    bool channel = false;
    for (uint32_t k = 0; k < n_p; ++k) {
        if (planes[k] >= width)
            return fail(B200_ERR_INVALID_ARGUMENT, "covariance plane %u is %u: the %s has %u planes", k, planes[k], what, width);
        if (seen & (1ull << planes[k])) return fail(B200_ERR_INVALID_ARGUMENT, "covariance plane %u listed twice", planes[k]);
        seen |= 1ull << planes[k];
        channel = channel || planes[k] >= 25;
    }
    const uint64_t n_s = S.planes_per_sample ? S.n_planes / S.planes_per_sample : 0;
    const uint64_t G = reduction_groups(h, grouped).size();
    const uint64_t want = n_s * G * S.n_entities * (1ull + n_p + (uint64_t)n_p * n_p) * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "%s covariance is %llu bytes, got %llu", what, (unsigned long long)want,
                    (unsigned long long)bytes);
    S.n_p = n_p;
    for (uint32_t k = 0; k < n_p; ++k) S.planes[k] = planes[k];
    const b200_sixdof::GroupTables &t = reduction_tables(h, src, grouped);
    return run_world_reduction(h, src, channel, cov_scratch_bytes(S, t.cov), dst, bytes, [&](double *out, void *scratch, int *n) {
        S.out = out;
        return launch_covariance(S, t.cov_dev, t.cov, scratch, n, h->stream);
    });
}

// The ring's width (row_width), not its planes per sample: a handle without a ring refuses every plane.
int b200_sixdof_trajectory_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes)
{
    return run_covariance(h, Rows::ring, false, planes, n_p, dst, bytes, "trajectory");
}

int b200_sixdof_state_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes)
{
    return run_covariance(h, Rows::state, false, planes, n_p, dst, bytes, "state");
}

int b200_sixdof_trajectory_group_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst,
                                            uint64_t bytes)
{
    return run_covariance(h, Rows::ring, true, planes, n_p, dst, bytes, "trajectory");
}

int b200_sixdof_state_group_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes)
{
    return run_covariance(h, Rows::state, true, planes, n_p, dst, bytes, "state");
}

// np.linspace(lo, hi, n + 1) into e[0 .. n]: i * step + lo, the product rounded before the sum (never an fma), e[n] = hi.
// Refused (non-zero) where numpy's histogram rules would be ill-defined: lo or hi not finite, lo >= hi, hi - lo not
// finite, step = 0, or edges that are not strictly increasing.
static int linspace_edges(double lo, double hi, uint32_t n, double *e)
{
    if (!std::isfinite(lo) || !std::isfinite(hi) || !(lo < hi) || !std::isfinite(hi - lo)) return 1;
    const double step = (hi - lo) / (double)n;
    if (step == 0.0) return 1;
    for (uint32_t i = 0; i < n; ++i) {
        volatile double m = (double)i * step;
        e[i] = m + lo;
    }
    e[n] = hi;
    for (uint32_t i = 0; i < n; ++i)
        if (!(e[i] < e[i + 1])) return 1;
    return 0;
}

// Histograms of the specs over the worlds, per group when `grouped` (hist_kernels.cu), into dst: the groups checked,
// then the handle's status, then the specs (each plane < width), then `bytes`.  The edges and the group table are
// computed here and copied to the device ahead of the launch.
static int run_histograms(b200_sixdof *h, Rows src, bool grouped, const b200_histogram *specs, uint32_t n_specs,
                          void *dst, uint64_t bytes, const char *what)
{
    int rc = reduction_ready(h, src, grouped, what);
    if (rc) return rc;
    CU(h, cudaSetDevice(h->device));
    HistParams P{};
    static_cast<StatsParams &>(P) = reduction_rows(h, src);
    const uint32_t width = reduction_width(h, src);
    bool channel = false;
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (n_specs == 0 || n_specs > B200_MAX_HISTOGRAMS)
        return fail(B200_ERR_INVALID_ARGUMENT, "%u histograms: 1 to %u", n_specs, B200_MAX_HISTOGRAMS);
    if (!specs) return fail(B200_ERR_INVALID_ARGUMENT, "null histogram specs");
    std::vector<double> edges;
    for (uint32_t k = 0; k < n_specs; ++k) {
        const b200_histogram &hs = specs[k];
        HistParams::Spec &sp = P.spec[k];
        if (hs.n_axes != 1 && hs.n_axes != 2)
            return fail(B200_ERR_INVALID_ARGUMENT, "histogram %u: %u axes, 1 or 2", k, hs.n_axes);
        if (hs.reserved != 0) return fail(B200_ERR_INVALID_ARGUMENT, "histogram %u: reserved field is not 0", k);
        if (hs.entity >= P.n_entities)
            return fail(B200_ERR_INVALID_ARGUMENT, "histogram %u: entity %llu of %llu", k, (unsigned long long)hs.entity,
                        (unsigned long long)P.n_entities);
        uint64_t cells = 1;
        for (uint32_t a = 0; a < hs.n_axes; ++a) {
            if (hs.plane[a] >= width)
                return fail(B200_ERR_INVALID_ARGUMENT, "histogram %u: plane %u, the %s has %u planes", k, hs.plane[a], what, width);
            if (hs.bins[a] == 0) return fail(B200_ERR_INVALID_ARGUMENT, "histogram %u: 0 bins", k);
            cells *= hs.bins[a];
            channel = channel || hs.plane[a] >= 25;
        }
        if (hs.n_axes == 2 && hs.plane[0] == hs.plane[1])
            return fail(B200_ERR_INVALID_ARGUMENT, "histogram %u: plane %u twice", k, hs.plane[0]);
        if (cells > B200_MAX_HISTOGRAM_CELLS)
            return fail(B200_ERR_INVALID_ARGUMENT, "histogram %u: %llu cells, at most %u", k, (unsigned long long)cells,
                        B200_MAX_HISTOGRAM_CELLS);
        sp.entity = hs.entity;
        sp.n_axes = hs.n_axes;
        sp.rec_off = P.record_len;
        sp.edge_off = edges.size();
        uint32_t n_edges = 0;
        for (uint32_t a = 0; a < hs.n_axes; ++a) {
            sp.plane[a] = hs.plane[a];
            sp.bins[a] = hs.bins[a];
            sp.lo[a] = hs.lo[a];
            sp.hi[a] = hs.hi[a];
            edges.resize(edges.size() + hs.bins[a] + 1);
            if (linspace_edges(hs.lo[a], hs.hi[a], hs.bins[a], edges.data() + edges.size() - (hs.bins[a] + 1)))
                return fail(B200_ERR_INVALID_ARGUMENT,
                            "histogram %u: range (%.17g, %.17g) in %u bins has no strictly increasing finite edges", k,
                            hs.lo[a], hs.hi[a], hs.bins[a]);
            n_edges += hs.bins[a] + 1;
        }
        sp.den = sp.hi[0] - sp.lo[0];
        P.smem_edges = std::max(P.smem_edges, n_edges);
        P.record_len += hs.n_axes == 2 ? 2 + cells : 3 + cells;
    }
    P.n_specs = n_specs;
    const uint64_t n_s = P.planes_per_sample ? P.n_planes / P.planes_per_sample : 0;
    const std::vector<uint64_t> sizes = reduction_groups(h, grouped);
    const uint64_t want = n_s * sizes.size() * P.record_len * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "%s histograms are %llu bytes, got %llu", what, (unsigned long long)want,
                    (unsigned long long)bytes);
    const std::vector<WorldGroup> table = hist_group_table(sizes.data(), sizes.size(), n_s * n_specs);
    const uint64_t edge_bytes = edges.size() * 8ull, table_bytes = table.size() * sizeof(WorldGroup);
    edges.resize(edges.size() + table_bytes / 8);  // one copy to the device: the edges, then the group table
    std::memcpy(edges.data() + edge_bytes / 8, table.data(), table_bytes);
    return run_world_reduction(h, src, channel, edge_bytes + table_bytes, dst, bytes, [&](double *out, void *scratch, int *n) {
        cudaError_t e = cudaMemcpyAsync(scratch, edges.data(), edge_bytes + table_bytes, cudaMemcpyHostToDevice, h->stream);
        if (e != cudaSuccess) return e;
        P.out = out;
        P.edges = (const double *)scratch;
        return launch_histograms(P, (const WorldGroup *)((char *)scratch + edge_bytes), table, n, h->stream);
    });
}

int b200_sixdof_trajectory_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                      uint64_t bytes)
{
    return run_histograms(h, Rows::ring, false, specs, n_specs, dst, bytes, "trajectory");
}

int b200_sixdof_state_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst, uint64_t bytes)
{
    return run_histograms(h, Rows::state, false, specs, n_specs, dst, bytes, "state");
}

int b200_sixdof_trajectory_group_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                            uint64_t bytes)
{
    return run_histograms(h, Rows::ring, true, specs, n_specs, dst, bytes, "trajectory");
}

int b200_sixdof_state_group_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                       uint64_t bytes)
{
    return run_histograms(h, Rows::state, true, specs, n_specs, dst, bytes, "state");
}

// Host-only, like b200_stats_merge: parts folded left to right with the kernels' cov_merge, entry by entry.
int b200_covariance_merge(const double *parts, uint32_t n_parts, uint64_t n_groups, uint32_t n_p, double *out)
{
    if (n_p == 0 || n_p > B200_MAX_COV_PLANES)
        return fail(B200_ERR_INVALID_ARGUMENT, "%u covariance planes: 1 to %u", n_p, B200_MAX_COV_PLANES);
    if (n_groups && (!out || (n_parts && !parts))) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
    const uint64_t R = 1 + n_p + (uint64_t)n_p * n_p;
    for (uint32_t k = 0; k < n_parts; ++k)
        for (uint64_t g = 0; g < n_groups; ++g) {
            const double n = parts[((uint64_t)k * n_groups + g) * R];
            if (!(n >= 0.0))
                return fail(B200_ERR_INVALID_ARGUMENT, "part %u, group %llu: count %g is not a count", k, (unsigned long long)g, n);
        }
    const double nan = std::nan("");
    for (uint64_t g = 0; g < n_groups; ++g) {
        double *o = out + g * R;
        for (uint32_t a = 0; a < n_p; ++a)
            for (uint32_t b = a; b < n_p; ++b) {
                CovEntry acc{0.0, 0.0, 0.0, 0.0};
                for (uint32_t k = 0; k < n_parts; ++k) {
                    const double *q = parts + ((uint64_t)k * n_groups + g) * R;
                    cov_merge(acc, CovEntry{q[0], q[1 + a], q[1 + b], q[1 + n_p + a * n_p + b]});
                }
                const bool any = acc.n > 0.0;
                if (a == 0 && b == 0) o[0] = acc.n;
                if (a == b) o[1 + a] = any ? acc.ma : nan;
                o[1 + n_p + a * n_p + b] = any ? acc.m : nan;
                o[1 + n_p + b * n_p + a] = any ? acc.m : nan;
            }
    }
    return B200_OK;
}

// The cross-rank step of a world-sharded campaign: host-only, no GPU needed (a Rust host merges its ranks' tables
// without torch).  Parts are folded left to right with the kernels' stats_merge, so the result does not depend on who
// calls it.
int b200_stats_merge(const double *parts, uint32_t n_parts, uint64_t n_groups, double *out)
{
    if (n_groups && (!out || (n_parts && !parts))) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
    const double nan = std::nan("");
    for (uint64_t g = 0; g < n_groups; ++g) {
        StatsGroup acc{0.0, 0.0, 0.0, 0.0, 0.0};
        for (uint32_t p = 0; p < n_parts; ++p) {
            const double *q = parts + ((uint64_t)p * n_groups + g) * 5;
            if (!(q[0] >= 0.0)) return fail(B200_ERR_INVALID_ARGUMENT, "part %u, group %llu: count %g is not a count", p,
                                             (unsigned long long)g, q[0]);
            stats_merge(acc, StatsGroup{q[0], q[1], q[2], q[3], q[4]});
        }
        double *o = out + g * 5;
        const bool any = acc.n > 0.0;
        o[0] = acc.n;
        o[1] = any ? acc.mean : nan;
        o[2] = any ? acc.m2 : nan;
        o[3] = any ? acc.mn : nan;
        o[4] = any ? acc.mx : nan;
    }
    return B200_OK;
}

// The fold parameters of the handle's summary accumulators; run_summary_fold fills in the rows.
static SummaryParams summary_params(const b200_sixdof *h)
{
    SummaryParams S{};
    S.ld = h->ld;
    S.n_bodies = h->n_bodies;
    S.n_entities = (uint32_t)h->desc.n_entities;
    S.n_thr = (uint32_t)h->sum_thr_list.size();
    S.ext = h->sum_extrema ? h->sum_ext : nullptr;
    S.thr = S.n_thr ? h->sum_thr : nullptr;
    for (uint32_t i = 0; i < S.n_thr; ++i) {
        const b200_threshold &t = h->sum_thr_list[i];
        S.t[i] = {(uint32_t)t.entity, t.plane, t.above ? 1 : 0, 0u, t.value};
    }
    S.n_mom = (uint32_t)h->sum_mom_planes.size();
    S.mom = S.n_mom ? h->sum_mom : nullptr;
    S.n_dwell = (uint32_t)h->sum_dwell_list.size();
    S.dwell = S.n_dwell ? h->sum_dwell : nullptr;
    for (uint32_t i = 0; i < S.n_dwell; ++i) {
        const b200_threshold &t = h->sum_dwell_list[i];
        S.d[i] = {(uint32_t)t.entity, t.plane, t.above ? 1 : 0, 0u, t.value};
    }
    S.width = row_width(h, false);
    for (uint32_t p = 0; p < S.width; ++p) {
        bool used = h->sum_extrema;
        for (uint32_t i = 0; i < S.n_thr; ++i) used = used || S.t[i].plane == p;
        for (uint32_t i = 0; i < S.n_dwell; ++i) used = used || S.d[i].plane == p;
        uint8_t slot = kNoMoment;
        for (uint32_t j = 0; j < S.n_mom; ++j)
            if (h->sum_mom_planes[j] == p) slot = (uint8_t)j;
        if (used || slot != kNoMoment) {
            S.mom_slot[S.n_planes] = slot;
            S.planes[S.n_planes++] = (uint8_t)p;
        }
    }
    return S;
}

static int summary_ready(b200_sixdof *h, const char *what)
{
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (!h->sum_begun) return fail(B200_ERR_INVALID_ARGUMENT, "%s: call b200_sixdof_summary_begin first", what);
    return B200_OK;
}

// Fold the samples of the ring (ring) or the state as rows, sample k at tick tick0 + k * tick_step: row[p] is plane p of
// sample 0, and each sample's planes start one segment stride after the one before it.  The channel planes are
// recomputed first where the fold reads one: with extrema, or a threshold, moment or dwell on a channel plane.
static int run_summary_fold(b200_sixdof *h, bool ring, uint64_t tick0, uint64_t tick_step)
{
    ++h->sum_gen;
    SummaryParams S = summary_params(h);
    const StatsParams P = ensemble_rows(h, ring);
    bool channel = false;
    for (uint32_t i = 0; i < S.n_planes; ++i) channel = channel || S.planes[i] >= 25;
    if (channel) {
        const int rc = refresh_channels(h, ring);
        if (rc) return rc;
    }
    uint32_t p = 0;
    for (uint32_t k = 0; k < P.n_segs; ++k)
        for (uint64_t j = 0; j < P.seg[k].n_planes && p < kMaxRow; ++j) S.row[p++] = P.seg[k].base + j * P.ld;
    S.row_stride = P.seg[0].stride;
    S.chan_stride = P.seg[P.n_segs - 1].stride;
    S.n_rows = P.n_planes / P.planes_per_sample;
    S.tick0 = tick0;
    S.tick_step = tick_step;
    int launches = 0;
    CU(h, launch_summary_fold(S, &launches, h->stream));
    h->timings.kernel_launches += (uint64_t)launches;
    return B200_OK;
}

// A threshold or dwell condition `what` i: 0 when it keeps the contract of include/b200_sixdof.h, else the refusal.
static int check_condition(const b200_sixdof *h, const b200_threshold &t, const char *what, uint32_t i)
{
    if (t.entity >= h->desc.n_entities)
        return fail(B200_ERR_INVALID_ARGUMENT, "%s %u: entity row %llu, the world has %llu", what, i,
                    (unsigned long long)t.entity, (unsigned long long)h->desc.n_entities);
    if (t.plane >= row_width(h, false))
        return fail(B200_ERR_INVALID_ARGUMENT, "%s %u: plane %u, a row has %u", what, i, t.plane, row_width(h, false));
    if (std::isnan(t.value)) return fail(B200_ERR_INVALID_ARGUMENT, "%s %u: the bound is NaN", what, i);
    return B200_OK;
}

// summary_begin and summary_start (`nothing`: the refusal of a spec that requests nothing): every argument checked
// before anything changes, then the accumulators allocated on first use, the spec stored and everything cleared on the
// handle's stream.
static int summary_start(b200_sixdof *h, const b200_summary_spec &sp, const char *nothing)
{
    ++h->sum_gen;
    CU(h, cudaSetDevice(h->device));
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (sp.n_thresholds > B200_MAX_THRESHOLDS)
        return fail(B200_ERR_INVALID_ARGUMENT, "%u thresholds: at most %u", sp.n_thresholds, B200_MAX_THRESHOLDS);
    if (!sp.extrema && sp.n_thresholds == 0 && sp.n_moments == 0 && sp.n_dwells == 0)
        return fail(B200_ERR_INVALID_ARGUMENT, "%s", nothing);
    if (sp.n_thresholds && !sp.thresholds) return fail(B200_ERR_INVALID_ARGUMENT, "null thresholds");
    for (uint32_t i = 0; i < sp.n_thresholds; ++i) {
        const int rc = check_condition(h, sp.thresholds[i], "threshold", i);
        if (rc) return rc;
    }
    const uint32_t R = row_width(h, false);
    if (sp.n_moments && !sp.moments) return fail(B200_ERR_INVALID_ARGUMENT, "null moment planes");
    for (uint32_t j = 0; j < sp.n_moments; ++j) {
        if (sp.moments[j] >= R) return fail(B200_ERR_INVALID_ARGUMENT, "moment %u: plane %u, a row has %u", j, sp.moments[j], R);
        for (uint32_t i = 0; i < j; ++i)
            if (sp.moments[i] == sp.moments[j])
                return fail(B200_ERR_INVALID_ARGUMENT, "moments: plane %u twice", sp.moments[j]);
    }
    if (sp.n_dwells > B200_MAX_DWELLS)
        return fail(B200_ERR_INVALID_ARGUMENT, "%u dwells: at most %u", sp.n_dwells, B200_MAX_DWELLS);
    if (sp.n_dwells && !sp.dwells) return fail(B200_ERR_INVALID_ARGUMENT, "null dwells");
    for (uint32_t i = 0; i < sp.n_dwells; ++i) {
        const int rc = check_condition(h, sp.dwells[i], "dwell", i);
        if (rc) return rc;
    }
    h->sum_begun = false;
    h->sum_ever = true;  // the channel set, and so R, stays as it is from here on
    if (sp.extrema && !h->sum_ext) CU(h, cudaMalloc(&h->sum_ext, 5ull * R * h->ld * 8ull));
    const uint64_t thr_bytes = h->desc.n_worlds * sp.n_thresholds * 26ull * 8ull;
    int rc = grow_device(h, &h->sum_thr, &h->sum_thr_bytes, thr_bytes);
    if (rc) return rc;
    if ((rc = grow_device(h, &h->sum_mom, &h->sum_mom_bytes, 4ull * sp.n_moments * h->ld * 8ull))) return rc;
    if ((rc = grow_device(h, &h->sum_dwell, &h->sum_dwell_bytes, h->desc.n_worlds * sp.n_dwells * 3ull * 8ull))) return rc;
    h->sum_extrema = sp.extrema != 0;
    h->sum_thr_list.assign(sp.thresholds, sp.thresholds + sp.n_thresholds);
    h->sum_mom_planes.assign(sp.moments, sp.moments + sp.n_moments);
    h->sum_dwell_list.assign(sp.dwells, sp.dwells + sp.n_dwells);
    int launches = 0;
    CU(h, launch_summary_clear(summary_params(h), &launches, h->stream));
    h->timings.kernel_launches += (uint64_t)launches;
    h->sum_begun = true;
    return B200_OK;
}

int b200_sixdof_summary_begin(b200_sixdof *h, uint32_t extrema, const b200_threshold *t, uint32_t n_thresholds)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    b200_summary_spec sp{};
    sp.extrema = extrema;
    sp.n_thresholds = n_thresholds;
    sp.thresholds = t;
    return summary_start(h, sp, "summary_begin: neither extrema nor thresholds");
}

int b200_sixdof_summary_start(b200_sixdof *h, const b200_summary_spec *spec)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (!spec) return fail(B200_ERR_INVALID_ARGUMENT, "null summary spec");
    return summary_start(h, *spec, "summary_start: no extrema, thresholds, moments or dwells");
}

int b200_sixdof_summary_add_state(b200_sixdof *h)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    int rc = summary_ready(h, "summary_add_state");
    if (rc) return rc;
    return run_summary_fold(h, false, h->tick, 0);
}

int b200_sixdof_summary_add_trajectory(b200_sixdof *h)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    int rc = summary_ready(h, "summary_add_trajectory");
    if (rc) return rc;
    if (!h->traj || h->traj_planes != 25)
        return fail(B200_ERR_INVALID_ARGUMENT, "summary_add_trajectory needs a B200_TRAJ_FULL trajectory ring");
    // sample k was recorded when the ticks since the reset reached (k + 1) * every (sixdof_tick.cuh traj slots)
    const uint64_t every = h->desc.trajectory_every;
    return run_summary_fold(h, true, h->tick - h->ticks_done + every, every);
}

// A per-body table of per_body bytes into dst, `table` writing bodies [b0, b0 + nb) of it: dst on the handle's GPU
// takes the table straight from the kernel; any other goes through the staging buffer in chunks of 256 MB.
extern "C++" {
template <class Table>
static int body_table_download(b200_sixdof *h, void *dst, uint64_t per_body, Table table)
{
    if (h->n_bodies * per_body == 0) return B200_OK;
    if (!dst) return fail(B200_ERR_INVALID_ARGUMENT, "null destination buffer");
    const bool direct = device_destination(h, dst);
    const uint64_t chunk = direct ? h->n_bodies : std::max<uint64_t>(1, std::min<uint64_t>(h->n_bodies, (256ull << 20) / per_body));
    int rc = B200_OK;
    if (!direct && (rc = ensure_staging(h, chunk * per_body))) return rc;
    for (uint64_t b0 = 0; b0 < h->n_bodies; b0 += chunk) {
        const uint64_t nb = std::min(chunk, h->n_bodies - b0);
        double *out = direct ? (double *)dst : h->staging;
        CU(h, table(b0, nb, out));
        h->timings.kernel_launches++;
        if (!direct) CU(h, cudaMemcpyAsync((char *)dst + b0 * per_body, out, nb * per_body, cudaMemcpyDefault, h->stream));
        CU(h, cudaStreamSynchronize(h->stream)); // the staging buffer is reused by the next chunk
    }
    return B200_OK;
}
}

int b200_sixdof_extrema_download(b200_sixdof *h, void *dst, uint64_t bytes)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    int rc = summary_ready(h, "extrema_download");
    if (rc) return rc;
    if (!h->sum_extrema) return fail(B200_ERR_INVALID_ARGUMENT, "extrema_download: summary_begin had no extrema");
    const uint32_t width = row_width(h, false);
    const uint64_t per_body = 5ull * width * 8ull;
    const uint64_t want = h->n_bodies * per_body;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "extrema are %llu bytes, got %llu", (unsigned long long)want,
                    (unsigned long long)bytes);
    return body_table_download(h, dst, per_body, [&](uint64_t b0, uint64_t nb, double *out) {
        return launch_extrema_table(h->sum_ext, h->ld, width, b0, nb, out, h->stream);
    });
}

int b200_sixdof_moments_download(b200_sixdof *h, void *dst, uint64_t bytes)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    int rc = summary_ready(h, "moments_download");
    if (rc) return rc;
    const uint32_t k = (uint32_t)h->sum_mom_planes.size();
    if (k == 0) return fail(B200_ERR_INVALID_ARGUMENT, "moments_download: the summary has no moments");
    const uint64_t per_body = 3ull * k * 8ull;
    const uint64_t want = h->n_bodies * per_body;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "moments are %llu bytes, got %llu", (unsigned long long)want,
                    (unsigned long long)bytes);
    return body_table_download(h, dst, per_body, [&](uint64_t b0, uint64_t nb, double *out) {
        return launch_moment_table(h->sum_mom, h->ld, k, b0, nb, out, h->stream);
    });
}

int b200_sixdof_thresholds_download(b200_sixdof *h, void *dst, uint64_t bytes)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    int rc = summary_ready(h, "thresholds_download");
    if (rc) return rc;
    if (h->sum_thr_list.empty()) return fail(B200_ERR_INVALID_ARGUMENT, "thresholds_download: summary_begin had no thresholds");
    const uint64_t want = h->desc.n_worlds * h->sum_thr_list.size() * 26ull * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "threshold events are %llu bytes, got %llu", (unsigned long long)want,
                    (unsigned long long)bytes);
    if (want == 0) return B200_OK;
    if (!dst) return fail(B200_ERR_INVALID_ARGUMENT, "null destination buffer");
    CU(h, cudaMemcpyAsync(dst, h->sum_thr, want, cudaMemcpyDefault, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return B200_OK;
}

int b200_sixdof_dwells_download(b200_sixdof *h, void *dst, uint64_t bytes)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    int rc = summary_ready(h, "dwells_download");
    if (rc) return rc;
    if (h->sum_dwell_list.empty()) return fail(B200_ERR_INVALID_ARGUMENT, "dwells_download: the summary has no dwells");
    const uint64_t want = h->desc.n_worlds * h->sum_dwell_list.size() * 3ull * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "dwell records are %llu bytes, got %llu", (unsigned long long)want,
                    (unsigned long long)bytes);
    if (want == 0) return B200_OK;
    if (!dst) return fail(B200_ERR_INVALID_ARGUMENT, "null destination buffer");
    CU(h, cudaMemcpyAsync(dst, h->sum_dwell, want, cudaMemcpyDefault, h->stream));
    CU(h, cudaStreamSynchronize(h->stream));
    return B200_OK;
}

// ---- derived channels (channel_kernels.cu)

// channel k of c: 0 when it keeps the contract of include/b200_sixdof.h, else the refusal
static int check_channel(const b200_channel &ch, uint32_t k)
{
    auto finite3 = [](const double *v) { return std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]); };
    auto zero3 = [](const double *v) { return v[0] == 0.0 && v[1] == 0.0 && v[2] == 0.0; };
    if (ch.reserved != 0) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: reserved field is not 0", k);
    if (ch.kind == B200_CHANNEL_NORM) {
        if (ch.n < 1 || ch.n > 3) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: a norm of %u planes, 1 to 3", k, ch.n);
        for (uint32_t i = 0; i < ch.n; ++i) {
            if (ch.plane[i] >= 25) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: plane %u, a row has 25", k, ch.plane[i]);
            for (uint32_t j = 0; j < i; ++j)
                if (ch.plane[j] == ch.plane[i]) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: plane %u twice", k, ch.plane[i]);
            if (!std::isfinite(ch.c[i])) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: offset %u is not finite", k, i);
        }
        if (!std::isfinite(ch.r0)) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: r0 is not finite", k);
        return B200_OK;
    }
    if (ch.kind == B200_CHANNEL_AXIS_ANGLE) {
        if (ch.n != 0 && ch.n != 3)
            return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: an axis angle takes n = 0 (fixed direction) or 3 (planes), not %u",
                        k, ch.n);
        if (ch.n == 3 && ch.plane[0] > 22)
            return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: planes %u .. %u run past plane 24", k, ch.plane[0], ch.plane[0] + 2);
        if (!finite3(ch.c)) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: the body axis is not finite", k);
        if (zero3(ch.c)) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: the body axis is zero", k);
        if (ch.n == 0 && !finite3(ch.d)) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: the direction is not finite", k);
        if (ch.n == 0 && zero3(ch.d)) return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: the direction is zero", k);
        return B200_OK;
    }
    return fail(B200_ERR_INVALID_ARGUMENT, "channel %u: unknown kind %u", k, ch.kind);
}

int b200_sixdof_set_channels(b200_sixdof *h, const b200_channel *c, uint32_t n)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (n > B200_MAX_CHANNELS) return fail(B200_ERR_INVALID_ARGUMENT, "%u channels: at most %u", n, B200_MAX_CHANNELS);
    if (n && !c) return fail(B200_ERR_INVALID_ARGUMENT, "null channels");
    if (h->traj && h->traj_planes != 25)
        return fail(B200_ERR_INVALID_ARGUMENT, "channels need a B200_TRAJ_FULL trajectory ring: this one is %u wide",
                    h->traj_planes);
    if (h->sum_ever)
        return fail(B200_ERR_INVALID_ARGUMENT, "set_channels after b200_sixdof_summary_begin: the summary's row width is fixed");
    for (uint32_t k = 0; k < n; ++k) {
        const int rc = check_channel(c[k], k);
        if (rc) return rc;
    }
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaStreamSynchronize(h->stream));  // no reduction in flight still reads the planes replaced here
    double *ring = nullptr, *state = nullptr;
    if (n) {
        const cudaError_t e = cudaMalloc(&state, (uint64_t)n * h->ld * 8ull);
        if (e != cudaSuccess) return cuda_fail(h, e, "cudaMalloc(channel state planes)");
        if (h->traj) {
            const cudaError_t e2 = cudaMalloc(&ring, h->desc.trajectory_capacity * n * h->ld * 8ull);
            if (e2 != cudaSuccess) {
                cudaFree(state);
                return cuda_fail(h, e2, "cudaMalloc(channel ring planes)");
            }
        }
    }
    if (h->chan_ring) CU(h, cudaFree(h->chan_ring));
    if (h->chan_state) CU(h, cudaFree(h->chan_state));
    h->chan_ring = ring;
    h->chan_state = state;
    h->channels.assign(c, c + n);
    ++h->rows_gen;
    return B200_OK;
}

uint32_t b200_sixdof_channels(const b200_sixdof *h) { return h ? (uint32_t)h->channels.size() : 0; }

// The channel planes of the ring's samples (ring) or of the state, recomputed, into dst = [samples][n_bodies][n_c] in
// slices of at most 256 MiB of samples through the staging buffer.
static int download_channels(b200_sixdof *h, bool ring, void *dst, uint64_t bytes, const char *what)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    const uint64_t n = ring ? b200_sixdof_trajectory_len(h) : 1, W = h->channels.size();
    const uint64_t per_sample = h->n_bodies * W * 8ull, want = n * per_sample;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "%s channels are %llu bytes, got %llu", what, (unsigned long long)want,
                    (unsigned long long)bytes);
    if (want == 0) return B200_OK;
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (!dst) return fail(B200_ERR_INVALID_ARGUMENT, "null destination buffer");
    int rc = refresh_channels(h, ring);
    if (rc) return rc;
    const double *planes = ring ? h->chan_ring : h->chan_state;
    const uint64_t chunk = std::max<uint64_t>(1, std::min<uint64_t>(n, (256ull << 20) / per_sample));
    if ((rc = ensure_staging(h, chunk * per_sample))) return rc;
    for (uint64_t s0 = 0; s0 < n; s0 += chunk) {
        const uint64_t ns = std::min(chunk, n - s0);
        CU(h, launch_traj_to_aos(planes + s0 * W * h->ld, h->staging, ns, h->n_bodies, h->ld, (uint32_t)W, h->stream));
        h->timings.kernel_launches++;
        CU(h, cudaMemcpyAsync((char *)dst + s0 * per_sample, h->staging, ns * per_sample, cudaMemcpyDefault, h->stream));
        CU(h, cudaStreamSynchronize(h->stream));
    }
    return B200_OK;
}

int b200_sixdof_trajectory_channels(b200_sixdof *h, void *dst, uint64_t bytes)
{
    return download_channels(h, true, dst, bytes, "trajectory");
}

int b200_sixdof_state_channels(b200_sixdof *h, void *dst, uint64_t bytes)
{
    return download_channels(h, false, dst, bytes, "state");
}

// ---- outcomes (outcome_kernels.cu)

// outcome k of the set: 0 when it names a record the handle has now (the summary in force, a device column), else the
// refusal.  Every outcome entry repeats it: a later summary_start may have dropped what an outcome names.
static int check_outcome(const b200_sixdof *h, const b200_outcome &o, uint32_t k)
{
    const uint64_t E = h->desc.n_entities;
    if (o.reserved != 0) return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: reserved field is not 0", k);
    const bool per_entity = o.kind == B200_OUTCOME_EXTREMA || o.kind == B200_OUTCOME_MOMENT || o.kind == B200_OUTCOME_COLUMN;
    if (per_entity ? o.entity >= E : o.entity != 0)
        return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: entity row %llu, %s", k, (unsigned long long)o.entity,
                    per_entity ? "beyond the world's entities" : "its kind takes none (0)");
    if (o.kind != B200_OUTCOME_COLUMN && o.column != 0)
        return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: column 0x%016llx, its kind takes none (0)", k,
                    (unsigned long long)o.column);
    auto bad_field = [&](uint32_t n) {
        return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: field %u, kind %u has fields 0 to %u", k, o.field, o.kind, n - 1);
    };
    auto past = [&](const char *what, size_t have) {
        return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: %s %u, the summary in force has %zu", k, what, o.index, have);
    };
    switch (o.kind) {
    case B200_OUTCOME_EXTREMA:
        if (o.field >= B200_EXTREMA_FIELDS) return bad_field(B200_EXTREMA_FIELDS);
        if (!h->sum_begun || !h->sum_extrema)
            return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: the summary in force has no extrema", k);
        if (o.index >= row_width(h, false))
            return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: extrema plane %u, a row has %u", k, o.index, row_width(h, false));
        return B200_OK;
    case B200_OUTCOME_THRESHOLD:
        if (o.field > 25) return bad_field(26);
        if (o.index >= (h->sum_begun ? h->sum_thr_list.size() : 0)) return past("threshold", h->sum_begun ? h->sum_thr_list.size() : 0);
        return B200_OK;
    case B200_OUTCOME_MOMENT:
        if (o.field >= 4) return bad_field(4);
        if (o.index >= (h->sum_begun ? h->sum_mom_planes.size() : 0)) return past("moment slot", h->sum_begun ? h->sum_mom_planes.size() : 0);
        return B200_OK;
    case B200_OUTCOME_DWELL:
        if (o.field >= B200_DWELL_FIELDS) return bad_field(B200_DWELL_FIELDS);
        if (o.index >= (h->sum_begun ? h->sum_dwell_list.size() : 0)) return past("dwell", h->sum_begun ? h->sum_dwell_list.size() : 0);
        return B200_OK;
    case B200_OUTCOME_COLUMN: {
        if (o.index != 0) return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: index %u, a column outcome takes 0", k, o.index);
        const Column *c = h->find(o.column);
        if (!c) return fail(B200_ERR_COMPONENT_NOT_FOUND, "outcome %u: component 0x%016llx not found", k, (unsigned long long)o.column);
        if (c->global)
            return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: column 0x%016llx is global, not per body", k, (unsigned long long)o.column);
        if (o.field >= c->width)
            return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: plane %u, the column has %u", k, o.field, c->width);
        return B200_OK;
    }
    case B200_OUTCOME_VALUES:
        if (o.field != 0) return bad_field(1);
        if (o.index != 0) return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: index %u, a values outcome takes 0", k, o.index);
        return B200_OK;
    default:
        return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: unknown kind %u", k, o.kind);
    }
}

static int check_outcomes(const b200_sixdof *h)
{
    if (h->outcomes.empty()) return fail(B200_ERR_INVALID_ARGUMENT, "no outcomes: call b200_sixdof_set_outcomes first");
    for (uint32_t k = 0; k < h->outcomes.size(); ++k) {
        const int rc = check_outcome(h, h->outcomes[k], k);
        if (rc) return rc;
    }
    return B200_OK;
}

// The outcome pass of the set in force (checked by check_outcomes): each outcome resolved to its record, the pointers
// taken from the handle now (summary_start may have moved the accumulators).
static OutcomeParams outcome_params(const b200_sixdof *h)
{
    OutcomeParams P{};
    const uint64_t E = h->desc.n_entities, ld = h->ld;
    for (uint32_t k = 0; k < h->outcomes.size(); ++k) {
        const b200_outcome &o = h->outcomes[k];
        OutcomeParams::Src s{nullptr, E, kOutCopy, k};
        switch (o.kind) {
        case B200_OUTCOME_EXTREMA:  // SoA: plane p * 5 + f of ld, body w * E + e
            s.src = h->sum_ext + ((uint64_t)o.index * B200_EXTREMA_FIELDS + o.field) * ld + o.entity;
            s.op = o.field >= 2 ? kOutTick : kOutCopy;
            break;
        case B200_OUTCOME_THRESHOLD:  // [w][n_thr][26]
            s.src = h->sum_thr + (uint64_t)o.index * 26 + o.field;
            s.stride = h->sum_thr_list.size() * 26;
            s.op = o.field == 0 ? kOutTick : kOutCopy;
            break;
        case B200_OUTCOME_MOMENT:  // SoA: (n, K, S1, S2) at plane j * 4 + f of ld
            s.src = h->sum_mom + (uint64_t)o.index * 4 * ld + o.entity;
            s.op = kOutCount + o.field;
            break;
        case B200_OUTCOME_DWELL:  // [w][n_dwell][3]
            s.src = h->sum_dwell + (uint64_t)o.index * B200_DWELL_FIELDS + o.field;
            s.stride = h->sum_dwell_list.size() * B200_DWELL_FIELDS;
            s.op = o.field == 0 ? kOutCopy : kOutTick;
            break;
        case B200_OUTCOME_COLUMN:
            s.src = h->find(o.column)->dev + (uint64_t)o.field * ld + o.entity;
            break;
        default:  // VALUES: written by set_outcomes
            continue;
        }
        P.o[P.n_src++] = s;
    }
    P.out = h->out_planes;
    P.ld_o = h->ld_o;
    P.ld = ld;
    P.n_worlds = h->desc.n_worlds;
    return P;
}

// The outcome planes of every source, written on the handle's stream (one launch; none with only VALUES outcomes).
// Never cached: the summaries fold, and b200_sixdof_device_plane hands out writable columns.
static int write_outcomes(b200_sixdof *h)
{
    int launches = 0;
    CU(h, launch_outcomes(outcome_params(h), &launches, h->stream));
    h->timings.kernel_launches += (uint64_t)launches;
    return B200_OK;
}

int b200_sixdof_set_outcomes(b200_sixdof *h, const b200_outcome *o, uint32_t n)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (n > B200_MAX_OUTCOMES) return fail(B200_ERR_INVALID_ARGUMENT, "%u outcomes: at most %u", n, B200_MAX_OUTCOMES);
    if (n && !o) return fail(B200_ERR_INVALID_ARGUMENT, "null outcomes");
    for (uint32_t k = 0; k < n; ++k) {
        const int rc = check_outcome(h, o[k], k);
        if (rc) return rc;
        if ((o[k].kind == B200_OUTCOME_VALUES) != (o[k].values != nullptr))
            return fail(B200_ERR_INVALID_ARGUMENT, "outcome %u: %s", k,
                        o[k].values ? "values given, its kind takes none (NULL)" : "null values");
    }
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaStreamSynchronize(h->stream));  // no reduction in flight still reads the planes replaced here
    const uint64_t ld_o = round_up(std::max<uint64_t>(h->desc.n_worlds, 1), 128);
    double *planes = nullptr;
    if (n) {
        cudaError_t e = cudaMalloc(&planes, (uint64_t)n * ld_o * 8ull);
        if (e != cudaSuccess) return cuda_fail(h, e, "cudaMalloc(outcome planes)");
        for (uint32_t k = 0; k < n && e == cudaSuccess; ++k)
            if (o[k].kind == B200_OUTCOME_VALUES)
                e = cudaMemcpy(planes + k * ld_o, o[k].values, h->desc.n_worlds * 8ull, cudaMemcpyDefault);
        if (e != cudaSuccess) {
            cudaFree(planes);
            return cuda_fail(h, e, "cudaMemcpy(outcome values)");
        }
    }
    ++h->rows_gen;
    if (h->out_planes) CU(h, cudaFree(h->out_planes));
    h->out_planes = planes;
    if (h->rank_planes) CU(h, cudaFree(h->rank_planes));  // the next rank call allocates for the new set
    h->rank_planes = nullptr;
    h->rank_bytes = 0;
    if (h->sobol_planes) CU(h, cudaFree(h->sobol_planes));
    h->sobol_planes = nullptr;
    h->sobol_bytes = 0;
    h->ld_o = ld_o;
    h->outcomes.assign(o, o + n);
    for (auto &x : h->outcomes) x.values = nullptr;
    int rc = build_outcome_tables(h, &h->desc.n_worlds, 1, false);
    if (!rc) rc = build_outcome_tables(h, h->group_sizes.data(), (uint32_t)h->group_sizes.size(), true);
    return rc;
}

uint32_t b200_sixdof_outcomes(const b200_sixdof *h) { return h ? (uint32_t)h->outcomes.size() : 0; }

// [n_worlds][P]: the outcome planes written, then turned into world-major rows (the layout kernel of the columns)
int b200_sixdof_outcome_values(b200_sixdof *h, void *dst, uint64_t bytes)
{
    int rc = reduction_ready(h, Rows::outcomes, false, "outcome");
    if (rc) return rc;
    CU(h, cudaSetDevice(h->device));
    const uint64_t P = h->outcomes.size(), want = h->desc.n_worlds * P * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "outcome values are %llu bytes, got %llu", (unsigned long long)want,
                    (unsigned long long)bytes);
    return run_world_reduction(h, Rows::outcomes, false, 0, dst, bytes, [&](double *out, void *, int *n) {
        *n = 1;
        return launch_soa_to_aos(h->out_planes, out, h->desc.n_worlds, (uint32_t)P, h->ld_o, h->stream);
    });
}

int b200_sixdof_outcome_stats(b200_sixdof *h, void *dst, uint64_t bytes)
{
    return run_world_stats(h, Rows::outcomes, false, dst, bytes, "outcome");
}

int b200_sixdof_outcome_group_stats(b200_sixdof *h, void *dst, uint64_t bytes)
{
    return run_world_stats(h, Rows::outcomes, true, dst, bytes, "outcome");
}

int b200_sixdof_outcome_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes)
{
    return run_quantiles(h, Rows::outcomes, false, q, n_q, dst, bytes, "outcome");
}

int b200_sixdof_outcome_group_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes)
{
    return run_quantiles(h, Rows::outcomes, true, q, n_q, dst, bytes, "outcome");
}

int b200_sixdof_outcome_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes)
{
    return run_covariance(h, Rows::outcomes, false, planes, n_p, dst, bytes, "outcome");
}

int b200_sixdof_outcome_group_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes)
{
    return run_covariance(h, Rows::outcomes, true, planes, n_p, dst, bytes, "outcome");
}

int b200_sixdof_outcome_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                   uint64_t bytes)
{
    return run_histograms(h, Rows::outcomes, false, specs, n_specs, dst, bytes, "outcome");
}

int b200_sixdof_outcome_group_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                         uint64_t bytes)
{
    return run_histograms(h, Rows::outcomes, true, specs, n_specs, dst, bytes, "outcome");
}

// The checks of a call over selected outcome planes (top worlds, ranks, sobol) on the outcome set, groups and
// selection, in order; least: the fewest planes; noun names the planes in the messages
static int outcome_selection(b200_sixdof *h, bool grouped, const uint32_t *planes, uint32_t n_p, uint32_t least,
                             const char *what, const char *noun = "rank")
{
    int rc = reduction_ready(h, Rows::outcomes, grouped, what);
    if (rc) return rc;
    CU(h, cudaSetDevice(h->device));
    const uint32_t P = (uint32_t)h->outcomes.size();
    if (!planes) return fail(B200_ERR_INVALID_ARGUMENT, "null %s planes", noun);
    if (n_p < least || n_p > P) return fail(B200_ERR_INVALID_ARGUMENT, "%u %s planes: %u to %u", n_p, noun, least, P);
    uint64_t seen = 0;
    for (uint32_t j = 0; j < n_p; ++j) {
        if (planes[j] >= P)
            return fail(B200_ERR_INVALID_ARGUMENT, "%s plane %u is %u: the outcome has %u planes", noun, j, planes[j], P);
        if (seen & (1ull << planes[j]))
            return fail(B200_ERR_INVALID_ARGUMENT, "%s plane %u listed twice", noun, planes[j]);
        seen |= 1ull << planes[j];
    }
    return B200_OK;
}

// The k worst worlds of the selected outcome planes, per group when `grouped` (topk_kernels.cu), into dst: the outcome
// set and groups checked, then the selection, k, largest and `bytes`; the handle's status in run_world_reduction.
static int run_top_worlds(b200_sixdof *h, bool grouped, const uint32_t *planes, uint32_t n_p, uint32_t k, int largest,
                          void *dst, uint64_t bytes)
{
    int rc = outcome_selection(h, grouped, planes, n_p, 1, "outcome top worlds", "top-worlds");
    if (rc) return rc;
    if (k == 0 || k > B200_MAX_TOP_WORLDS)
        return fail(B200_ERR_INVALID_ARGUMENT, "top worlds k = %u: 1 to %u", k, B200_MAX_TOP_WORLDS);
    if (largest != 0 && largest != 1) return fail(B200_ERR_INVALID_ARGUMENT, "top worlds largest = %d: 0 or 1", largest);
    const uint64_t G = reduction_groups(h, grouped).size();
    const uint64_t want = G * n_p * (1ull + 2ull * k) * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "outcome top worlds are %llu bytes, got %llu", (unsigned long long)want,
                    (unsigned long long)bytes);
    TopkParams S{};
    S.planes = h->out_planes;
    S.ld = h->ld_o;
    S.n_p = n_p;
    S.k = k;
    S.largest = largest;
    for (uint32_t j = 0; j < n_p; ++j) S.plane[j] = planes[j];
    const b200_sixdof::GroupTables &t = reduction_tables(h, Rows::outcomes, grouped);
    S.groups = t.stats_dev;
    S.order = t.order_dev;
    const uint64_t tasks = G * n_p;
    h->topk_read_sum = tasks;  // the small-group routes read every task once
    rc = run_world_reduction(h, Rows::outcomes, false, topk_scratch_bytes(S, t.stats), dst, bytes,
                             [&](double *out, void *scratch, int *n) {
                                 S.out = out;
                                 return launch_top_worlds(S, t.stats, t.order, scratch, n, &h->topk_read_sum, h->stream);
                             });
    h->topk_reads = rc == B200_OK ? (double)h->topk_read_sum / (double)tasks : 0.0;
    return rc;
}

int b200_sixdof_outcome_top_worlds(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, uint32_t k, int largest,
                                   void *dst, uint64_t bytes)
{
    return run_top_worlds(h, false, planes, n_p, k, largest, dst, bytes);
}

int b200_sixdof_outcome_group_top_worlds(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, uint32_t k, int largest,
                                         void *dst, uint64_t bytes)
{
    return run_top_worlds(h, true, planes, n_p, k, largest, dst, bytes);
}

double b200_sixdof_top_worlds_reads(const b200_sixdof *h) { return h ? h->topk_reads : 0.0; }

// Midranks of the selected outcome planes within each group (rank_kernels.cu) into the handle's rank planes, then into
// dst: as [n_worlds][n_p] rows, or (corr) as the rank correlation records, the covariance of the rank planes (the
// covariance kernels, unchanged) turned into [n, rho].  The outcome set and groups checked, then the selection, then
// `bytes`, then the handle's status.  The outcome planes are only read.

// The parameters of a rank call over the handle's rank planes (grown to n_p planes)
static int rank_params(b200_sixdof *h, bool grouped, const uint32_t *planes, uint32_t n_p, RankParams &S)
{
    const uint64_t ld = h->ld_o;
    const int rc = grow_device(h, &h->rank_planes, &h->rank_bytes, n_p * ld * 8ull + ld);
    if (rc) return rc;
    const b200_sixdof::GroupTables &t = reduction_tables(h, Rows::outcomes, grouped);
    S = RankParams{};
    S.planes = h->out_planes;
    S.ld = ld;
    S.n_p = n_p;
    for (uint32_t j = 0; j < n_p; ++j) S.plane[j] = planes[j];
    S.groups = t.stats_dev;
    S.order = t.order_dev;
    S.ranks = h->rank_planes;
    S.mask = (uint8_t *)(h->rank_planes + n_p * ld);
    return B200_OK;
}

// The covariance of the rank planes as the state of a handle with one entity
static CovParams rank_cov_params(const b200_sixdof *h, uint32_t n_p)
{
    CovParams C{};
    C.seg[0] = {h->rank_planes, n_p, n_p * h->ld_o};
    C.n_segs = 1;
    C.planes_per_sample = n_p;
    C.n_planes = n_p;
    C.ld = h->ld_o;
    C.n_worlds = h->desc.n_worlds;
    C.n_entities = 1;
    C.n_p = n_p;
    for (uint32_t j = 0; j < n_p; ++j) C.planes[j] = j;
    return C;
}

static int run_ranks(b200_sixdof *h, bool grouped, bool corr, const uint32_t *planes, uint32_t n_p, void *dst,
                     uint64_t bytes)
{
    if (h) {  // it rewrites the rank planes a sharded call fills
        h->sr.active = false;
        rank_shard_free(h->sr.Q);
    }
    int rc = outcome_selection(h, grouped, planes, n_p, corr ? 2 : 1, corr ? "outcome rank correlation" : "outcome ranks");
    if (rc) return rc;
    const uint64_t G = reduction_groups(h, grouped).size(), W = h->desc.n_worlds;
    const uint64_t want = corr ? G * (1ull + (uint64_t)n_p * n_p) * 8ull : W * n_p * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "outcome %s %llu bytes, got %llu", corr ? "rank correlation is" : "ranks are",
                    (unsigned long long)want, (unsigned long long)bytes);
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (bytes == 0) return B200_OK;
    const uint64_t ld = h->ld_o;
    RankParams S;
    if ((rc = rank_params(h, grouped, planes, n_p, S))) return rc;
    const b200_sixdof::GroupTables &t = reduction_tables(h, Rows::outcomes, grouped);
    const uint64_t tasks = G * n_p, rank_scratch = rank_scratch_bytes(S, t.stats, t.order);
    h->rank_read_sum = tasks;  // the small-group routes read every task once
    if (!corr) {
        rc = run_world_reduction(h, Rows::outcomes, false, rank_scratch, dst, bytes, [&](double *out, void *scratch, int *n) {
            cudaError_t e = launch_ranks(S, W, t.stats, t.order, scratch, n, &h->rank_read_sum, h->stream);
            if (e != cudaSuccess) return e;
            *n += 1;
            return launch_soa_to_aos(h->rank_planes, out, W, n_p, ld, h->stream);
        });
    } else {
        // the covariance of the rank planes, its table before the scratch
        CovParams C = rank_cov_params(h, n_p);
        const uint64_t table = G * (1ull + n_p + (uint64_t)n_p * n_p) * 8ull;
        const uint64_t scratch = table + std::max(rank_scratch, cov_scratch_bytes(C, t.cov));
        rc = run_world_reduction(h, Rows::outcomes, false, scratch, dst, bytes, [&](double *out, void *scr, int *n) {
            int a = 0, b = 0, c = 0;
            void *rest = (char *)scr + table;
            cudaError_t e = launch_ranks(S, W, t.stats, t.order, rest, &a, &h->rank_read_sum, h->stream);
            C.out = (double *)scr;
            if (e == cudaSuccess) e = launch_covariance(C, t.cov_dev, t.cov, rest, &b, h->stream);
            if (e == cudaSuccess) e = launch_rank_correlation((const double *)scr, out, G, n_p, &c, h->stream);
            *n = a + b + c;
            return e;
        });
    }
    h->rank_reads = rc == B200_OK ? (double)h->rank_read_sum / (double)tasks : 0.0;
    return rc;
}

int b200_sixdof_outcome_ranks(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes)
{
    return run_ranks(h, false, false, planes, n_p, dst, bytes);
}

int b200_sixdof_outcome_group_ranks(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes)
{
    return run_ranks(h, true, false, planes, n_p, dst, bytes);
}

int b200_sixdof_outcome_rank_correlation(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes)
{
    return run_ranks(h, false, true, planes, n_p, dst, bytes);
}

int b200_sixdof_outcome_group_rank_correlation(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst,
                                               uint64_t bytes)
{
    return run_ranks(h, true, true, planes, n_p, dst, bytes);
}

double b200_sixdof_rank_reads(const b200_sixdof *h) { return h ? h->rank_reads : 0.0; }

// ---- Sobol indices (sobol_kernels.cu) ----

// *ptr grown to need_bytes as grow_device, but a failed allocation is not sticky: it returns B200_ERR_OUT_OF_MEMORY and
// leaves the handle usable (with *ptr freed)
static int grow_device_soft(b200_sixdof *h, double **ptr, uint64_t *have_bytes, uint64_t need_bytes, const char *what)
{
    if (*have_bytes >= need_bytes) return B200_OK;
    if (*ptr) CU(h, cudaFree(*ptr));
    *ptr = nullptr;
    *have_bytes = 0;
    const cudaError_t e = cudaMalloc(ptr, need_bytes);
    if (e == cudaErrorMemoryAllocation) {
        (void)cudaGetLastError();
        *ptr = nullptr;
        return fail(B200_ERR_OUT_OF_MEMORY, "%s: out of device memory for %llu bytes", what, (unsigned long long)need_bytes);
    }
    CU(h, e);
    *have_bytes = need_bytes;
    return B200_OK;
}

// The Sobol records of the selected outcomes (include/b200_sixdof.h b200_sixdof_outcome_sobol): the derived planes into
// the handle's Sobol buffer, their covariance on the sample axis (the covariance kernels, unchanged) at the front of the
// scratch, then the bootstrap and the records.
static int run_sobol(b200_sixdof *h, bool grouped, const uint32_t *planes, uint32_t n_p, uint32_t d, uint32_t n_boot,
                     uint64_t seed, void *dst, uint64_t bytes)
{
    int rc = outcome_selection(h, grouped, planes, n_p, 1, "outcome sobol", "sobol");
    if (rc) return rc;
    if (d < 1 || d > B200_MAX_SOBOL_INPUTS)
        return fail(B200_ERR_INVALID_ARGUMENT, "sobol: %u inputs, 1 to %u", d, B200_MAX_SOBOL_INPUTS);
    const uint32_t q = d + 2;
    const std::vector<uint64_t> sizes = reduction_groups(h, grouped);
    std::vector<uint64_t> samples(sizes.size());
    for (size_t g = 0; g < sizes.size(); ++g) {
        if (sizes[g] % q && grouped)
            return fail(B200_ERR_INVALID_ARGUMENT, "sobol: group %zu has %llu worlds, not a multiple of d + 2 = %u", g,
                        (unsigned long long)sizes[g], q);
        if (sizes[g] % q)
            return fail(B200_ERR_INVALID_ARGUMENT, "sobol: the batch has %llu worlds, not a multiple of d + 2 = %u",
                        (unsigned long long)sizes[g], q);
        samples[g] = sizes[g] / q;
        if (samples[g] >> 32)
            return fail(B200_ERR_INVALID_ARGUMENT, "sobol: group %zu has %llu samples, at most 2^32 - 1", g,
                        (unsigned long long)samples[g]);
    }
    if (n_boot > B200_MAX_SOBOL_RESAMPLES)
        return fail(B200_ERR_INVALID_ARGUMENT, "sobol: %u resamples, at most %u", n_boot, B200_MAX_SOBOL_RESAMPLES);
    const uint64_t G = sizes.size(), W = h->desc.n_worlds, N = W / q;
    const uint64_t want = G * n_p * (3ull + 4ull * d) * 8ull;
    if (bytes != want)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "outcome sobol records are %llu bytes, got %llu", (unsigned long long)want,
                    (unsigned long long)bytes);
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (bytes == 0) return B200_OK;
    if (!dst) return fail(B200_ERR_INVALID_ARGUMENT, "null destination buffer");
    SobolParams S{};
    S.planes = h->out_planes;
    S.ld_o = h->ld_o;
    S.n_p = n_p;
    for (uint32_t j = 0; j < n_p; ++j) S.plane[j] = planes[j];
    S.d = d;
    S.n_samples = N;
    S.ld = round_up(std::max<uint64_t>(N, 1), 128);
    const uint64_t plane_bytes = (uint64_t)n_p * q * S.ld * 8ull, list_bytes = (uint64_t)n_p * S.ld * 4ull;
    if ((rc = grow_device_soft(h, &h->sobol_planes, &h->sobol_bytes, plane_bytes + list_bytes + n_p * S.ld, "sobol")))
        return rc;
    S.sp = h->sobol_planes;
    S.list = (uint32_t *)((char *)h->sobol_planes + plane_bytes);
    S.mask = (uint8_t *)((char *)h->sobol_planes + plane_bytes + list_bytes);
    // the covariance of the derived planes: output k is sample k of a one-entity state of q planes, over the group
    // table of the sample axis that b200_sixdof_set_world_groups would build for groups of N_g worlds
    CovParams C{};
    C.seg[0] = {h->sobol_planes, q, (uint64_t)q * S.ld};
    C.n_segs = 1;
    C.planes_per_sample = q;
    C.n_planes = (uint64_t)n_p * q;
    C.ld = S.ld;
    C.n_worlds = N;
    C.n_entities = 1;
    C.n_p = q;
    for (uint32_t j = 0; j < q; ++j) C.planes[j] = j;
    const std::vector<WorldGroup> table = cov_group_table(samples.data(), G, 1);
    const uint64_t cov_bytes = G * n_p * (1ull + q + (uint64_t)q * q) * 8ull, table_bytes = G * sizeof(WorldGroup);
    const uint64_t front = cov_bytes + round_up(table_bytes, 8);
    const uint64_t scratch = front + std::max(cov_scratch_bytes(C, table), sobol_scratch_bytes(S, G * n_p, n_boot));
    // the staging buffer grown here, so that running out of memory leaves the handle usable
    const uint64_t stage = std::max<uint64_t>(round_up(scratch, 8) + (device_destination(h, dst) ? 0 : bytes), 8);
    if ((rc = grow_device_soft(h, &h->staging, &h->staging_bytes, stage, "sobol"))) return rc;
    return run_world_reduction(h, Rows::outcomes, false, scratch, dst, bytes, [&](double *out, void *scr, int *n) {
        double *cov = (double *)scr;
        WorldGroup *groups = (WorldGroup *)((char *)scr + cov_bytes);
        void *rest = (char *)scr + front;
        cudaError_t e = cudaMemcpyAsync(groups, table.data(), table_bytes, cudaMemcpyHostToDevice, h->stream);
        int a = 0, b = 0, c = 0;
        if (e == cudaSuccess) e = launch_sobol_planes(S, &a, h->stream);
        C.out = cov;
        if (e == cudaSuccess) e = launch_covariance(C, groups, table, rest, &b, h->stream);
        if (e == cudaSuccess) e = launch_sobol_indices(S, cov, groups, G, n_boot, seed, out, rest, &c, h->stream);
        *n = a + b + c;
        return e;
    });
}

int b200_sixdof_outcome_sobol(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, uint32_t d, uint32_t n_boot,
                              uint64_t seed, void *dst, uint64_t bytes)
{
    return run_sobol(h, false, planes, n_p, d, n_boot, seed, dst, bytes);
}

int b200_sixdof_outcome_group_sobol(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, uint32_t d, uint32_t n_boot,
                                    uint64_t seed, void *dst, uint64_t bytes)
{
    return run_sobol(h, true, planes, n_p, d, n_boot, seed, dst, bytes);
}

// ---- world-sharded ranks (rank_kernels.cu: sharded_rank_round) ----

int b200_sixdof_sharded_ranks_begin(b200_sixdof *h, int grouped, const uint32_t *planes, uint32_t n_p, uint32_t rank,
                                    uint32_t n_ranks, uint64_t *max_round_bytes)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (!max_round_bytes) return fail(B200_ERR_INVALID_ARGUMENT, "null max_round_bytes");
    h->sr.active = false;  // a call still pending is discarded, and its scratch freed
    rank_shard_free(h->sr.Q);
    int rc = outcome_selection(h, grouped != 0, planes, n_p, 1, "sharded outcome ranks");
    if (rc) return rc;
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    if (rank >= n_ranks) return fail(B200_ERR_INVALID_ARGUMENT, "rank %u of %u ranks", rank, n_ranks);
    // a window's offsets exchange is n_ranks u32 per place: from here on even one place is not below the round cap
    if ((uint64_t)n_ranks * 4 >= sharded_rank_round_bytes())
        return fail(B200_ERR_INVALID_ARGUMENT, "sharded ranks: %u ranks, at most %llu", n_ranks,
                    (unsigned long long)(sharded_rank_round_bytes() / 4 - 1));
    RankParams S;
    if ((rc = write_outcomes(h)) || (rc = rank_params(h, grouped != 0, planes, n_p, S))) return rc;
    b200_sixdof::ShardedRanks &c = h->sr;
    RankShard &Q = c.Q;
    Q.S = S;
    Q.table = reduction_tables(h, Rows::outcomes, grouped != 0).stats;
    Q.rank = rank;
    Q.n_ranks = n_ranks;
    Q.step = 0;
    Q.level = 0;
    Q.xbytes = Q.xpos = 0;
    Q.slices.clear();
    Q.slice = 0;
    Q.bad_group = ~0ull;
    Q.reads = 0;
    c.grouped = grouped != 0;
    c.gen = rows_generation(h, true);
    c.partial_bytes = 0;
    c.tasks = Q.table.size() * n_p;
    c.ready = false;
    c.active = true;
    *max_round_bytes = sharded_rank_round_bytes();
    return B200_OK;
}

// the checks every round and end make first: a call begun, on the outcome planes it began on
static int sharded_ranks_pending(b200_sixdof *h, const char *what)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    if (!h->sr.active) return fail(B200_ERR_INVALID_ARGUMENT, "sharded ranks %s without a begin", what);
    if (h->sr.gen != rows_generation(h, true)) {
        h->sr.active = false;
        rank_shard_free(h->sr.Q);
        return fail(B200_ERR_INVALID_ARGUMENT, "sharded ranks %s: the handle's outcomes changed since the begin", what);
    }
    if (h->status != B200_OK) return fail(h->status, "handle is in a failed state");
    return B200_OK;
}

int b200_sixdof_sharded_ranks_round(b200_sixdof *h, const void *reduced, uint64_t reduced_bytes, void *partial,
                                    uint64_t partial_cap, uint64_t *partial_bytes)
{
    int rc = sharded_ranks_pending(h, "round");
    if (rc) return rc;
    b200_sixdof::ShardedRanks &c = h->sr;
    if (c.ready) return fail(B200_ERR_INVALID_ARGUMENT, "sharded ranks: the ranks are ready, call the end");
    if (reduced_bytes != c.partial_bytes)
        return fail(B200_ERR_INVALID_ARGUMENT, "sharded ranks: %llu reduced bytes, the last round sent %llu",
                    (unsigned long long)reduced_bytes, (unsigned long long)c.partial_bytes);
    if (reduced_bytes && !reduced) return fail(B200_ERR_INVALID_ARGUMENT, "null reduced words");
    if (!partial_bytes) return fail(B200_ERR_INVALID_ARGUMENT, "null partial_bytes");
    const uint64_t most = sharded_rank_round_bytes();
    if (partial_cap < most || !partial)
        return fail(B200_ERR_INVALID_ARGUMENT, "sharded ranks: a partial of %llu bytes, the begin asked for %llu",
                    (unsigned long long)partial_cap, (unsigned long long)most);
    CU(h, cudaSetDevice(h->device));
    int launches = 0;
    uint64_t out = 0;
    const cudaError_t e = sharded_rank_round(c.Q, reduced, partial, &out, &launches, h->stream);
    h->timings.kernel_launches += (uint64_t)launches;
    if (e == cudaErrorMemoryAllocation) {  // not sticky: the call ends, the handle stays usable
        (void)cudaGetLastError();
        c.active = false;
        rank_shard_free(c.Q);
        return fail(B200_ERR_OUT_OF_MEMORY, "sharded ranks: out of device memory for the call's scratch");
    }
    if (e != cudaSuccess) {
        c.active = false;
        return cuda_fail(h, e, "sharded_rank_round");
    }
    if (c.Q.bad_group != ~0ull) {
        c.active = false;
        rank_shard_free(c.Q);
        const uint64_t g = c.Q.bad_group;
        return fail(B200_ERR_INVALID_ARGUMENT, "sharded ranks: group %llu holds %llu complete worlds over the ranks, above "
                    "the %llu a task can index", (unsigned long long)g, (unsigned long long)c.Q.n_global[g],
                    (unsigned long long)sharded_rank_max_worlds());
    }
    c.partial_bytes = *partial_bytes = out;
    c.ready = out == 0;
    return B200_OK;
}

int b200_sixdof_sharded_ranks_end(b200_sixdof *h, void *ranks_dst, uint64_t ranks_bytes, void *cov_dst,
                                  uint64_t cov_bytes)
{
    int rc = sharded_ranks_pending(h, "end");
    if (rc) return rc;
    b200_sixdof::ShardedRanks &c = h->sr;
    if (!c.ready) return fail(B200_ERR_INVALID_ARGUMENT, "sharded ranks: end before the last round");
    rank_shard_free(c.Q);  // the rank planes hold the result
    const uint32_t n_p = c.Q.S.n_p;
    const uint64_t W = h->desc.n_worlds, G = c.Q.table.size();
    const uint64_t want_r = W * n_p * 8ull, want_c = G * (1ull + n_p + (uint64_t)n_p * n_p) * 8ull;
    if (ranks_dst && ranks_bytes != want_r)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "sharded ranks are %llu bytes, got %llu", (unsigned long long)want_r,
                    (unsigned long long)ranks_bytes);
    if (cov_dst && cov_bytes != want_c)
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "sharded rank covariance is %llu bytes, got %llu",
                    (unsigned long long)want_c, (unsigned long long)cov_bytes);
    if (ranks_dst)
        rc = run_world_reduction(h, Rows::outcomes, false, 0, ranks_dst, ranks_bytes, [&](double *out, void *, int *n) {
            *n = 1;
            return launch_soa_to_aos(h->rank_planes, out, W, n_p, h->ld_o, h->stream);
        });
    if (!rc && cov_dst) {
        const b200_sixdof::GroupTables &t = reduction_tables(h, Rows::outcomes, c.grouped);
        CovParams C = rank_cov_params(h, n_p);
        rc = run_world_reduction(h, Rows::outcomes, false, cov_scratch_bytes(C, t.cov), cov_dst, cov_bytes,
                                 [&](double *out, void *scratch, int *n) {
                                     C.out = out;
                                     return launch_covariance(C, t.cov_dev, t.cov, scratch, n, h->stream);
                                 });
    }
    if (rc) return rc;
    h->rank_reads = c.tasks ? (double)c.Q.reads / (double)c.tasks : 0.0;
    c.active = false;
    return B200_OK;
}

int b200_sixdof_trajectory_reset(b200_sixdof *h)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    h->ticks_done = 0;
    ++h->rows_gen;
    return B200_OK;
}

uint64_t b200_sixdof_tick_count(const b200_sixdof *h) { return h ? h->tick : 0; }

int b200_sixdof_set_stream(b200_sixdof *h, void *cuda_stream, int use_own_stream)
{
    if (!h) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
    CU(h, cudaSetDevice(h->device));
    CU(h, cudaStreamSynchronize(h->stream));
    if (!use_own_stream) {
        if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
        h->stream = (cudaStream_t)cuda_stream;
        h->own_stream = false;
    } else if (!h->own_stream) {
        CU(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        h->own_stream = true;
    }
    return B200_OK;
}

int b200_sixdof_timings(const b200_sixdof *h, b200_timings *out)
{
    if (!h || !out) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
    *out = h->timings;
    return B200_OK;
}

int b200_sixdof_status(const b200_sixdof *h) { return h ? h->status : B200_ERR_INVALID_ARGUMENT; }

void *b200_sixdof_device_plane(b200_sixdof *h, uint64_t id, uint32_t plane)
{
    if (!h) return nullptr;
    Column *c = h->find(id);
    if (!c || c->global || plane >= c->width) return nullptr;
    if (id == B200_ID_INERTIA) h->mass_class_off = true; // the caller may now write masses the handle never sees
    return c->dev + (uint64_t)plane * h->ld;
}

uint64_t b200_sixdof_plane_stride(const b200_sixdof *h) { return h ? h->ld : 0; }

double b200_probe_copy_gbs(int device, uint64_t bytes, int iters)
{
    if (b200_device_count() <= 0) return -1.0;
    if (device >= 0 && cudaSetDevice(device) != cudaSuccess) return -1.0;
    void *a = nullptr, *b = nullptr;
    if (cudaMalloc(&a, bytes) != cudaSuccess || cudaMalloc(&b, bytes) != cudaSuccess) { cudaFree(a); (void)cudaGetLastError(); return -1.0; }
    cudaMemset(a, 1, bytes);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    double best = 0.0;
    for (int i = 0; i < iters + 2; ++i) {
        cudaEventRecord(e0);
        cudaMemcpyAsync(b, a, bytes, cudaMemcpyDeviceToDevice);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        if (i >= 2 && ms > 0) best = std::max(best, 2.0 * bytes / (ms * 1e-3) / 1e9);
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaFree(a); cudaFree(b);
    return best;
}

// The EGM08 term stream the library builds at create (egm08_tables) for a degree-L coefficient pair: host-only, no GPU
// needed — lets a host (and tests/test_host_logic.py, against the oracle's tables) check what the kernel will read.
uint64_t b200_egm08_stream_len(uint32_t max_degree) { return 4ull * (max_degree + 1ull) * (max_degree + 2ull); }

int b200_egm08_stream(uint32_t max_degree, const double *c_bar, const double *s_bar, double *out, uint64_t out_len)
{
    if (!c_bar || !s_bar || !out) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
    if (max_degree > 128) return fail(B200_ERR_INVALID_ARGUMENT, "EGM08 max_degree must be 0..128 (got %u)", max_degree);
    if (out_len != b200_egm08_stream_len(max_degree))
        return fail(B200_ERR_VALUE_SIZE_MISMATCH, "the degree-%u stream holds %llu f64 (got %llu)", max_degree,
                    (unsigned long long)b200_egm08_stream_len(max_degree), (unsigned long long)out_len);
    const std::vector<double> t = egm08_tables((int)max_degree, c_bar, s_bar);
    std::memcpy(out, t.data(), t.size() * sizeof(double));
    return B200_OK;
}

// Self-test of the EXACT mode's shared-divisor divisions against div.rn.f64 (layout_kernels.cu:selftest_div_kernel):
// n_groups groups of four dividends over one divisor; out[0] = results that differ in any bit (must be 0),
// out[1] = groups answered without the __ddiv_rn fallback.
int b200_selftest_shared_divisor(int device, uint64_t seed, uint64_t n_groups, uint64_t *out)
{
    if (!out) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
    if (b200_device_count() <= 0) return B200_ERR_NO_DEVICE;
    if (device >= 0 && cudaSetDevice(device) != cudaSuccess) return cuda_fail(nullptr, cudaGetLastError(), "cudaSetDevice");
    unsigned long long *counts = nullptr, host[2] = {0, 0};
    if (cudaMalloc(&counts, sizeof host) != cudaSuccess) return cuda_fail(nullptr, cudaGetLastError(), "cudaMalloc(selftest)");
    cudaError_t e = cudaMemset(counts, 0, sizeof host);
    if (e == cudaSuccess) e = launch_selftest_div(seed, n_groups, counts, nullptr);
    if (e == cudaSuccess) e = cudaMemcpy(host, counts, sizeof host, cudaMemcpyDeviceToHost);
    cudaFree(counts);
    if (e != cudaSuccess) return cuda_fail(nullptr, e, "shared-divisor self-test");
    out[0] = host[0]; out[1] = host[1];
    return B200_OK;
}

double b200_probe_fp64_gflops(int device, int iters)
{
    if (b200_device_count() <= 0) return -1.0;
    if (device >= 0 && cudaSetDevice(device) != cudaSuccess) return -1.0;
    cudaDeviceProp prop{};
    int dev = 0;
    cudaGetDevice(&dev);
    cudaGetDeviceProperties(&prop, dev);
    const int blocks = prop.multiProcessorCount * 8;
    double *out = nullptr;
    if (cudaMalloc(&out, (size_t)blocks * 256 * 8) != cudaSuccess) return -1.0;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    double best = 0.0;
    for (int i = 0; i < 5; ++i) {
        cudaEventRecord(e0);
        launch_probe_fp64(out, iters, blocks, nullptr);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        if (i >= 1 && ms > 0) best = std::max(best, 2.0 * 8.0 * iters * blocks * 256.0 / (ms * 1e-3) / 1e9);
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaFree(out);
    return best;
}

} // extern "C"
