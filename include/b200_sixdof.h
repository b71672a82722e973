/*
 * b200_sixdof.h — C ABI of the H100-native 6DOF rigid-body integrator.
 *
 * This library replaces, on the six_dof() hot path only, the executor seam of
 * elodin-sys/elodin's nox-py host:
 *
 *   enum WorldExec { Jax, Cranelift }            libs/nox-py/src/exec.rs:53-94
 *   CraneliftExec::invoke_batch(world, n, ..)    libs/nox-py/src/cranelift_exec.rs:129-195
 *   type TickFn = unsafe extern "C" fn(*const *const u8, *mut *mut u8)
 *                                                libs/nox-py/src/cranelift_exec.rs:11
 *   ExecMetadata{arg_ids, ret_ids, arg_slots}    libs/nox-py/src/exec.rs:18-29
 *
 * Everything below is plain C: opaque handle, POD descriptors, raw pointers and
 * sizes.  No C++/torch types cross the boundary; no exceptions cross it either
 * (every entry point returns an int status, 0 = ok, message via b200_last_error()).
 *
 * Data model (mirrors libs/nox-py/src/world.rs:25-29 `Column{buffer, entity_ids}`):
 *   a column is a dense little-endian f64 array [n_worlds][n_entities][width],
 *   row i of a world = i-th spawned entity that owns the component.  The
 *   reference has no world axis (one OS process per Monte-Carlo world,
 *   libs/monte-carlo/src/lib.rs:2083); n_worlds = 1 reproduces its layout
 *   byte for byte.  Columns are addressed by ComponentId = FNV-1a-64(name) with
 *   bit 63 cleared (libs/impeller2/src/types.rs:36-45).
 *
 * On the device every column is stored SoA: `width` planes of
 * n_worlds*n_entities doubles each (body index b = world*n_entities + entity).
 *
 * Threading: a handle is single-thread-affine, like the reference executor
 * ("moved once, never shared", cranelift_exec.rs:31-51).  One handle per GPU.
 */
#ifndef B200_SIXDOF_H
#define B200_SIXDOF_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_SIXDOF_ABI_VERSION 3u

/* ---- status codes (0 = ok).  Names follow libs/nox-py/src/error.rs:7-44 ---- */
enum {
    B200_OK = 0,
    B200_ERR_COMPONENT_NOT_FOUND = 1, /* Error::ComponentNotFound            */
    B200_ERR_VALUE_SIZE_MISMATCH = 2, /* Error::ValueSizeMismatch            */
    B200_ERR_INVALID_ARGUMENT = 3,    /* Error::UnexpectedInput / MissingArg */
    B200_ERR_UNSUPPORTED = 4,         /* effector / integrator not built in  */
    B200_ERR_CUDA = 5,                /* Error::CraneliftBackend(String) analogue: backend failure (sticky per handle) */
    B200_ERR_NO_DEVICE = 6,           /* no CUDA device: there is NO CPU fallback */
    B200_ERR_OUT_OF_MEMORY = 7
};

/* ---- well-known component ids (FNV-1a-64 & ~(1<<63)); SURVEY §8a-7 ---- */
#define B200_ID_WORLD_ACCEL          0x019091805bc057f4ull
#define B200_ID_SIMULATION_TIME_STEP 0x08e7ddbb2cceaab5ull
#define B200_ID_TICK                 0x1e7683ef2ebc7684ull
#define B200_ID_WORLD_VEL            0x4b03b28a841edd5full
#define B200_ID_WORLD_POS            0x5d1c198a8e96e26eull
#define B200_ID_INERTIA              0x5fd14829c04c0f91ull
#define B200_ID_FORCE                0x675ad8afb3eeebe4ull

/* ---- integrators: libs/nox-py/src/integrator/{rk4,semi_implicit}.rs ---- */
enum {
    B200_INTEGRATOR_RK4 = 0,          /* Rk4::compile, rk4.rs:77-125 (incl. the v0-stage behaviour) */
    B200_INTEGRATOR_SEMI_IMPLICIT = 1 /* semi_implicit_euler, semi_implicit.rs:42-62 */
};

/* ---- arithmetic mode ---- */
enum {
    /* literal operation order of libs/nox/src/{spatial,quaternion}.rs, no FMA
     * contraction, IEEE div/sqrt: bit-identical to oracle/sixdof_oracle.c */
    B200_MATH_EXACT = 0,
    /* FMA contraction, hoisted reciprocals (hardware seed + 2 Newton steps), cross-product
     * rotations, R^-1/R cancelled around the mass divide, effectors folded once per launch;
     * agrees with EXACT to <= 1e-12 relative per tick (tests/test_parity_gpu.py states and
     * checks the tolerance).  Documented deviations from the literal arithmetic: the stage-1
     * term `0 * WorldAccel` (rk4.rs:85-104) is not evaluated, so a non-finite WorldAccel input
     * does not poison the step; denormal inputs to 1/x and 1/sqrt(x) flush to zero. */
    B200_MATH_FAST = 1
};

/* ---- trajectory ring contents (b200_sixdof_desc.trajectory_flags) ---- */
enum {
    /* a sample also carries WorldAccel[6] and Force[6] (the stage-4 values the tick leaves in the
     * ECS columns): 25 f64 per body instead of 13, i.e. every column `commit_world_head_unified`
     * (impeller2_server.rs:390-438) would have written for that telemetry tick */
    B200_TRAJ_FULL = 1
};

/* ---- built-in effectors (SURVEY §8a-12, §8a-8).  Evaluated in array order
 * inside every integrator stage on the stage state, accumulating into Force
 * after clear_forces (libs/nox-py/src/six_dof.rs:148-150,195). ---- */
enum {
    /* F.lin += g * m           examples/ball/sim.py:56-58, examples/rocket/main.py:292-294
     * p[0..2] = g */
    B200_EFF_GRAVITY_CONST = 1,
    /* quadratic drag on the stage velocity, examples/ball/sim.py:99-116
     * p[0] = Cd*rho, p[1] = area; column (optional) = wind (width 3), or wind + per-body
     * [Cd*rho, area] (width 5: Monte-Carlo worlds with their own drag parameters);
     * NOTE (reference behaviour): result torque is reset to 0. */
    B200_EFF_DRAG_QUADRATIC = 2,
    /* F.lin += (q @ axis) * thrust      examples/rocket/main.py:429-431
     * p[0..2] = body axis; column (width 1) = thrust per body */
    B200_EFF_THRUST_BODY = 3,
    /* F += q @ wrench (body -> world)   examples/rocket/main.py:407-413 (layout [tau,f])
     *                                   examples/falcon9/sim.py:659-672 (layout [f,tau], flag below)
     * column (width 6) = body-frame wrench per body */
    B200_EFF_WRENCH_BODY = 4,
    /* point-mass gravity + Coriolis + centrifugal in a rotating frame,
     * examples/falcon9/sim.py:350-361 + frames.py:91-109
     * p[0] = mu, p[1..3] = frame angular velocity */
    B200_EFF_GRAVITY_FRAME = 5,
    /* GraphQuery.edge_fold gravity, sequential fold per source body over its
     * out-edges in spawn order (libs/nox-py/src/graph.rs:177-236,
     * python/elodin/__init__.py:454-557); Force := fold(init 0).
     * NEWTON  : examples/three-body/main.py:63-70    p[0] = G
     * SOFTENED: examples/n-body/sim.py:349-361       p[0] = K^2, p[1] = softening */
    B200_EFF_GRAVITY_EDGES_NEWTON = 6,
    B200_EFF_GRAVITY_EDGES_SOFTENED = 7,
    /* F += column, a world-frame wrench [tau(3), f(3)] whose value is computed outside six_dof (a host system,
     * recorded telemetry): `force + SpatialForce(..)` of examples/cube-sat/main.py:516-527,
     * examples/drone/sim.py:99-103.  column (width 6). */
    B200_EFF_WRENCH_WORLD = 8,
    /* Reaction-wheel edge fold, examples/cube-sat/main.py:492-505: Force := fold over the body's K wheels (its
     * out-edges, spawn order) of SpatialForce(torque = q @ tau_k), init SpatialForce().  column (width 3K, K <= 8)
     * = the K wheel torques [tau_1 .. tau_K] of each body, body frame.  Like every edge_fold it OVERWRITES Force. */
    B200_EFF_TORQUE_BODY_FOLD = 9,
    /* point mass + J2 zonal gravity, libs/nox-py/python/elodin/j2.py:5-29 (J2.compute_field), applied as
     * force + SpatialForce(linear=field).  p[0] = mu, p[1] = J2, p[2] = r_ref */
    B200_EFF_GRAVITY_J2 = 10,
    /* spherical-harmonic gravity, libs/nox-py/python/elodin/egm08.py (EGM08.compute_field), applied as
     * force + SpatialForce(linear=field) (examples/cube-sat/main.py:516-527).  p[0] = mu, p[1] = r_ref, p[2] = max_degree L
     * (<= 128); table0 / table1 = the fully normalised C / S coefficients, [(L+1)][(L+1)] f64 row-major (row = degree) —
     * what the reference loads from C_normal.npy / S_normal.npy (a run-time download, so no golden pins it: with C20
     * alone the field equals GRAVITY_J2's to rounding).  Both math modes evaluate it with the oracle's operation order. */
    B200_EFF_GRAVITY_EGM08 = 11
};

#define B200_EFF_FLAG_WRENCH_LINEAR_FIRST 1u /* wrench column is [f(3), tau(3)] (falcon9) */

#define B200_MAX_EFFECTORS 8u

typedef struct b200_effector {
    uint32_t kind;          /* B200_EFF_*                                           */
    uint32_t flags;         /* B200_EFF_FLAG_*                                      */
    double   p[8];          /* constants, meaning per kind                          */
    uint64_t column_id;     /* ComponentId of the per-body input column, 0 = none   */
    uint32_t column_width;  /* f64 per body in that column                          */
    uint32_t reserved;
    uint64_t n_edges;       /* GRAVITY_EDGES_*: directed edges, spawn order         */
    const uint32_t *edge_from; /* entity row index within a world                   */
    const uint32_t *edge_to;
    const uint8_t *entity_mask; /* [n_entities] or NULL: 1 = the effector applies to that entity row.
                                   Mirrors the reference's query join (query.rs:672-710): an @el.map
                                   effector only runs on entities that own every component it reads
                                   (e.g. drag only on bodies with a `wind` component).  Copied at create.
                                   GRAVITY_EDGES_* refuse a mask (B200_ERR_UNSUPPORTED): the fold's
                                   members are the sources of its edges. */
    const double *table0;       /* ABI v3.  GRAVITY_EGM08: C coefficients; copied at create; NULL otherwise  */
    const double *table1;       /*          GRAVITY_EGM08: S coefficients                                     */
    uint64_t table_len;         /*          (L+1)^2                                                            */
} b200_effector;

typedef struct b200_sixdof_desc {
    uint32_t abi_version;      /* B200_SIXDOF_ABI_VERSION                            */
    uint32_t integrator;       /* B200_INTEGRATOR_*                                  */
    uint32_t math_mode;        /* B200_MATH_*                                        */
    uint32_t n_effectors;      /* <= B200_MAX_EFFECTORS                              */
    uint64_t n_entities;       /* bodies per world (rows of every Body column)       */
    uint64_t n_worlds;         /* Monte-Carlo world batch (>= 1)                     */
    double   sim_time_step;    /* SimulationTimeStep component (globals.rs:9); stage dt, rk4.rs:90 */
    double   time_step;        /* six_dof(time_step=..) override of the final combine dt (rk4.rs:83);
                                  NaN = none (use sim_time_step)                      */
    const b200_effector *effectors;
    int32_t  device;           /* CUDA ordinal, -1 = current device                  */
    uint32_t max_fused_ticks;  /* ticks one launch may keep in registers (0/1 = one tick per launch);
                                  only used when no effector couples bodies          */
    uint32_t trajectory_every; /* 0 = off; k = record (pos,vel) every k ticks         */
    uint32_t invoke_chunk_bodies; /* b200_sixdof_invoke_batch splits the world axis into ranges of about
                                  this many bodies so that range k's download overlaps range k+1's
                                  upload and ticks; 0 = default (131072)                */
    uint64_t trajectory_capacity; /* samples the device ring can hold                 */
    uint32_t trajectory_flags; /* B200_TRAJ_*                                        */
    uint32_t reserved0;        /* must be 0                                          */
} b200_sixdof_desc;

typedef struct b200_timings {  /* TickTimings analogue, libs/nox-py/src/profile.rs — of the last
                                  invoke_batch: busy spans of the upload copy engine, the compute stream
                                  and the download copy engine (they overlap) and the call's wall time */
    double h2d_upload_ms;
    double kernel_invoke_ms;
    double d2h_download_ms;
    double invoke_wall_ms;
    uint64_t kernel_launches;  /* launches of this library's kernels since create   */
    uint64_t ticks;            /* ticks integrated since create                      */
} b200_timings;

typedef struct b200_sixdof b200_sixdof; /* opaque */

/* FNV-1a-64(name) & ~(1<<63): ComponentId::new, libs/impeller2/src/types.rs:40-45 */
uint64_t b200_component_id(const char *name);

/* thread-local message of the last failing call (never NULL) */
const char *b200_last_error(void);

/* number of visible CUDA devices, or a negative status; never falls back to CPU */
int b200_device_count(void);

/* Page-locked host memory for column buffers (optional: any host pointer works,
 * pinned ones copy at full PCIe speed and asynchronously). */
void *b200_host_alloc(uint64_t bytes);
/* ... on the NUMA node of `device`'s PCIe root (-1 = current device): mmap + mbind + cudaHostRegister; falls back to
 * b200_host_alloc when the node is unknown.  With 4 GPUs per socket the host memory system, not PCIe, bounds the
 * columns' round trip unless every rank's buffers are node-local. */
void *b200_host_alloc_local(uint64_t bytes, int device);
void b200_host_free(void *p); /* either kind */
/* diagnostics: NUMA node of a GPU's PCIe root / of the first page of a host buffer; -1 = unknown */
int b200_device_numa_node(int device);
int b200_host_node_of(const void *p);

/* Build an executor for one world batch.  Replaces CraneliftExec::new
 * (cranelift_exec.rs:54-127): allocates device-resident SoA columns and the
 * output tables.  All columns start zeroed except inertia-independent defaults;
 * callers upload initial state with b200_sixdof_upload / _invoke_batch. */
int b200_sixdof_create(const b200_sixdof_desc *desc, b200_sixdof **out);
void b200_sixdof_destroy(b200_sixdof *h);

/* ExecMetadata.arg_ids / ret_ids (exec.rs:18-29).  Inputs in first-init order,
 * outputs sorted by ComponentId (BTreeMap order) — SURVEY §8a-7.  Returns the
 * count; writes at most `cap` ids. */
uint32_t b200_sixdof_input_ids(const b200_sixdof *h, uint64_t *ids, uint32_t cap);
uint32_t b200_sixdof_output_ids(const b200_sixdof *h, uint64_t *ids, uint32_t cap);
/* byte length of a column's host buffer (n_worlds*n_entities*width*8; 8 for the
 * two globals), 0 if the handle has no such column */
uint64_t b200_sixdof_column_bytes(const b200_sixdof *h, uint64_t component_id);

/* Host (or device: the copy direction is inferred, cudaMemcpyDefault) AoS column
 * -> device SoA planes, and back.  `bytes` must equal b200_sixdof_column_bytes
 * (else B200_ERR_VALUE_SIZE_MISMATCH, as cranelift_exec.rs:175-177,188-190).
 * Either buffer may be device memory on the handle's GPU, the two globals' 8-byte
 * buffers included.  Both run on the handle's stream, after the work already queued
 * there.  upload returns once a host source has been read (the caller may reuse it);
 * from a device source it returns at once, the copy stream-ordered.  download
 * returns with the data in `dst`. */
int b200_sixdof_upload(b200_sixdof *h, uint64_t component_id, const void *src, uint64_t bytes);
int b200_sixdof_download(b200_sixdof *h, uint64_t component_id, void *dst, uint64_t bytes);

/* Advance the device-resident world n_ticks (asynchronous on the handle's
 * stream).  tick += n_ticks. */
int b200_sixdof_step(b200_sixdof *h, uint64_t n_ticks);
int b200_sixdof_sync(b200_sixdof *h);

/* The reference-shaped call: CraneliftExec::invoke_batch (cranelift_exec.rs:129-195).
 * in_cols[i]  = host buffer of input_ids[i]  (borrowed for the call only)
 * out_cols[j] = host buffer of output_ids[j] (caller-owned, never aliasing an input)
 * Uploads every input column, integrates max(n_ticks,1) ticks on the device,
 * downloads every output column, synchronises.
 * Because the state is device-resident between calls, two entries may be NULL:
 *   in_cols[i]  == NULL: the column is not dirty — the host has not modified it since the previous call
 *                        (World::dirty_components, libs/nox-py/src/world.rs:43,249-252) — the device copy stands;
 *   out_cols[j] == NULL: the caller does not read that column after this batch (e.g. WorldAccel / Force between
 *                        telemetry cycles, pass-through Inertia): it is neither downloaded nor filled.
 * Any buffer may be device memory on the handle's GPU (tick and simulation_time_step included); a call with
 * a device buffer other than the two globals runs on the pipelined world ranges.  Every copy out of an input
 * and into an output is ordered after the work already queued on the handle's stream, and the call returns
 * with every output written. */
int b200_sixdof_invoke_batch(b200_sixdof *h, const uint8_t *const *in_cols,
                             uint8_t *const *out_cols, uint64_t n_ticks);

/* TickFn-shaped shim (cranelift_exec.rs:11): one tick, bound to a thread-local
 * handle.  Returns void like the reference; errors are sticky on the handle. */
int b200_sixdof_bind_tick(b200_sixdof *h);
void b200_sixdof_tick(const uint8_t *const *in_cols, uint8_t **out_cols);

/* Trajectory ring: samples of (world_pos[7], world_vel[6]) — with B200_TRAJ_FULL also
 * (world_accel[6], force[6]) — taken every `trajectory_every` ticks.  Download layout
 * [samples][n_worlds][n_entities][width], width = b200_sixdof_trajectory_width() = 13 | 25.
 * The ring lets a telemetry_rate < simulation_rate run stay device-resident between samples:
 * upload once, step, read the samples back in one transfer. */
uint64_t b200_sixdof_trajectory_len(const b200_sixdof *h);
uint32_t b200_sixdof_trajectory_width(const b200_sixdof *h);
int b200_sixdof_trajectory_download(b200_sixdof *h, void *dst, uint64_t bytes);
int b200_sixdof_trajectory_reset(b200_sixdof *h);

/* ---- retained worlds: the full rows of chosen worlds, gathered on the device, so that an ensemble campaign keeps a
 * few real trajectories (the nominal run, a sample for a spaghetti plot, flagged runs) beside its statistics.
 * worlds[0 .. n) are world indices below n_worlds, in any order, repeats allowed; a null handle, n = 0, a null list or
 * an index >= n_worlds returns B200_ERR_INVALID_ARGUMENT (naming the index), a wrong `bytes`
 * B200_ERR_VALUE_SIZE_MISMATCH.  The list goes to the device once per call.  dst may be host memory or device memory
 * on the handle's GPU (written directly); host rows go through the staging buffer in slices of at most 256 MiB of
 * samples.  Both entries run on the handle's stream, return once dst is filled and count their launches in
 * timings.kernel_launches. ---- */
/* rows of chosen worlds: dst = [trajectory_len][n][n_entities][trajectory_width] f64, the rows of
 * b200_sixdof_trajectory_download for worlds[0..n) in that order.  An empty ring takes bytes = 0 and launches nothing. */
int b200_sixdof_trajectory_download_worlds(b200_sixdof *h, const uint64_t *worlds, uint32_t n, void *dst, uint64_t bytes);
/* the current state of chosen worlds: dst = [n][n_entities][25] f64 (world_pos, world_vel, world_accel, force) */
int b200_sixdof_state_download_worlds(b200_sixdof *h, const uint64_t *worlds, uint32_t n, void *dst, uint64_t bytes);

/* ---- ensemble statistics: the world axis reduced on the device, so that a Monte-Carlo campaign records dispersion
 * over time without moving every world's state to the host.  A group is 5 f64 over the worlds of one sampled value of
 * one entity:  count  = worlds whose value is finite (a double, exact up to 2^53),
 *              mean, m2 = sum (x - mean)^2, min, max  over those finite values only  (std = sqrt(m2 / count));
 * a group with count = 0 holds NaN in the other four.  A non-finite world is therefore never averaged in: a diverged
 * run shows up as a missing count.  Near the top of the f64 range: where m2 exceeds DBL_MAX (and every |x| <= 2^1000)
 * m2 is +inf, never 0 or NaN; mean and m2 may be non-finite only where max|x| or m2 exceeds about 2^990; a finite
 * result always keeps full accuracy.  Partial groups are merged with Chan et al.'s pairwise update in a fixed order (no
 * atomics): the same input gives the same bits on every call, and a sample's bits do not depend on how many other
 * samples are reduced with it.  Both device entries run on the handle's stream, return once dst is filled (like
 * b200_sixdof_trajectory_download), count their launches in timings.kernel_launches, and take host or device dst;
 * `bytes` must match exactly (else B200_ERR_VALUE_SIZE_MISMATCH). ---- */
#define B200_STATS_FIELDS 5u  /* count, mean, m2 = sum (x - mean)^2, min, max  over the finite values of the worlds */
/* the samples now in the trajectory ring, reduced over the world axis:
 * dst = [trajectory_len][n_entities][trajectory_width][5] f64.  An empty ring takes bytes = 0 and launches nothing. */
int b200_sixdof_trajectory_stats(b200_sixdof *h, void *dst, uint64_t bytes);
/* the current device state: world_pos, world_vel, world_accel, force (the 25-component B200_TRAJ_FULL sample layout):
 * dst = [n_entities][25][5] f64 */
int b200_sixdof_state_stats(b200_sixdof *h, void *dst, uint64_t bytes);
/* host-only: merge n_parts tables of n_groups stat groups each ([n_parts][n_groups][5]), left to right in part order,
 * into out[n_groups][5] — the cross-rank step of a world-sharded campaign (ranks exchange their tables over any channel;
 * every rank that merges the same tables in the same order gets the same bits).  Needs no GPU.  Histogram tables
 * (b200_sixdof_trajectory_histograms) need no merge entry: they are integer counts and merge by elementwise addition. */
int b200_stats_merge(const double *parts, uint32_t n_parts, uint64_t n_groups, double *out);

/* ---- ensemble quantiles: per-row percentile envelopes over the worlds, on the device.  For one group (one sampled
 * value of one entity) take the n worlds whose value is finite (NaN and +-inf are dropped, as in the statistics) and
 * order them by IEEE totalOrder (so -0 < +0): x_(0) <= ... <= x_(n-1).  For a level q in [0, 1]:
 *   n == 0         -> NaN
 *   h = (n - 1) * q            one correctly rounded f64 multiply
 *   h >= n - 1     -> x_(n-1)
 *   else i = floor(h), t = h - i, a = x_(i), b = x_(i+1), d = b - a;  t >= 0.5 -> b - d * (1 - t),  else a + d * t
 * with correctly rounded, uncontracted f64 operations in both math modes.  This is numpy's default ("linear")
 * np.quantile(x[np.isfinite(x)], q) operation for operation; the two can differ only in the sign of a zero, where numpy's
 * partition leaves -0 and +0 in arbitrary order.  A result is two order statistics and that lerp, so it is exact and
 * does not depend on the algorithm, the launch shape or the order of atomics.
 * Route: up to 8192 worlds each group is sorted in shared memory (one read of the planes, no scratch); above that, a
 * radix select reads the planes at most 8 times on any data (3 on continuous data).  It needs about 198 KB of device
 * scratch per group and runs the groups in slices of about 1350 (a fixed launch sequence per slice), so the scratch,
 * which lives in the handle's staging buffer, is at most 256 MiB whatever the ring or entity count.  Quantile tables
 * cannot be merged after the fact (unlike b200_stats_merge): a world-sharded campaign reduces them together, in rounds,
 * with b200_sixdof_sharded_quantiles_begin / _round / _end below.
 * Both entries return the handle's sticky status if it has failed; they take 1 .. B200_MAX_QUANTILES levels
 * q[0 .. n_q) (any order, duplicates allowed; NaN or outside [0, 1]: B200_ERR_INVALID_ARGUMENT), run on the handle's
 * stream, return once dst is filled, take host or device dst, count their launches in timings.kernel_launches (1 below
 * 8192 worlds, else 18 per slice) and need `bytes` to match exactly (else B200_ERR_VALUE_SIZE_MISMATCH). ---- */
#define B200_MAX_QUANTILES 16u
/* the ring's samples: dst = [trajectory_len][n_entities][trajectory_width][n_q] f64.  An empty ring takes bytes = 0 and
 * launches nothing. */
int b200_sixdof_trajectory_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes);
/* the current world_pos, world_vel, world_accel, force planes: dst = [n_entities][25][n_q] f64 */
int b200_sixdof_state_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes);
/* reads of the reduced planes the last quantile call (grouped or not) made, averaged over its (world group, plane,
 * entity) triples (1 on the shared-memory routes) */
double b200_sixdof_quantile_reads(const b200_sixdof *h);

/* ---- world-sharded quantiles: the quantile tables above (ring, state or outcomes, grouped or not) of a campaign whose
 * worlds are split over several handles ("ranks", usually one per GPU), exact, over the union of their worlds.  Every
 * group takes the radix select (quantile_kernels.cu); its passes count keys into integer histograms, which add exactly
 * across ranks, and its plan is a function of those counts alone.  So the host drives rounds: each rank sends the u32
 * words of a round (`partial`), the host sums them elementwise over the ranks with one all-reduce (SUM of unsigned 32-bit
 * words, over any channel: NCCL, gloo, MPI, or a test adding arrays), and hands each rank the sums (`reduced`) in its next
 * round call.  Every rank plans from the same sums, so every rank makes the same rounds, with the same sizes, and ends on
 * the same order statistics: the table equals, bit for bit (the sign of a zero included: totalOrder keys), the matching
 * unsharded entry on one handle holding the ranks' worlds in rank order, for any rank count >= 1 and any split.
 *   Rounds.  The groups run in the unsharded entries' slices (the 256 MiB scratch cap) inside the round sequence.  A
 *   slice takes at most 8 rounds: a count round (one u32 per triple of the slice), then at most 7 histogram rounds (per
 *   triple of the slice 2^14 u32 counters and 32 u64 keys, as 64 u32 words), fewer where every rank of a slice is
 *   finished early; a range whose global count is 1 is finished by copying its key (the rank that holds it) into words
 *   the other ranks leave 0.  b200_sixdof_quantile_reads, set by the end, counts per triple the count pass and every
 *   pass with work for it.
 *   Preconditions (a C host checks them itself; sharding.gather_quantiles does): every rank passes the same source,
 *   grouping, levels, entity count, ring length and outcome count, a rank's groups are the global groups cut to its
 *   worlds (the same G on every rank; a group may be empty on a rank), and the global world count is below 2^32.
 *   Between begin and end the handle's rows must not change: a step, upload, invoke_batch, trajectory_reset,
 *   set_channels, set_outcomes or set_world_groups (and for B200_QUANTILE_OUTCOMES a summary begin, start or add, which
 *   the outcome planes are computed from) makes the next round or end fail with B200_ERR_INVALID_ARGUMENT (and discards
 *   the call); any other reduction may run between rounds.  Writes through a b200_sixdof_device_plane pointer are not
 *   seen by the handle: a host that writes planes that way between rounds gets a table of mixed rows.  The call's device scratch is its own, not the
 *   staging buffer: about 66 KB per triple of the largest slice (at most about 90 MiB) plus the table. ---- */
enum { B200_QUANTILE_RING = 0, B200_QUANTILE_STATE = 1, B200_QUANTILE_OUTCOMES = 2 };
/* Checks what the matching quantile entry checks, in the same order (the groups when grouped, the outcomes for
 * B200_QUANTILE_OUTCOMES, the sticky status, the levels), after B200_ERR_INVALID_ARGUMENT for a null handle, a source
 * that is none of the three or a null max_round_bytes; discards a call still pending; fixes the source, grouping and
 * levels of the call and writes its largest round in bytes (0: no triple, the first round ends the call). */
int b200_sixdof_sharded_quantiles_begin(b200_sixdof *h, uint32_t source, int grouped, const double *q, uint32_t n_q,
                                        uint64_t *max_round_bytes);
/* One round: `reduced` = the ranks' elementwise sum of this rank's previous partial (NULL, 0 on the first call), host or
 * device memory; writes the next round's words to `partial` (host or device memory, partial_cap >= begin's
 * max_round_bytes) and their size to *partial_bytes, and returns once they are there (reduced and partial may be the
 * same buffer: the sums are read first); *partial_bytes == 0: the table is ready.  The sums are read on the handle's
 * stream, which is not ordered after other streams: a device `reduced` written by another stream (an NCCL all-reduce)
 * must be complete before the call.  B200_ERR_INVALID_ARGUMENT, with the call left as it was, for reduced_bytes that is
 * not the previous partial_bytes, a too small partial or a round after the last one; and, discarding it, for a round
 * without a begin or after the rows changed. */
int b200_sixdof_sharded_quantiles_round(b200_sixdof *h, const void *reduced, uint64_t reduced_bytes, void *partial,
                                        uint64_t partial_cap, uint64_t *partial_bytes);
/* dst (host or device): exactly the layout and size of the matching unsharded entry (trajectory_ / state_ /
 * outcome_[group_]quantiles; else B200_ERR_VALUE_SIZE_MISMATCH).  B200_ERR_INVALID_ARGUMENT for an end without a begin,
 * before the last round, or after the rows changed.  Ends the call. */
int b200_sixdof_sharded_quantiles_end(b200_sixdof *h, void *dst, uint64_t bytes);

/* ---- ensemble covariance: the joint spread of chosen components over the worlds, on the device.  A selection is
 * planes[0 .. n_p) of the B200_TRAJ_FULL sample layout (world_pos 0-6, world_vel 7-12, world_accel 13-18, force 19-24),
 * 1 <= n_p <= B200_MAX_COV_PLANES, distinct, in the caller's order.  A group is one (sample, entity), and its record is
 * 1 + n_p + n_p^2 f64:
 *   n           the worlds whose n_p selected values are ALL finite (listwise deletion: unlike the statistics, which
 *               count per plane, a world with one NaN / +-inf among the selected values is left out of every entry;
 *               non-finite values in planes that are not selected exclude nothing),
 *   mean[n_p]   over those worlds,
 *   M[n_p][n_p] the co-moments sum (x_a - mean_a)(x_b - mean_b), row-major, M[b][a] the same bits as M[a][b]
 *               (covariance = M / n, numpy's ddof = 0);
 * a group with n = 0 holds NaN after n.  Near the top of the f64 range, as for the statistics: M[a][a] beyond DBL_MAX
 * (every |x_a| <= 2^1000) is +inf, never 0 or NaN; an entry (a, b) may be non-finite only where max|x_a|, max|x_b|,
 * M[a][a] or M[b][b] exceeds about 2^990.  Chunks of worlds are summed shifted by the chunk's first complete world and
 * merged with Chan et al.'s update in a fixed order (no atomics); the chunking depends on (n_worlds, n_entities) alone,
 * so the same input gives the same bits on every call, a sample's bits do not depend on the ring, and an entry (a, b)
 * has the same bits in any selection that holds both planes and has the same complete worlds.  Device scratch (in the
 * handle's staging buffer) stays under 256 MiB: large calls run their groups in slices, which changes no bits.
 * Both entries return the handle's sticky status if it has failed, then B200_ERR_INVALID_ARGUMENT for an empty or too
 * long selection, a duplicate plane or a plane >= the width (b200_sixdof_trajectory_width for the ring, 25 for the
 * state), then B200_ERR_VALUE_SIZE_MISMATCH unless `bytes` matches exactly.  They run on the handle's stream, return once
 * dst (host or device) is filled and count their launches in timings.kernel_launches. ---- */
#define B200_MAX_COV_PLANES 25u
/* the ring's samples: dst = [trajectory_len][n_entities][1 + n_p + n_p^2] f64.  An empty ring takes bytes = 0. */
int b200_sixdof_trajectory_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes);
/* the current world_pos, world_vel, world_accel, force planes: dst = [n_entities][1 + n_p + n_p^2] f64 */
int b200_sixdof_state_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes);
/* host-only: merge n_parts tables of n_groups records each ([n_parts][n_groups][1 + n_p + n_p^2]) left to right, in
 * part order, into out[n_groups][1 + n_p + n_p^2], with the update the kernels use (M[a][b] is read from a <= b).
 * A negative or NaN count is B200_ERR_INVALID_ARGUMENT.  Needs no GPU. */
int b200_covariance_merge(const double *parts, uint32_t n_parts, uint64_t n_groups, uint32_t n_p, double *out);

/* ---- ensemble histograms: per-row bin counts over the worlds, on the device.  A spec is one entity row and one or two
 * axes; an axis is a plane of the B200_TRAJ_FULL sample layout, a range lo < hi and n bins.  Its edges are
 * np.linspace(lo, hi, n + 1)'s: step = (hi - lo) / n, edge_i = i * step + lo (multiply, then add), edge_n = hi.
 * Only finite values are counted in bins, as in the statistics.
 *   1D record, 3 + n f64:  nonfinite (worlds whose value is NaN / +-inf), below (x < lo), above (x > hi), then the
 *     counts of np.histogram(x[np.isfinite(x)], bins=n, range=(lo, hi)), with numpy's own rule, operation for operation
 *     (uncontracted, correctly rounded, in both math modes): keep lo <= x <= hi; f = ((x - lo) / (hi - lo)) * n;
 *     i = trunc(f); i == n -> n - 1; then i - 1 if x < edge_i, and i + 1 if x >= edge_{i+1} and i != n - 1.
 *   2D record, 2 + na * nb f64:  nonfinite (either value non-finite), outside (both finite, at least one out of range),
 *     then the counts of np.histogram2d(x, y, bins=(na, nb), range=((lo_a, hi_a), (lo_b, hi_b))) over the worlds with
 *     both values finite, row-major; per axis searchsorted(edges, v, side='right') - 1, with v == hi in the last bin.
 * Every world is counted once: 1D nonfinite + below + above + sum(counts) = n_worlds, 2D nonfinite + outside +
 * sum(counts) = n_worlds.  Counts are f64, exact below 2^53, and integer sums are exact in any order, so the table does
 * not depend on the launch shape or the order of the device's atomics, and the tables of a world-sharded campaign merge
 * by elementwise addition into exactly the table of the union of their worlds (there is no merge entry: add them).
 * A row's records are the specs' records concatenated in spec order: the ring's dst = [trajectory_len][sum of the record
 * lengths] f64 (an empty ring takes bytes = 0 and launches nothing), the state's dst = [sum of the record lengths].
 * Both entries return B200_ERR_INVALID_ARGUMENT for a null handle, then the handle's sticky status if it has failed,
 * then B200_ERR_INVALID_ARGUMENT for: null specs, n_specs of 0 or above B200_MAX_HISTOGRAMS, n_axes not 1 or 2, a
 * reserved field that is not 0, entity >= n_entities, a plane >= the width (b200_sixdof_trajectory_width for the ring,
 * 25 for the state), a 2D spec with the same plane twice, n = 0, more than B200_MAX_HISTOGRAM_CELLS cells (n for 1D,
 * na * nb for 2D), lo or hi not finite, lo >= hi, hi - lo not finite, step = 0, or edges that are not strictly
 * increasing (a range too narrow for its bins); then B200_ERR_VALUE_SIZE_MISMATCH unless `bytes` matches exactly.  They
 * run on the handle's stream (one memset and one launch), return once dst (host or device) is filled and count their
 * launches in timings.kernel_launches. ---- */
#define B200_MAX_HISTOGRAMS 8u
#define B200_MAX_HISTOGRAM_CELLS 4096u
typedef struct b200_histogram {
    uint64_t entity;     /* entity row within a world                                   */
    uint32_t n_axes;     /* 1 or 2                                                      */
    uint32_t plane[2];   /* B200_TRAJ_FULL layout; plane[1] unused for 1D               */
    uint32_t bins[2];
    uint32_t reserved;   /* must be 0                                                   */
    double   lo[2], hi[2];
} b200_histogram;
int b200_sixdof_trajectory_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                      uint64_t bytes);
int b200_sixdof_state_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst, uint64_t bytes);

/* ---- grouped ensembles: the statistics and histograms above, one table per group of worlds (one sweep point of a
 * campaign).  A group is a contiguous world range: group g holds the worlds [sizes[0] + .. + sizes[g-1], .. + sizes[g]);
 * a host reorders its plan so that every sweep point is contiguous.  Empty groups are allowed.  Group g's record has the
 * same bits as the ungrouped entry on a handle whose n_worlds = sizes[g] holds exactly those worlds (statistics: the
 * chunking of a group depends on its size and n_entities alone; histograms: integer counts, exact in any order); an
 * empty group has count 0 and NaN in its statistics, and zero counts.  The grouped tables put the group axis after the
 * sample axis; with G = 1 and sizes = {n_worlds} they are the ungrouped tables.  Setting groups changes nothing the
 * ungrouped entries return.  The grouped entries check what the ungrouped ones check, in the same order, and return
 * B200_ERR_INVALID_ARGUMENT while no groups are set; they run on the handle's stream, return once dst (host or device)
 * is filled and count their launches in timings.kernel_launches (statistics: one or two per slice of groups and planes,
 * slices keeping the chunk partials in the staging buffer at most 256 MiB; histograms: one memset and one launch).
 * Quantiles: a result is two order statistics and a fixed lerp, so any route gives a group the bits of its own handle.
 * Each group takes the route of its own size: up to 256 worlds (empty groups included) the warp sort, up to 8192 the
 * block sort, above that the radix select.  A call launches once per sort route that has groups, plus 18 launches per
 * slice of the large groups' (group, plane, entity) triples (at most about 1350 triples a slice, whole (group, plane)
 * rows or entity ranges of one row); b200_sixdof_quantile_reads averages the reads over every (group, plane, entity).
 * An empty group gives NaN at every level.  Grouped quantile tables of a world-sharded campaign, with each rank's groups
 * cut to its worlds, are reduced together with b200_sixdof_sharded_quantiles_begin (grouped = 1), as the ungrouped ones.
 * Covariance: group g is chunked as a batch of sizes[g] worlds would be, and an empty group is one chunk of no worlds,
 * with n = 0 and NaN after it.  A call launches one chunk launch, plus a merge launch where a group of the slice has
 * more than one chunk, per slice of groups and samples, slices keeping the chunk partials at most 256 MiB.  Grouped
 * covariance tables of a world-sharded campaign, with each rank's groups cut to its worlds, merge with
 * b200_covariance_merge (a group a rank does not hold has n = 0, the identity of the merge). ---- */
#define B200_MAX_WORLD_GROUPS 1024u
/* sizes[0 .. n_groups): consecutive world counts, each >= 0, summing to n_worlds; n_groups = 0 clears the setting.
 * B200_ERR_INVALID_ARGUMENT for a null handle, more than B200_MAX_WORLD_GROUPS groups, null sizes with n_groups > 0 or
 * sizes that do not sum to n_worlds (the setting is then unchanged).  The group table is built and copied to the device
 * here, once per setting. */
int b200_sixdof_set_world_groups(b200_sixdof *h, const uint64_t *sizes, uint32_t n_groups);
/* the current number of groups, 0 = none */
uint32_t b200_sixdof_world_groups(const b200_sixdof *h);
/* the ring's samples: dst = [trajectory_len][G][n_entities][trajectory_width][5] f64 */
int b200_sixdof_trajectory_group_stats(b200_sixdof *h, void *dst, uint64_t bytes);
/* the current state: dst = [G][n_entities][25][5] f64 */
int b200_sixdof_state_group_stats(b200_sixdof *h, void *dst, uint64_t bytes);
/* the ring's samples: dst = [trajectory_len][G][sum of the record lengths] f64 */
int b200_sixdof_trajectory_group_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                            uint64_t bytes);
/* the current state: dst = [G][sum of the record lengths] f64 */
int b200_sixdof_state_group_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                       uint64_t bytes);
/* the ring's samples: dst = [trajectory_len][G][n_entities][trajectory_width][n_q] f64 */
int b200_sixdof_trajectory_group_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes);
/* the current state: dst = [G][n_entities][25][n_q] f64 */
int b200_sixdof_state_group_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes);
/* the ring's samples: dst = [trajectory_len][G][n_entities][1 + n_p + n_p^2] f64 */
int b200_sixdof_trajectory_group_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst,
                                            uint64_t bytes);
/* the current state: dst = [G][n_entities][1 + n_p + n_p^2] f64 */
int b200_sixdof_state_group_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes);

/* ---- run summaries: the time axis reduced on the device, per world, so that a Monte-Carlo campaign keeps each run's
 * extrema and threshold events without moving its trajectory to the host.  A row is one recorded state in the
 * B200_TRAJ_FULL layout (world_pos[7], world_vel[6], world_accel[6], force[6]: planes 0..24) at one tick.
 * Extrema, per (world, entity, plane), 5 f64:
 *   min, max              over the rows whose value is finite (NaN while there is none),
 *   min_tick, max_tick    tick of the row that holds min / max; among equal values the earliest tick wins,
 *   first_nonfinite_tick  tick of the first row whose value is NaN or +-inf;
 * a tick field is -1 where it never applied.
 * Thresholds, per (world, threshold), 26 f64: the tick of the first row where the value of (entity, plane) is strictly
 * below (above = 0) or above (above != 0) `value` (NaN never fires), then the entity's 25 planes at that row; tick -1
 * and NaN planes while it has not fired.  This is a first-time condition, not a crossing: a world that starts beyond
 * the bound fires at its first row.
 * Every comparison is strict and ties go to the smaller tick, so folding the same rows in any grouping or order, or
 * folding a row twice, gives the same bits; no field involves arithmetic.  Ticks have the resolution of the rows folded
 * (telemetry rows, not ticks).  Every entry runs on the handle's stream and leaves the sticky status alone on success;
 * each one called before b200_sixdof_summary_begin fails with B200_ERR_INVALID_ARGUMENT. ---- */
#define B200_EXTREMA_FIELDS 5u   /* min, max, min_tick, max_tick, first_nonfinite_tick */
#define B200_MAX_THRESHOLDS 8u
typedef struct b200_threshold {
    uint64_t entity;  /* entity row within a world (< n_entities)                  */
    uint32_t plane;   /* 0..24 in the B200_TRAJ_FULL row layout, e.g. 6 = world_pos z */
    int32_t  above;   /* 0: fires on value < bound; otherwise on value > bound         */
    double   value;   /* the bound (not NaN)                                           */
} b200_threshold;
/* Start (or start over): extrema != 0 keeps the extrema table; t[0 .. n_thresholds) are copied.  Allocates the device
 * accumulators on first use (extrema: 1000 B per body; thresholds: 208 B per world and threshold) and clears them.
 * B200_ERR_INVALID_ARGUMENT: entity >= n_entities, plane >= 25, a NaN bound, n_thresholds > B200_MAX_THRESHOLDS, or
 * neither extrema nor thresholds. */
int b200_sixdof_summary_begin(b200_sixdof *h, uint32_t extrema, const b200_threshold *t, uint32_t n_thresholds);
/* fold the current device state as one row at the current tick (b200_sixdof_tick_count) */
int b200_sixdof_summary_add_state(b200_sixdof *h);
/* fold the b200_sixdof_trajectory_len samples now in the ring (B200_TRAJ_FULL only, else B200_ERR_INVALID_ARGUMENT);
 * sample k is the row at tick (tick_count - T) + (k + 1) * trajectory_every, T = ticks stepped since the last
 * b200_sixdof_trajectory_reset (or create) by b200_sixdof_step and b200_sixdof_invoke_batch together.  An empty ring
 * launches nothing. */
int b200_sixdof_summary_add_trajectory(b200_sixdof *h);
/* dst = [n_worlds][n_entities][25][5] f64; refused when begin had no extrema */
int b200_sixdof_extrema_download(b200_sixdof *h, void *dst, uint64_t bytes);
/* dst = [n_worlds][n_thresholds][26] f64: tick, then the 25 planes; refused when begin had no thresholds */
int b200_sixdof_thresholds_download(b200_sixdof *h, void *dst, uint64_t bytes);
/* Both downloads take host or device dst, return once it is filled, need `bytes` to match exactly (else
 * B200_ERR_VALUE_SIZE_MISMATCH) and count their launches in timings.kernel_launches, as the statistics entries do. */

/* Run scores, folded by the same two entries in the same launch as the extrema (each plane a fold needs is read once):
 * Moments, per (world, entity, selected plane): over the rows whose value is finite, in the order they are folded,
 *   the first finite value sets K, then for each finite x:  y = x - K;  S1 = S1 + y;  S2 = S2 + y*y;  n = n + 1
 *   (each operation correctly rounded, the product never contracted, in both math modes).  The table record is
 *   (n, mean = K + S1 / n, m2 = S2 - S1 * (S1 / n) clamped at 0), with m2 = +inf where S2 overflowed and NaN mean and
 *   m2 while n = 0.  The bits depend only on the sequence of finite rows folded, so any ring size gives the same table;
 *   unlike the extrema, folding a row twice counts it twice.
 * Dwells, per (world, dwell), 3 f64: rows = the number of rows folded whose value of (entity, plane) is strictly below
 *   (above = 0) or above (above != 0) `value` (NaN never counts), first_tick / last_tick = the smallest / largest tick
 *   of such a row (-1 while none).  first_tick is the tick of a threshold on the same condition; last_tick of an error
 *   norm above a tolerance is the settling time.  Folding a row twice counts it twice. */
#define B200_MOMENT_FIELDS 3u    /* n, mean, m2 */
#define B200_DWELL_FIELDS 3u     /* rows, first_tick, last_tick */
#define B200_MAX_DWELLS 8u
typedef struct b200_summary_spec {
    uint32_t extrema;                     /* != 0: keep the extrema table                                */
    uint32_t n_thresholds;                /* 0 .. B200_MAX_THRESHOLDS                                    */
    const b200_threshold *thresholds;
    uint32_t n_moments;                   /* 0 .. R distinct planes (< R), in table order                */
    uint32_t n_dwells;                    /* 0 .. B200_MAX_DWELLS                                        */
    const uint32_t *moments;
    const b200_threshold *dwells;         /* the condition of a threshold: entity, plane < R, above, value */
} b200_summary_spec;
/* Start (or start over) every run summary of *spec.  b200_sixdof_summary_begin(h, e, t, n) is this entry with no
 * moments and no dwells, with the same launches and bits.  Allocates the moment accumulators (32 B per body and
 * selected plane) and dwell records (24 B per world and dwell) on first use and clears them.
 * B200_ERR_INVALID_ARGUMENT, with the summary started before left in force: a null spec, nothing requested, more than
 * B200_MAX_THRESHOLDS thresholds or B200_MAX_DWELLS dwells, a null list with a count, an entity >= n_entities, a plane
 * >= R, duplicate moment planes, or a NaN bound. */
int b200_sixdof_summary_start(b200_sixdof *h, const b200_summary_spec *spec);
/* dst = [n_worlds][n_entities][n_moments][3] f64 (n, mean, m2); refused when the summary has no moments */
int b200_sixdof_moments_download(b200_sixdof *h, void *dst, uint64_t bytes);
/* dst = [n_worlds][n_dwells][3] f64 (rows, first_tick, last_tick); refused when the summary has no dwells */
int b200_sixdof_dwells_download(b200_sixdof *h, void *dst, uint64_t bytes);
/* Both take host or device dst and count their launches like the extrema and threshold downloads. */

/* ---- derived channels: per-body quantities computed on the device from a body's 25-plane row (B200_TRAJ_FULL layout)
 * and reduced like the state components.  With n_c channels set, channel k is plane 25 + k of the row every ensemble
 * entry reduces, ring and state alike, so a row is R = 25 + n_c planes wide in: the statistics and quantiles (plain and
 * grouped: dst [..][n_entities][R][..]), covariance selections and histogram specs (a plane < R), and the run summaries
 * (threshold planes < R; extrema dst = [n_worlds][n_entities][R][5]).  A threshold record stays tick + the 25 raw planes.
 * trajectory_download, trajectory_width, the *_download_worlds entries, the NCCL all-gather and both merge entries do not
 * change.  With n_c = 0 (the default) every entry is what it is without this section; with channels set, planes 0..24 of
 * every table keep their bits.
 *   B200_CHANNEL_NORM: n in 1..3 distinct planes p[0..n) (each < 25), offsets c[0..n), r0:
 *     d_i = x[p_i] - c_i;  s = d_0*d_0;  s = s + d_1*d_1;  s = s + d_2*d_2  (terms i < n, in that order);  sqrt(s) - r0
 *     every operation correctly rounded and uncontracted in both math modes: numpy's bits for the same expression.
 *     Squares that overflow give +inf.  Speed: planes (10, 11, 12); distance from a point: (4, 5, 6) with c = the point;
 *     altitude over a sphere: r0 = its radius.
 *   B200_CHANNEL_AXIS_ANGLE: the angle in [0, pi] between the body-frame axis c (finite, not zero) rotated into the world
 *     frame and a world direction v: the fixed vector d (n = 0, finite, not zero), or planes plane[0] .. plane[0] + 2
 *     of the row (n = 3; plane[0] = 10 gives the velocity: inertial angle of attack / flight-path angle):
 *       u = qrot(q, c)  (q = planes 0..3; the EXACT rotation of the tick, q * [c, 0] * q.inverse(), in both math modes)
 *       x = u cross v;  s = sqrt((x.x*x.x + x.y*x.y) + x.z*x.z);  t = (u.x*v.x + u.y*v.y) + u.z*v.z;  atan2(s, t)
 *     correctly rounded and uncontracted up to s and t; atan2 is CUDA's double atan2 (2 ulp maximum error, CUDA Math API).
 *     Neither q nor v needs to be normalised.  A zero v (a body at rest) gives atan2(0, 0) = 0.
 * NaN or +-inf inputs give non-finite values, which the reductions drop like any other non-finite value.  Every entry
 * that reads a channel plane recomputes the channels first (one launch on the handle's stream, counted in
 * timings.kernel_launches): statistics, quantiles and extrema whenever n_c > 0; covariance, histograms and thresholds
 * only when their selection names a channel plane. ---- */
#define B200_MAX_CHANNELS 8u
enum { B200_CHANNEL_NORM = 1, B200_CHANNEL_AXIS_ANGLE = 2 };
typedef struct b200_channel {
    uint32_t kind;       /* B200_CHANNEL_*                                                              */
    uint32_t n;          /* NORM: 1..3 planes; AXIS_ANGLE: 0 = fixed direction d, 3 = planes plane[0] .. +2 */
    uint32_t plane[3];   /* planes of the 25-plane row                                                  */
    uint32_t reserved;   /* must be 0                                                                   */
    double   c[3];       /* NORM: offsets; AXIS_ANGLE: body axis                                        */
    double   d[3];       /* AXIS_ANGLE with n = 0: world direction                                      */
    double   r0;         /* NORM: subtracted from the norm                                              */
} b200_channel;
/* c[0 .. n) replaces the channel set; n = 0 clears it.  B200_ERR_INVALID_ARGUMENT, with the setting unchanged, for: a
 * null handle, n > B200_MAX_CHANNELS, null c with n > 0, an unknown kind, a bad n, a plane >= 25, duplicate NORM planes,
 * an AXIS_ANGLE plane triple past plane 24, a non-zero reserved field, a non-finite constant, a zero axis or fixed
 * direction, a 13-wide ring (a handle without a ring is allowed), or a handle on which b200_sixdof_summary_begin was
 * called (it fixes the row width of its accumulators).  Allocates capacity * n * ld f64 for the ring's channels and
 * n * ld for the state's. */
int b200_sixdof_set_channels(b200_sixdof *h, const b200_channel *c, uint32_t n);
/* the number of channels set (0 for a null handle) */
uint32_t b200_sixdof_channels(const b200_sixdof *h);
/* the channels of the ring's samples: dst = [trajectory_len][n_worlds][n_entities][n_c] f64 (host or device) */
int b200_sixdof_trajectory_channels(b200_sixdof *h, void *dst, uint64_t bytes);
/* the channels of the current state: dst = [n_worlds][n_entities][n_c] f64 (host or device) */
int b200_sixdof_state_channels(b200_sixdof *h, void *dst, uint64_t bytes);

/* ---- outcomes: one f64 per world, taken from the run summaries, a device column or host values, and reduced over the
 * worlds by the ensemble reductions above.  This joins the two families: the apogee percentiles per sweep point, the
 * impact-point covariance, the probability that a threshold fired or a settling-time histogram, without a per-world
 * table reaching the host.
 *   kind       field                                       value of world w
 *   EXTREMA    0..4: min, max, min_tick, max_tick,         the extrema record of (w, entity, plane `index` < R)
 *              first_nonfinite_tick
 *   THRESHOLD  0: tick; 1 + p: plane p (0..24) of the row  threshold `index`'s record of w
 *   MOMENT     0..3: count, mean, std, rms                 moment slot `index` (the spec's order) of (w, entity)
 *   DWELL      0..2: rows, first_tick, last_tick           dwell `index`'s record of w
 *   COLUMN     a plane of the column (< its width)         the column's current device value for (w, entity): a
 *                                                          dispersed input (inertia plane 6 = mass) or the final state
 *   VALUES     0                                           values[w], copied by set_outcomes
 * Value rules: a tick field that holds -1 ("never") is NaN, so the reductions, which drop non-finite values, leave out
 * the worlds where the event never happened (the count of a threshold's tick is the number of worlds that fired, and
 * count / n_worlds the event probability; a histogram counts them in `nonfinite`).  Every other field keeps its bits,
 * except the moments: count, mean and m2 are those of b200_sixdof_moments_download, then std = sqrt(m2 / n) and
 * rms = sqrt(mean * mean + m2 / n), each operation correctly rounded (numpy's bits for the same expression).
 * Every outcome entry first writes the outcome planes, P planes of n_worlds values, with one launch on the handle's
 * stream (counted in timings.kernel_launches; never cached: the summaries and columns change under it), then runs the
 * reduction on them as on a state of one entity: the tables have the layout and the bits of the state_* entries of a
 * handle with n_entities = 1 whose first P state planes hold the outcome values (E = 1 below).  Grouped entries use the
 * groups of b200_sixdof_set_world_groups.  Every entry checks the outcome set against the summary in force (a later
 * summary_start can drop what an outcome names) and refuses it, naming the outcome, with B200_ERR_INVALID_ARGUMENT, as
 * it refuses a handle without outcomes; then it checks what the state_* entry checks, in the same order. ---- */
#define B200_MAX_OUTCOMES 25u   /* = B200_MAX_COV_PLANES: one covariance call takes every outcome */
enum { B200_OUTCOME_EXTREMA = 1, B200_OUTCOME_THRESHOLD = 2, B200_OUTCOME_MOMENT = 3,
       B200_OUTCOME_DWELL = 4, B200_OUTCOME_COLUMN = 5, B200_OUTCOME_VALUES = 6 };
typedef struct b200_outcome {
    uint32_t kind;        /* B200_OUTCOME_*                                                  */
    uint32_t field;       /* see the table above                                             */
    uint32_t index;       /* EXTREMA: plane < R; THRESHOLD / DWELL: which one; MOMENT: slot  */
    uint32_t reserved;    /* must be 0                                                       */
    uint64_t entity;      /* EXTREMA, MOMENT, COLUMN: entity row (< n_entities); else 0      */
    uint64_t column;      /* COLUMN: component id; else 0                                    */
    const double *values; /* VALUES: n_worlds f64, copied by set_outcomes; else NULL         */
} b200_outcome;
/* o[0 .. n) replaces the outcome set; n = 0 clears it.  B200_ERR_INVALID_ARGUMENT, with the previous set left in force,
 * for: a null handle, n > B200_MAX_OUTCOMES, null o with n > 0, an unknown kind, a bad field, index or entity, a
 * non-zero reserved field, entity or column set where the kind takes none, a summary the summary in force does not have
 * (no extrema, a threshold, dwell or moment slot past its count, an extrema plane >= R), a global column (tick, time
 * step), a column plane >= its width, or null values; B200_ERR_COMPONENT_NOT_FOUND for an unknown column id.  Allocates
 * P * ld_o f64, ld_o = n_worlds rounded up to 128. */
int b200_sixdof_set_outcomes(b200_sixdof *h, const b200_outcome *o, uint32_t n);
/* the number of outcomes set (0 for a null handle) */
uint32_t b200_sixdof_outcomes(const b200_sixdof *h);
/* dst = [n_worlds][P] f64: the outcome values themselves (host or device; for small campaigns and tests) */
int b200_sixdof_outcome_values(b200_sixdof *h, void *dst, uint64_t bytes);
/* dst = [P][5] f64, the state statistics' fields */
int b200_sixdof_outcome_stats(b200_sixdof *h, void *dst, uint64_t bytes);
/* dst = [G][P][5] f64 */
int b200_sixdof_outcome_group_stats(b200_sixdof *h, void *dst, uint64_t bytes);
/* dst = [P][n_q] f64 */
int b200_sixdof_outcome_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes);
/* dst = [G][P][n_q] f64 */
int b200_sixdof_outcome_group_quantiles(b200_sixdof *h, const double *q, uint32_t n_q, void *dst, uint64_t bytes);
/* planes < P: dst = [1 + n_p + n_p^2] f64 */
int b200_sixdof_outcome_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes);
/* dst = [G][1 + n_p + n_p^2] f64 */
int b200_sixdof_outcome_group_covariance(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst,
                                         uint64_t bytes);
/* spec.entity = 0, planes < P: dst = [sum of the record lengths] f64 */
int b200_sixdof_outcome_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                   uint64_t bytes);
/* dst = [G][sum of the record lengths] f64 */
int b200_sixdof_outcome_group_histograms(b200_sixdof *h, const b200_histogram *specs, uint32_t n_specs, void *dst,
                                         uint64_t bytes);

/* ---- worst worlds: the k worlds with the largest or smallest value of each selected outcome, per group of worlds,
 * found on the device; their world indices feed retained rows (World.build(..., retain=)) and per-run databases.
 *   Contract  for a task (group g, selected outcome p) the candidates are the worlds w of the group whose outcome value
 *             x_w is finite (NaN and +-inf are dropped, as by every reduction: a tick that never happened is never a
 *             worst run; to find diverged worlds, ask a threshold's tick with largest = 0, the earliest firing);
 *             count = the number of candidates.
 *   Order     the IEEE totalOrder key of the quantile entries (-0 < +0), ascending for largest = 0 and descending for
 *             largest = 1; ties are always broken by ascending world index.  The record holds the first min(k, count)
 *             candidates in that order: a function of the data alone, whatever the route, launch shape or slicing.
 *             numpy: u = x.view(uint64), key = where(u >> 63, ~u, u | 1 << 63), complemented for largest, then
 *             np.lexsort((world, key))[:k] over the finite worlds.
 *   Record    per task 1 + 2k f64: [count, value_0 .. value_{k-1}, world_0 .. world_{k-1}]; values keep their bits,
 *             worlds are the handle's world indices (not indices within the group), exact as f64 below 2^53; slots past
 *             count hold NaN and -1.
 *   Bound     groups of at most 8192 worlds are sorted in shared memory after one read of the planes.  Larger ones
 *             take a radix select of the composite key (value key, world index) with a fixed launch sequence: a count
 *             pass, at most 8 histogram passes of 2^14 bins (5 over the value keys, 3 more over the world indices of
 *             one value key tied more than 8192 times) and one gather: at most 10 reads of the planes on any data, 3 on
 *             continuous data.  b200_sixdof_top_worlds_reads reports the reads of the last call, averaged over its
 *             tasks.
 *   Memory    device scratch of at most 256 MiB (the large tasks run in slices), in the staging buffer; a host
 *             destination takes the table through the staging buffer after the scratch.
 * Each entry checks, in this order: what every outcome entry checks (the outcome set, naming a refused outcome; the
 * groups for the grouped entry); null planes, n_p of 0 or more than P, a plane >= P or listed twice; k of 0 or more
 * than B200_MAX_TOP_WORLDS; largest not 0 or 1 (all B200_ERR_INVALID_ARGUMENT); then the byte count
 * (B200_ERR_VALUE_SIZE_MISMATCH) and the sticky status.  Like every outcome entry it first writes the outcome planes
 * and is never cached. ---- */
#define B200_MAX_TOP_WORLDS 1024u
/* dst = [n_p][1 + 2k] f64 (host or device) */
int b200_sixdof_outcome_top_worlds(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, uint32_t k, int largest,
                                   void *dst, uint64_t bytes);
/* dst = [G][n_p][1 + 2k] f64, groups of b200_sixdof_set_world_groups */
int b200_sixdof_outcome_group_top_worlds(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, uint32_t k, int largest,
                                         void *dst, uint64_t bytes);
/* average plane reads per task of the last top-worlds call (0 for a null handle or before any call) */
double b200_sixdof_top_worlds_reads(const b200_sixdof *h);

/* ---- rank correlation: midranks of chosen outcomes within each group of worlds, and the Spearman correlation of
 * those ranks, computed on the device; with partial rank correlation (Exec.outcome_sensitivity) the measure of how much
 * each dispersed input drives an outcome, robust to ties, non-linearity and single huge values.
 *   Task      (group g, selected outcome j) over a selection of n_p distinct outcome planes; the ungrouped entries
 *             treat all worlds as one group.
 *   Complete  the worlds of group g whose n_p selected values are all finite (listwise deletion, as for the
 *             covariance); n_g = their count.
 *   Midrank   of a complete world w in plane j: less + (eq + 1) / 2, less = the complete worlds of the group with a
 *             smaller value, eq = those with an equal value, w included (scipy.stats.rankdata(x, method="average")
 *             over the complete worlds).  Values compare numerically: -0 and +0 are one value (unlike the totalOrder
 *             key of the quantile and top-worlds entries).  Every midrank is a half-integer, exact in f64; a world
 *             that is not complete gets NaN.  Nothing breaks ties, so the ranks are a function of the data alone,
 *             whatever the route, launch shape or slicing.
 *   Rho       the covariance record of the rank planes (the outcome covariance kernels, unchanged) turned into
 *             rho[a][b] = M[a][b] / sqrt(M[a][a] * M[b][b]), each operation correctly rounded (numpy's bits for the
 *             same expression); exactly 1 on the diagonal of a plane that varies; NaN in the row and column of a plane
 *             that is constant over the complete worlds (M[a][a] = 0, as scipy.stats.spearmanr), and everywhere when
 *             n < 2.
 *   Record    per group 1 + n_p^2 f64: [n, rho[n_p][n_p] row-major].
 *   Bound     the selected planes are read once per call for completeness (a byte per world in the handle's rank
 *             buffer).  Groups of at most 8192 worlds are then sorted in shared memory after one read.  Larger ones
 *             take an MSD bucket pass over the value keys: a count pass, at most 5 histogram levels of 2^14 bins (a bin
 *             one key wide is one tie run, ranked with no sort; a bin of at most 8192 worlds is a bucket, sorted in
 *             shared memory; a larger one refines at the next level) and one scatter: at most 7 reads of a task's plane
 *             on any data, 3 where the first level leaves no bin above 8192 worlds (values of one sign over a few
 *             binades), plus one read of the bucket area.  b200_sixdof_rank_reads reports the reads of the last call,
 *             averaged over its tasks (the completeness read not counted).
 *   Memory    the rank planes, n_p * ld_o f64 and ld_o bytes, are allocated by the first rank call (grown by a later
 *             one with more planes) and freed by set_outcomes and destroy: a handle that never asks for ranks
 *             allocates nothing more.  The outcome planes are only read.  Device scratch (in the staging buffer) of
 *             about 42 bytes per world of a large group's task, at most 256 MiB (the large tasks run in slices) unless
 *             one task alone needs more.
 * Each entry checks, in this order: what every outcome entry checks (the outcome set, naming a refused outcome; the
 * groups for the grouped entries); null planes, n_p of 0 (ranks) or below 2 (correlation), n_p above P, a plane >= P
 * or listed twice (all B200_ERR_INVALID_ARGUMENT); then the byte count (B200_ERR_VALUE_SIZE_MISMATCH) and the sticky
 * status.  Like every outcome entry it first writes the outcome planes of the summaries and columns (never the VALUES
 * planes) and is never cached; it runs on the handle's stream, returns once dst (host or device) is filled and counts
 * its launches in timings.kernel_launches. ---- */
/* dst = [n_worlds][n_p] f64 midranks (host or device; for small campaigns and tests, like outcome_values) */
int b200_sixdof_outcome_ranks(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes);
/* dst = [n_worlds][n_p] f64 midranks within each group of b200_sixdof_set_world_groups */
int b200_sixdof_outcome_group_ranks(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes);
/* dst = [1 + n_p^2] f64 */
int b200_sixdof_outcome_rank_correlation(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst, uint64_t bytes);
/* dst = [G][1 + n_p^2] f64 */
int b200_sixdof_outcome_group_rank_correlation(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, void *dst,
                                               uint64_t bytes);
/* average plane reads per task of the last rank call (0 for a null handle or before any call) */
double b200_sixdof_rank_reads(const b200_sixdof *h);

/* ---- variance-based sensitivity: first-order and total Sobol indices of chosen outcomes of a Saltelli campaign
 * (monte_carlo.saltelli), with bootstrap spreads, computed on the device.  Unlike rank correlation they see
 * non-monotone effects and interactions: S1_i is the share of an output's variance input i explains alone, ST_i that
 * share with every interaction it takes part in.
 *   Layout    sample j of a group is its worlds [j (d + 2), (j + 1) (d + 2)) in order: [A_j, AB_j^(1) .. AB_j^(d), B_j]
 *             (AB^(i) = A with input i taken from B; SALib's layout without second-order rows).  Every group's world
 *             count (n_worlds, ungrouped) must be a multiple of d + 2; N_g = its samples.
 *   Task      (group g, selected outcome y).  Sample j is complete for y when its d + 2 values of y are finite and
 *             every difference below is finite; listwise deletion is per output, so each output has its own n.
 *   Planes    a complete sample gives a = f(A_j), b = f(B_j), D_i = f(AB_j^(i)) - f(A_j) (correctly rounded); an
 *             incomplete one NaN in all d + 2.  The point record comes from the covariance record [n, m[d+2],
 *             M[d+2][d+2]] of the planes (a, b, D_1 .. D_d) over the task's samples: the outcome covariance kernels,
 *             chunking and merge on the group table of the sample axis (sizes N_g), so it equals the covariance of a
 *             handle whose worlds are the samples.  With each operation correctly rounded, in this order:
 *               V    = (M_aa + M_bb) / (2n) + ((m_a - m_b) * (m_a - m_b)) * 0.25     np.var(np.r_[fA, fB])
 *               EbD  = M_bDi / n + m_b * m_Di                                      mean(fB (fABi - fA)), Saltelli 2010
 *               EDD  = M_DiDi / n + m_Di * m_Di                                    mean((fA - fABi)^2), Jansen
 *               S1_i = EbD / V;  ST_i = EDD / (2 V)
 *             V is NaN where n < 2; S1 and ST are NaN where n < 2 or V is not > 0 (a constant output).
 *   Bootstrap n_boot resamples (0: none, at most B200_MAX_SOBOL_RESAMPLES).  Draw t in [0, n) of resample r takes
 *             complete sample c[umulhi64(x, n)], c = the task's complete samples in sample order, x = mix(seed +
 *             0x9E3779B97F4A7C15 (r 2^32 + t + 1)) mod 2^64, mix = SplitMix64's output function (z ^= z >> 30;
 *             z *= 0xBF58476D1CE4E5B9; z ^= z >> 27; z *= 0x94D049BB133111EB; z ^= z >> 31).  The stream depends on
 *             neither the group nor the output.  With the draws shifted by the point record's means (a' = a - m_a, ..),
 *             sums s_a, s_aa, s_b, s_bb and per input s_D, s_DD, s_bD, and e_x = s_x / n:
 *               V(r)   = ((s_aa/n - e_a e_a) + (s_bb/n - e_b e_b)) * 0.5 + dm * dm * 0.25,  dm = (m_a + e_a) - (m_b + e_b)
 *               EbD(r) = s_bD/n + m_b e_D + m_D e_b + m_b m_D;   EDD(r) = s_DD/n + 2 m_D e_D + m_D m_D
 *             S1(r) and ST(r) as above, NaN where n < 2 or V(r) is not > 0.  The record carries the sample standard
 *             deviation (ddof 1) of the finite S1(r) and ST(r) per input (NaN below 2) and the count of resamples with
 *             V(r) > 0.  The summation order is fixed (no floating-point atomics): the same inputs give the same bits on
 *             every call, stream and destination.
 *   Record    per (group, output) 3 + 4d f64: [n, V, n_boot_ok, S1[d], ST[d], S1_sd[d], ST_sd[d]].
 *   Memory    the derived planes, lists and completeness bytes, n_p ((d + 2) 8 + 5) ld bytes (ld = the sample count
 *             rounded up to 128), are allocated by the first Sobol call (grown by a later, larger one) and freed by
 *             set_outcomes and destroy; they are not the rank planes.  Device scratch (in the staging buffer): the
 *             covariance table, the group table of the samples, and the covariance's or the bootstrap's scratch (at most
 *             256 MiB; the bootstrap runs its tasks in slices, which changes no bits).  A failed allocation returns
 *             B200_ERR_OUT_OF_MEMORY and leaves the handle usable.  The outcome planes are only read.
 * Each entry checks, in this order: what every outcome entry checks (the outcome set; the groups for the grouped
 * entry); null planes, n_p of 0 or above P, a plane >= P or listed twice; d of 0 or above B200_MAX_SOBOL_INPUTS; a world
 * or group count that d + 2 does not divide, or a group of 2^32 samples or more; n_boot above B200_MAX_SOBOL_RESAMPLES
 * (all B200_ERR_INVALID_ARGUMENT); then the byte count (B200_ERR_VALUE_SIZE_MISMATCH) and the sticky status.  Like
 * every outcome entry it first writes the outcome planes of the summaries and columns, runs on the handle's stream,
 * returns once dst (host or device) is filled and counts its launches in timings.kernel_launches. ---- */
#define B200_MAX_SOBOL_INPUTS 23u         /* d + 2 derived planes fit one covariance selection */
#define B200_MAX_SOBOL_RESAMPLES 10000u
/* dst = [n_p][3 + 4d] f64 */
int b200_sixdof_outcome_sobol(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, uint32_t d, uint32_t n_boot,
                              uint64_t seed, void *dst, uint64_t bytes);
/* dst = [G][n_p][3 + 4d] f64, per group of b200_sixdof_set_world_groups */
int b200_sixdof_outcome_group_sobol(b200_sixdof *h, const uint32_t *planes, uint32_t n_p, uint32_t d, uint32_t n_boot,
                                    uint64_t seed, void *dst, uint64_t bytes);

/* ---- world-sharded ranks: the midranks above (grouped or not) of a campaign whose worlds are split over several
 * handles ("ranks"), over the union of their worlds, and the covariance record of each rank's rank planes.  A midrank is
 * not a function of the ranks' local midranks, so the ranks exchange what the bucket pass counts, in rounds with the
 * protocol of the sharded quantiles: each rank sends the u32 words of a round (`partial`), the host sums them
 * elementwise over the ranks (SUM of unsigned 32-bit words, over any channel) and hands each rank the sums (`reduced`)
 * in its next round call.  Afterwards the rank planes of every rank hold the campaign midranks of its own worlds: bit
 * for bit the rows of b200_sixdof_outcome_[group_]ranks on one handle holding every rank's worlds in rank order, for any
 * rank count >= 1 and any split (empty ranks and empty groups included).  The rank correlation of the campaign is then
 * the rank correlation (b200_sixdof_outcome_rank_correlation's formula) of the covariance records of the ranks merged in
 * rank order with b200_covariance_merge: with one rank the unsharded record's bits.
 *   Exchanges.  Every (group, plane) task whose group holds a complete world on some rank takes the MSD bucket pass
 *   (the shared-memory routes would see only local worlds), with an exchange before each step that needs the other
 *   ranks' counts or keys:
 *     sizes    once per call: every group's complete worlds and worlds, rank-slotted (G * n_ranks * 2 u32: rank r
 *              writes slots (g * n_ranks + r) * 2 + {0, 1}, the others leave them 0), so every rank knows each group's
 *              global count and every rank's share.  The tasks are cut into slices from these alike on every rank.
 *     hist     at most 5 per slice: each task's counts of its ranges' 2^14 bins at one level (2^14 u32 per range).  Plan 0
 *              starts from the whole key range (min and max do not add), so the levels are at shifts 50, 36, 22, 8 and
 *              0 and every bin is one key wide after at most 5.  A bin one key wide, or of one world over every rank, is
 *              a tie run ranked base + (count + 1) / 2 with no further exchange; one of at most 8192 worlds is a bucket;
 *              a larger one refines at the next level.  A task of at most 8192 complete worlds is one bucket at once.
 *              After the last level each rank puts its bucket worlds and their keys in a list of its own (the scatter,
 *              the last read of the plane).
 *     windows  the slice's buckets, in windows of their first key's place in the slice's key words: a window holds
 *              W = max(1, min(4,186,111, floor(2^23 / n_ranks) - 1)) places, so both of its exchanges stay below
 *              32 MiB (n_ranks < 2^23, so even a window of one place does):
 *       offsets  each bucket's count on each rank, rank-slotted (W * n_ranks u32, at the bucket's first place).
 *       keys     every key of the window's buckets as a u64 (two u32 words, W + 8192 at most), each rank writing its
 *                own at the bucket's place plus its offset and leaving the other words 0.  Each rank then sorts the
 *                window's buckets that hold its worlds in shared memory and writes its worlds' midranks from two
 *                binary searches of the sorted keys; world indices never travel.
 *   So one sizes exchange per call, then per slice at most 5 histogram exchanges and two per window of its keys (one
 *   window unless the slice's buckets hold more than W worlds), fewer where the summed counts show no work.  The
 *   sizes exchange is G * n_ranks * 8 bytes and a histogram exchange 64 KiB per range; these two can pass 32 MiB (the
 *   max_round_bytes begin reports, whatever the campaign's size) and are then sent in rounds of at most that many
 *   bytes.  Every key of every bucket reaches every rank, a window at a time: about 8
 *   bytes per complete world and selected plane, as much as gathering the planes; what the rounds buy is device memory
 *   per rank bounded by its own worlds and a window, never every rank's planes.  A task reads the rank's plane at most
 *   6 times (5 histogram passes and the scatter; the completeness read not counted); b200_sixdof_rank_reads, set by the
 *   end, averages them over every (group, plane) task of the call, a group with no complete world on any rank counting
 *   none.
 *   Memory.  The rank planes of the unsharded entries.  Device scratch of the call's own (not the staging buffer),
 *   allocated as the call needs it and freed by its end (or by a discard, a failure or the next begin):
 *     - per task of a slice, for its worlds on this rank: 48 bytes per complete world (its pieces, bucket list and
 *       keys: only pieces that hold worlds of this rank are kept) and 4 per world, plus 32 bytes per 8193 complete
 *       worlds over every rank (the ranges); the slices are cut so that this is at most 256 MiB on the rank holding
 *       the most of each group, unless one task alone needs more;
 *     - the histograms of two consecutive levels, 64 KiB per range that exists (a range holds more than 8192 worlds
 *       over every rank; tens of ranges on continuous values);
 *     - the exchange: at most 32 MiB, or one level's histograms or the sizes (G * n_ranks * 8 bytes) if they are
 *       larger.  The sizes grow with the rank count: 8 KiB per rank at 1024 groups, about 64 GiB of device memory
 *       (and as much host memory, which the sizes round reads back) near the limit of 2^23 - 1 ranks.
 *   A cudaMalloc that fails ends the call with B200_ERR_OUT_OF_MEMORY and leaves the handle usable.
 *   At most 8,388,607 ranks (2^23 - 1): the begin refuses more with B200_ERR_INVALID_ARGUMENT.
 *   Preconditions (a C host checks them itself; sharding.gather_ranks does): every rank passes the same grouping,
 *   planes, n_ranks and outcome count and a distinct rank, a rank's groups are the global groups cut to its worlds (the
 *   same G on every rank; a group may be empty on a rank).  A group of more than 1,073,872,895 complete worlds over the
 *   ranks (what a world state can index) fails the sizes round with B200_ERR_INVALID_ARGUMENT on every rank.
 *   Between begin and end the handle's outcome planes must not change: a step, upload, invoke_batch,
 *   trajectory_reset, set_channels, set_outcomes, set_world_groups, summary begin, start or add makes the next round or
 *   end fail with B200_ERR_INVALID_ARGUMENT and discards the call.  Any call of an unsharded rank entry
 *   (b200_sixdof_outcome_[group_]ranks or _rank_correlation) discards it too, since it rewrites the rank planes; any
 *   other reduction may run between rounds. ---- */
/* Checks what b200_sixdof_outcome_[group_]ranks checks, in the same order (the outcome set, the groups when grouped,
 * the selection of 1 .. P planes), then the sticky status, then rank < n_ranks and n_ranks < 2^23
 * (B200_ERR_INVALID_ARGUMENT), after B200_ERR_INVALID_ARGUMENT for a null handle or a null max_round_bytes; discards a
 * call still pending; writes the outcome planes of the summaries, fixes the grouping, planes, rank and n_ranks of the
 * call and writes its largest round in bytes. */
int b200_sixdof_sharded_ranks_begin(b200_sixdof *h, int grouped, const uint32_t *planes, uint32_t n_p, uint32_t rank,
                                    uint32_t n_ranks, uint64_t *max_round_bytes);
/* One round, with the contract of b200_sixdof_sharded_quantiles_round: `reduced` = the ranks' elementwise sum of this
 * rank's previous partial (NULL, 0 on the first call), `partial` (partial_cap >= begin's max_round_bytes) receives the
 * next round's words, *partial_bytes == 0: the rank planes are ready.  The same refusals, and
 * B200_ERR_INVALID_ARGUMENT, discarding the call, for a group too large (above). */
int b200_sixdof_sharded_ranks_round(b200_sixdof *h, const void *reduced, uint64_t reduced_bytes, void *partial,
                                    uint64_t partial_cap, uint64_t *partial_bytes);
/* ranks_dst (host or device, or NULL) = [n_worlds][n_p] f64: the campaign midranks of this rank's worlds; cov_dst (host
 * or device, or NULL) = [G, or 1 ungrouped][1 + n_p + n_p^2] f64: the covariance record (b200_sixdof_outcome_covariance's
 * layout and kernels) of the rank planes over this rank's complete worlds.  A destination's bytes must match exactly
 * (else B200_ERR_VALUE_SIZE_MISMATCH).  B200_ERR_INVALID_ARGUMENT for an end without a begin, before the last round, or
 * after the outcomes changed.  Ends the call. */
int b200_sixdof_sharded_ranks_end(b200_sixdof *h, void *ranks_dst, uint64_t ranks_bytes, void *cov_dst,
                                  uint64_t cov_bytes);

/* plumbing */
uint64_t b200_sixdof_tick_count(const b200_sixdof *h);
/* Run the handle's work on a caller-owned cudaStream_t (`cuda_stream`, where NULL is
 * the legacy default stream, e.g. torch.cuda.current_stream().cuda_stream), or, with
 * use_own_stream != 0, go back to the handle's private non-blocking stream.  Waits for
 * the work queued on the stream it leaves.  On a caller stream, every entry is ordered
 * after the work already queued on that stream, and the caller's later work on it sees
 * what the entry did (b200_sixdof_step: the new state, e.g. through
 * b200_sixdof_device_plane, with no sync in between).  Entries that return data
 * (downloads, invoke_batch, reductions) return with it complete.  The private stream
 * has no ordering with any other stream: a caller that shares buffers with the handle
 * there synchronises first. */
int b200_sixdof_set_stream(b200_sixdof *h, void *cuda_stream, int use_own_stream);
int b200_sixdof_timings(const b200_sixdof *h, b200_timings *out);
int b200_sixdof_status(const b200_sixdof *h);                  /* sticky status of the handle */
/* raw device plane pointer (plane p of a column), for zero-copy interop (NCCL gather).  Asking for an Inertia
 * plane lets the caller change masses behind the handle's back: from that call on, the handle reads every mass
 * on every tick (it no longer trusts its per-segment summary of which masses are regular). */
void *b200_sixdof_device_plane(b200_sixdof *h, uint64_t component_id, uint32_t plane);
uint64_t b200_sixdof_plane_stride(const b200_sixdof *h); /* doubles between planes */

/* ---- multi-GPU (SURVEY §8e).  Worlds shard across GPUs — one handle per GPU, one process (or thread) per
 * handle, no data-path collective — exactly like the reference's one-OS-process-per-world Monte-Carlo driver
 * (libs/monte-carlo/src/lib.rs:2083).  The one exchange is the end-of-run gather of the trajectory ring, over
 * NCCL (NVLink 4 / NVSwitch).  NCCL is bound at run time (dlopen of libnccl.so.2: the copy the host process already
 * loaded, else the system one); b200_comm_available() == 0 means it could not be found. ---- */
#define B200_COMM_ID_BYTES 128u                      /* sizeof(ncclUniqueId) */
typedef struct b200_comm b200_comm;                   /* opaque: one NCCL communicator rank */
int b200_comm_available(void);
int b200_comm_version(void);                          /* NCCL version code, 0 if unavailable */
/* rank 0 creates the id and hands its bytes to every rank over any channel the host has (the reference's
 * Monte-Carlo driver would put it in context.json); then every rank calls b200_comm_create. */
int b200_comm_unique_id(uint8_t *out, uint32_t bytes);
int b200_comm_create(const uint8_t *id, int n_ranks, int rank, int device, b200_comm **out);
void b200_comm_destroy(b200_comm *c);
int b200_comm_rank(const b200_comm *c);
int b200_comm_size(const b200_comm *c);
double b200_comm_last_ms(const b200_comm *c);         /* device time of the last gather (layout kernel + collective) */
/* World-sharded all-gather of the trajectory ring.  Rank r holds worlds_per_rank[r] worlds (same samples, entities
 * and ring width everywhere; ragged world counts allowed).  On return `dst` (device or host memory) holds
 * [sum(worlds)][samples][n_entities][width] f64 in rank order on every rank; dst_bytes must equal
 * b200_sixdof_trajectory_gather_bytes(). */
uint64_t b200_sixdof_trajectory_gather_bytes(const b200_sixdof *h, const uint64_t *worlds_per_rank, int n_ranks);
int b200_sixdof_trajectory_allgather(b200_sixdof *h, b200_comm *c, const uint64_t *worlds_per_rank, void *dst,
                                     uint64_t dst_bytes);

/* ONE world, source rows split over the ranks (SURVEY §8e second case; needs dense edge_fold gravity, n_worlds = 1,
 * n_entities divisible by the rank count).  Every rank creates the same handle and uploads the same initial state,
 * then calls this instead of b200_sixdof_step: per tick it folds and integrates its own rows and all-gathers the
 * rows' new position / velocity planes over NCCL; after the call every rank holds the complete world (WorldPos,
 * WorldVel, WorldAccel, Force).  Each rank's tick samples the trajectory ring for its own rows only, and the ring is not
 * gathered: with more than one rank, a handle with a trajectory ring is refused (B200_ERR_UNSUPPORTED); with one rank
 * the ring is complete.  Any other entry (step, upload, invoke_batch, trajectory_reset) may run between two calls.
 * At N = 1024 replicas (every GPU integrates the whole world, no exchange) are faster — the tick is a ~10 us
 * latency chain and the exchange adds to it; row shards pay off for worlds of several thousand bodies
 * (DESIGN.md §7, measured by bench.py `multi_gpu.nbody_1024_single_world`). */
int b200_sixdof_step_row_sharded(b200_sixdof *h, b200_comm *c, uint64_t n_ticks);

/* Peer window for the row-sharded world: compute and exchange without a collective in the tick loop.  Every rank
 * allocates a window (the x, v planes of the whole world, twice — tick-count parity — plus one delivery counter per
 * rank), the ranks swap the windows' CUDA IPC handles through the communicator and map each other's.  With a window
 * attached, b200_sixdof_step_row_sharded runs per tick: wait until every rank's rows of this tick count have landed
 * here -> gravity from the window -> integrate own rows -> store the rows' new x, v straight into every rank's window
 * over NVLink and release each counter.  Only the call's last tick still all-gathers (attitude, WorldAccel, Force of
 * the other ranks' rows).  Results are bit-identical to the NCCL route and to replicas.  The window counts its own
 * ticks (zeroed by attach), so a trajectory reset or any other operation on the handle between calls is safe.
 * Collective: every rank of `c` calls attach (and detach / b200_comm_destroy) with handles of the same shape; one
 * window per communicator.  Returns B200_ERR_UNSUPPORTED on every rank if any rank cannot map the windows (no IPC
 * between the processes) — the NCCL route keeps working.  B200_ROW_PEER=0 ignores an attached window. */
#define B200_MAX_PEERS 16
int b200_comm_peer_attach(b200_comm *c, b200_sixdof *h);
int b200_comm_peer_attached(const b200_comm *c);
void b200_comm_peer_detach(b200_comm *c);

/* Concurrent host<->device copy bandwidth of one GPU through pinned `host` (>= h2d_bytes + d2h_bytes): out[0] = H2D
 * GB/s, out[1] = D2H GB/s, both directions running at once — the ceiling an invoke_batch round trip sits under. */
int b200_probe_pcie_gbs(int device, void *host, uint64_t h2d_bytes, uint64_t d2h_bytes, int iters, double *out);
/* The same with kernels instead of the copy engines (SMs reading / writing mapped pinned host memory, `blocks` CTAs of
 * 256 threads per direction): B200_ERR_UNSUPPORTED when `host` is not mapped into the device address space. */
int b200_probe_zero_copy_gbs(int device, void *host, uint64_t h2d_bytes, uint64_t d2h_bytes, int iters, int blocks, double *out);

/* FP64 / HBM probes used by bench.py to report the roofs next to the kernel
 * numbers (device-timed, returns GB/s resp. GFLOP/s, <0 on error) */
double b200_probe_copy_gbs(int device, uint64_t bytes, int iters);
double b200_probe_fp64_gflops(int device, int iters);
/* The term stream a GRAVITY_EGM08 effector of this degree is evaluated from (DESIGN.md §5): eight f64 per (m, l) term in
 * consumption order — recursion constants of A at (l, m) and of B at (l+1, m+1), C, S, nq1, nq2.  Host-only. */
uint64_t b200_egm08_stream_len(uint32_t max_degree);
int b200_egm08_stream(uint32_t max_degree, const double *c_bar, const double *s_bar, double *out, uint64_t out_len);
/* Self-test of the EXACT mode's division-by-a-shared-divisor route (sixdof_device.cuh ex::div_rcp) against the GPU's
 * IEEE division on n_groups pseudo-random operand groups covering every encoding class: out[0] = results differing
 * in any bit (0 on a correct build), out[1] = groups that did not need the __ddiv_rn fallback. */
int b200_selftest_shared_divisor(int device, uint64_t seed, uint64_t n_groups, uint64_t *out);

#ifdef __cplusplus
}
#endif
#endif /* B200_SIXDOF_H */
