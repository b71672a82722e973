// sm_90a per-body integrator kernels of the six_dof() hot path (K1/K2/K4/K5 of SURVEY §2.4).
//
//   body_exact_kernel       EXACT arithmetic: one thread per body, the whole tick (clear_forces, effectors x4,
//                           calc_accel x4, stage advance x4, final combine, renormalise) in registers, n_ticks
//                           ticks per launch.
//   body_fast_spec_kernel   FAST arithmetic compiled per effector signature (the default FAST route).
//   body_fast_kernel        FAST arithmetic with the run-time effector interpreter (effector lists no signature covers).
#include <cstdint>
#include <cstring>

#include "sixdof_tick.cuh"
#include "sixdof_launch.h"

namespace b200 {

// ================================================================== EXACT body kernel

template <int INTEG, int BLOCK, int MINB, bool UNR = false, uint32_t SEQ = SEQ_INTERPRET>
__global__ void __launch_bounds__(BLOCK, MINB) body_exact_kernel(const __grid_constant__ StepParams P)
{
    const uint64_t b = (uint64_t)blockIdx.x * BLOCK + threadIdx.x;
    if (b >= P.n_bodies) return;

    Pose x0 = load_pose(P.pos, P.ld, b);
    Motion v0 = load_motion(P.vel, P.ld, b);
    Motion a_out = load_motion(P.acc, P.ld, b);
    Motion f_out = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    const Inertia I = load_inertia(P.ine, P.ld, b);
    const GravReg no_greg{};

    uint32_t traj_phase = 0; // one 64-bit division per launch, not per tick (see fast_ticks)
    uint64_t traj_slot = 0;
    if (P.traj_every) { traj_phase = (uint32_t)(P.tick0 % P.traj_every); traj_slot = P.tick0 / P.traj_every; }
    for (uint32_t t = 0; t < P.n_ticks; ++t) {
        exact_tick<INTEG, false, UNR, SEQ>(P, b, x0, v0, a_out, f_out, I, no_greg);
        if (P.traj_every && ++traj_phase == P.traj_every) {
            traj_phase = 0;
            if (traj_slot < P.traj_capacity) {
                traj_store_state(P, b, traj_slot, x0, v0);
                if (P.traj_planes == 25) traj_store_af(P, b, traj_slot, a_out, f_out);
            }
            ++traj_slot;
        }
    }
    store_pose(P.pos, P.ld, b, x0);
    store_motion(P.vel, P.ld, b, v0);
    store_motion(P.acc, P.ld, b, a_out);
    store_motion(P.frc, P.ld, b, f_out);
}

// ================================================================== FAST body kernels

// Effector columns are consumed inside the (uniform) effector switch, i.e. after the state
// loads and the reciprocal prologue; prefetching them first puts their HBM latency under the
// state loads instead of behind them.
__device__ __forceinline__ void prefetch_effector_columns(const StepParams &P, uint64_t b)
{
    for (uint32_t e = 0; e < P.n_eff; ++e) {
        const double *col = P.eff[e].col;
        if (!col) continue;
        const uint32_t w = P.eff[e].col_width;
        for (uint32_t k = 0; k < w; ++k) asm volatile("prefetch.global.L1 [%0];" ::"l"(col + (uint64_t)k * P.ld + b));
    }
    if (P.gforce)
        for (uint32_t k = 0; k < 9; ++k) asm volatile("prefetch.global.L1 [%0];" ::"l"(P.gforce + (uint64_t)k * P.ld + b));
}

template <int INTEG, int BLOCK, int MINB, bool TRAJ>
__global__ void __launch_bounds__(BLOCK, MINB) body_fast_kernel(const __grid_constant__ StepParams P)
{
    const uint64_t b = (uint64_t)blockIdx.x * BLOCK + threadIdx.x;
    if (b >= P.n_bodies) return;
    prefetch_effector_columns(P, b);
    Pose x0 = load_pose(P.pos, P.ld, b);
    Motion v0 = load_motion(P.vel, P.ld, b);
    const Inertia I = load_inertia(P.ine, P.ld, b);
    Motion a_last, f_last;
    fast_ticks<INTEG, TRAJ>(P, b, x0, v0, I, a_last, f_last, P.n_ticks, P.tick0, P.write_fa != 0, GravReg{});
    store_pose(P.pos, P.ld, b, x0);
    store_motion(P.vel, P.ld, b, v0);
    if (P.write_fa) {
        store_motion(P.acc, P.ld, b, a_last);
        store_motion(P.frc, P.ld, b, f_last);
    }
}


// ------------------------------------------------------------------ specialised FAST kernels
//
// One instantiation per (integrator, effector signature): the per-body effector inputs are loaded next to the
// 14 to 17 state planes — every load of a body is in flight before the first dependent instruction — and the tick is
// compiled for exactly that effector set.  BPT = bodies per thread: 2 reads every plane as double2 (LDG.E.128,
// body pair 2t, 2t+1) and integrates the pair back to back, so the second body's loads stay in flight under the
// first body's arithmetic.
template <int BPT> struct VecIO;
template <> struct VecIO<1> {
    static __device__ __forceinline__ void ld(const double *p, uint64_t i, double (&o)[1]) { o[0] = p[i]; }
    static __device__ __forceinline__ void st(double *p, uint64_t i, const double (&v)[1], bool) { p[i] = v[0]; }
};
template <> struct VecIO<2> {
    static __device__ __forceinline__ void ld(const double *p, uint64_t i, double (&o)[2])
    {
        const double2 v = *reinterpret_cast<const double2 *>(p + i); // i even, plane base 16-byte aligned (host-checked)
        o[0] = v.x; o[1] = v.y;
    }
    static __device__ __forceinline__ void st(double *p, uint64_t i, const double (&v)[2], bool both)
    {
        if (both) *reinterpret_cast<double2 *>(p + i) = make_double2(v[0], v[1]);
        else p[i] = v[0]; // odd tail: the pair's second body lies outside this launch's range
    }
};

#define B200_LDV(base, plane, expr)                                                        \
    do {                                                                                   \
        double t_[BPT];                                                                    \
        VecIO<BPT>::ld((base) + (uint64_t)(plane) * P.ld, b0, t_);                         \
        _Pragma("unroll") for (int k = 0; k < BPT; ++k) { expr = t_[k]; }                  \
    } while (0)
#define B200_STV(base, plane, expr)                                                        \
    do {                                                                                   \
        double t_[BPT];                                                                    \
        _Pragma("unroll") for (int k = 0; k < BPT; ++k) { t_[k] = expr; }                  \
        VecIO<BPT>::st((base) + (uint64_t)(plane) * P.ld, b0, t_, both);                   \
    } while (0)

template <int INTEG, uint32_t SIG, bool TRAJ, int BLOCK, int MINB, int BPT>
__global__ void __launch_bounds__(BLOCK, MINB) body_fast_spec_kernel(const __grid_constant__ StepParams P)
{
    // Odd launches walk the planes from the far end: the tail of the state the previous launch read and wrote last is
    // still in the 50 MB L2 when this launch starts — read it first, before this launch's own traffic evicts it, and the
    // rewrite lands on lines that are still dirty instead of costing a second DRAM write (scripts/tune_snake.py A/B-times it
    // against B200_SNAKE=0).
    const unsigned blk = P.reverse ? gridDim.x - 1u - blockIdx.x : blockIdx.x;
    const uint64_t b0 = ((uint64_t)blk * BLOCK + threadIdx.x) * BPT;
    // a torque (I^-1) changes the angular velocity of practically every body, and the signatures that carry one also
    // change the linear velocity (gravity, wrench force): they store WorldVel unconditionally (their pair kernels sit
    // at the 168-register bound, where tracking the changed planes would spill)
    constexpr bool TORQUE = (SIG & (SIG_WRENCH | SIG_WHEELS | SIG_WWORLD)) != 0;
    const unsigned live = TORQUE ? 0u : __ballot_sync(0xffffffffu, b0 < P.n_bodies); // lanes that reach the stores
    if (b0 >= P.n_bodies) return;
    const bool both = b0 + (BPT - 1) < P.n_bodies;

    Pose x[BPT];
    Motion v[BPT];
    Inertia I[BPT];
    EffIn in[BPT];
    B200_LDV(P.pos, 0, x[k].q.i); B200_LDV(P.pos, 1, x[k].q.j); B200_LDV(P.pos, 2, x[k].q.k); B200_LDV(P.pos, 3, x[k].q.w);
    B200_LDV(P.pos, 4, x[k].x.x); B200_LDV(P.pos, 5, x[k].x.y); B200_LDV(P.pos, 6, x[k].x.z);
    B200_LDV(P.vel, 0, v[k].ang.x); B200_LDV(P.vel, 1, v[k].ang.y); B200_LDV(P.vel, 2, v[k].ang.z);
    B200_LDV(P.vel, 3, v[k].lin.x); B200_LDV(P.vel, 4, v[k].lin.y); B200_LDV(P.vel, 5, v[k].lin.z);
    // The inertia diagonal is read by I^-1 (body-frame and world-frame torques) and by the Force column's torque
    // R (I .* u), which is formed on a batch's last launch (write_fa) and for full trajectory samples; every other
    // launch leaves the three planes in HBM and never reads the zeros below.
    if (TORQUE || P.write_fa || (TRAJ && P.traj_planes == 25)) {
        B200_LDV(P.ine, 0, I[k].diag.x); B200_LDV(P.ine, 1, I[k].diag.y); B200_LDV(P.ine, 2, I[k].diag.z);
    } else {
#pragma unroll
        for (int k = 0; k < BPT; ++k) I[k].diag = Vec3{0.0, 0.0, 0.0};
    }
    // The mass-class summary (P.mass_class; the host passes it only to signature-0 launches with a +0 gravity that form
    // no Force): one byte per warp of pairs, 1 when mass_is_regular holds for all 64 masses of the segment.  Such a warp
    // integrates with m = 1 — the same bits — and leaves the mass plane in HBM; a warp whose byte is 0 reads the plane
    // and, when its whole segment lies in this launch, records what it found.
    uint8_t *const mass_class = SIG == 0u && BPT == 2 ? P.mass_class : nullptr;
    const bool mass_known = mass_class && mass_class[b0 >> 6] != 0; // warp-uniform
    if (mass_known) {
#pragma unroll
        for (int k = 0; k < BPT; ++k) I[k].m = 1.0;
    } else {
        B200_LDV(P.ine, 6, I[k].m);
        if (mass_class && (b0 | 63u) < P.n_bodies) { // every lane of the warp is live and holds two bodies
            bool regular = true;
#pragma unroll
            for (int k = 0; k < BPT; ++k) regular &= mass_is_regular(I[k].m);
            if (__all_sync(0xffffffffu, regular) && (threadIdx.x & 31u) == 0) mass_class[b0 >> 6] = 1;
        }
    }
#pragma unroll
    for (int k = 0; k < BPT; ++k) {
        in[k].thrust = 0.0; in[k].cd_rho = in[k].area = 0.0;
        in[k].wr_t = in[k].wr_f = in[k].wind = in[k].wheels = in[k].ww_t = in[k].ww_f = Vec3{0.0, 0.0, 0.0};
    }
    if (SIG & SIG_THRUST) B200_LDV(P.spec.thrust, 0, in[k].thrust);
    if (SIG & SIG_WRENCH) {
        B200_LDV(P.spec.wr_t, 0, in[k].wr_t.x); B200_LDV(P.spec.wr_t, 1, in[k].wr_t.y); B200_LDV(P.spec.wr_t, 2, in[k].wr_t.z);
        B200_LDV(P.spec.wr_f, 0, in[k].wr_f.x); B200_LDV(P.spec.wr_f, 1, in[k].wr_f.y); B200_LDV(P.spec.wr_f, 2, in[k].wr_f.z);
    }
    if (SIG & SIG_WHEELS) { // the three wheel torques only ever enter as their sum (the rotation is linear)
        Vec3 w[BPT][3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            B200_LDV(P.spec.wheels, 3 * q + 0, w[k][q].x); B200_LDV(P.spec.wheels, 3 * q + 1, w[k][q].y); B200_LDV(P.spec.wheels, 3 * q + 2, w[k][q].z);
        }
#pragma unroll
        for (int k = 0; k < BPT; ++k)
            in[k].wheels = Vec3{w[k][0].x + w[k][1].x + w[k][2].x, w[k][0].y + w[k][1].y + w[k][2].y, w[k][0].z + w[k][1].z + w[k][2].z};
    }
    if (SIG & SIG_WWORLD) {
        B200_LDV(P.spec.wworld, 0, in[k].ww_t.x); B200_LDV(P.spec.wworld, 1, in[k].ww_t.y); B200_LDV(P.spec.wworld, 2, in[k].ww_t.z);
        B200_LDV(P.spec.wworld, 3, in[k].ww_f.x); B200_LDV(P.spec.wworld, 4, in[k].ww_f.y); B200_LDV(P.spec.wworld, 5, in[k].ww_f.z);
    }
    if (SIG & SIG_DRAG) {
        B200_LDV(P.spec.drag, 0, in[k].wind.x); B200_LDV(P.spec.drag, 1, in[k].wind.y); B200_LDV(P.spec.drag, 2, in[k].wind.z);
        if (SIG & SIG_DRAG_PB) { B200_LDV(P.spec.drag, 3, in[k].cd_rho); B200_LDV(P.spec.drag, 4, in[k].area); }
    }

    // A (WorldPos, WorldVel) sample on every launch of one tick: the pair stores it from here as one 16-byte store per
    // plane — the per-body 8-byte stores inside fast_ticks fill half of every sector, and the other half arrives a whole
    // tick of arithmetic later
    const bool defer_traj = TRAJ && BPT == 2 && both && P.n_ticks == 1 && P.traj_planes == 13;
    Motion a_last[BPT], f_last[BPT];
    // Only one-tick launches track the changed WorldVel planes: in a launch of several ticks the stores are amortised
    // over the ticks, and the tracking inside the tick loop costs the FP64-bound fused loop its unrolling (~9 %).
    const bool track_vel = !TORQUE && P.n_ticks == 1;
    uint32_t vel_changed = track_vel ? 0u : 0x3fu; // WorldVel planes the launch changed for either body of the pair
#pragma unroll
    for (int k = 0; k < BPT; ++k)
        if (k == 0 || both) {
            if (track_vel)
                fast_ticks<INTEG, TRAJ, false, SIG>(P, b0 + k, x[k], v[k], I[k], a_last[k], f_last[k], 1u, P.tick0,
                                                    P.write_fa != 0, GravReg{}, in[k], !defer_traj, &vel_changed);
            else
                fast_ticks<INTEG, TRAJ, false, SIG>(P, b0 + k, x[k], v[k], I[k], a_last[k], f_last[k], P.n_ticks, P.tick0,
                                                    P.write_fa != 0, GravReg{}, in[k], !defer_traj);
        }
    if (TRAJ && BPT == 2 && defer_traj && P.traj_every) {
        const uint64_t after = P.tick0 + 1;
        const uint64_t slot = after / P.traj_every - 1;
        if (after % P.traj_every == 0 && slot < P.traj_capacity) {
            double *t = P.traj + slot * 13ull * P.ld + b0;
            auto put = [&](int plane, double v0, double v1) { __stcs(reinterpret_cast<double2 *>(t + (uint64_t)plane * P.ld), make_double2(v0, v1)); };
            constexpr int o = BPT - 1; // index of the pair's second body (0 when the kernel is compiled for one body per thread)
            put(0, x[0].q.i, x[o].q.i); put(1, x[0].q.j, x[o].q.j); put(2, x[0].q.k, x[o].q.k); put(3, x[0].q.w, x[o].q.w);
            put(4, x[0].x.x, x[o].x.x); put(5, x[0].x.y, x[o].x.y); put(6, x[0].x.z, x[o].x.z);
            put(7, v[0].ang.x, v[o].ang.x); put(8, v[0].ang.y, v[o].ang.y); put(9, v[0].ang.z, v[o].ang.z);
            put(10, v[0].lin.x, v[o].lin.x); put(11, v[0].lin.y, v[o].lin.y); put(12, v[0].lin.z, v[o].lin.z);
        }
    }

    B200_STV(P.pos, 0, x[k].q.i); B200_STV(P.pos, 1, x[k].q.j); B200_STV(P.pos, 2, x[k].q.k); B200_STV(P.pos, 3, x[k].q.w);
    B200_STV(P.pos, 4, x[k].x.x); B200_STV(P.pos, 5, x[k].x.y); B200_STV(P.pos, 6, x[k].x.z);
    // WorldVel is updated in place, so a plane whose bits no tick changed is already what a store would write: a torque-
    // free tick leaves the angular planes as they were, a force-free one the linear planes.  The warp decides per plane
    // (whole 32-byte sectors, never a partial one that could cost the L2 a read-modify-write).
    const uint32_t vel_store = track_vel ? __reduce_or_sync(live, vel_changed) : 0x3fu;
    if (vel_store & 1u) B200_STV(P.vel, 0, v[k].ang.x);
    if (vel_store & 2u) B200_STV(P.vel, 1, v[k].ang.y);
    if (vel_store & 4u) B200_STV(P.vel, 2, v[k].ang.z);
    if (vel_store & 8u) B200_STV(P.vel, 3, v[k].lin.x);
    if (vel_store & 16u) B200_STV(P.vel, 4, v[k].lin.y);
    if (vel_store & 32u) B200_STV(P.vel, 5, v[k].lin.z);
    if (P.write_fa) {
        B200_STV(P.acc, 0, a_last[k].ang.x); B200_STV(P.acc, 1, a_last[k].ang.y); B200_STV(P.acc, 2, a_last[k].ang.z);
        B200_STV(P.acc, 3, a_last[k].lin.x); B200_STV(P.acc, 4, a_last[k].lin.y); B200_STV(P.acc, 5, a_last[k].lin.z);
        B200_STV(P.frc, 0, f_last[k].ang.x); B200_STV(P.frc, 1, f_last[k].ang.y); B200_STV(P.frc, 2, f_last[k].ang.z);
        B200_STV(P.frc, 3, f_last[k].lin.x); B200_STV(P.frc, 4, f_last[k].lin.y); B200_STV(P.frc, 5, f_last[k].lin.z);
    }
}

// ================================================================== launchers

// the instantiation without trajectory code for launches that record nothing, the generic one otherwise
#define BODY_FAST(INTEG, BLOCK, MINB)                                                        \
    do {                                                                                     \
        if (P.traj_every) body_fast_kernel<INTEG, BLOCK, MINB, true><<<g(BLOCK), BLOCK, 0, s>>>(P);  \
        else body_fast_kernel<INTEG, BLOCK, MINB, false><<<g(BLOCK), BLOCK, 0, s>>>(P);      \
    } while (0)

// ------------------------------------------------------------------ effector list -> signature
//
// A signature covers an effector list when the folded result does not depend on anything the compile-time form
// cannot express: no entity masks (query-join membership), at most one thrust / wrench / drag / frame effector,
// no wrench ahead of the drag (apply_drag resets the torque accumulated before it), a drag that has its wind
// column, the edge_fold gravity first.  Everything else keeps the run-time interpreter.
static uint32_t spec_signature(StepParams &Q)
{
    uint32_t sig = 0;
    int n_thrust = 0, n_wrench = 0, n_drag = 0, n_frame = 0;
    bool wrench_seen = false;
    StepParams::Spec sp{};
    for (uint32_t i = 0; i < Q.n_eff; ++i) {
        const EffDev &E = Q.eff[i];
        if (E.mask) return SIG_GENERIC;
        switch (E.kind) {
        case B200_EFF_GRAVITY_CONST:
            sp.g[0] += E.p[0]; sp.g[1] += E.p[1]; sp.g[2] += E.p[2];
            break;
        case B200_EFF_DRAG_QUADRATIC:
            if (!E.col || wrench_seen || ++n_drag > 1) return SIG_GENERIC;
            sig |= SIG_DRAG | (E.col_width == 5 ? SIG_DRAG_PB : 0u);
            sp.kd = 0.5 * E.p[0] * E.p[1];
            sp.drag = E.col;
            break;
        case B200_EFF_THRUST_BODY:
            if (!E.col || ++n_thrust > 1) return SIG_GENERIC;
            sig |= SIG_THRUST;
            sp.axis[0] = E.p[0]; sp.axis[1] = E.p[1]; sp.axis[2] = E.p[2];
            sp.thrust = E.col;
            break;
        case B200_EFF_WRENCH_BODY: {
            if (!E.col || ++n_wrench > 1) return SIG_GENERIC;
            wrench_seen = true;
            sig |= SIG_WRENCH;
            const uint64_t to = (E.flags & B200_EFF_FLAG_WRENCH_LINEAR_FIRST) ? 3 : 0;
            sp.wr_t = E.col + to * Q.ld;
            sp.wr_f = E.col + (3 - to) * Q.ld;
            break;
        }
        case B200_EFF_GRAVITY_FRAME:
            if (++n_frame > 1) return SIG_GENERIC;
            sig |= SIG_FRAME;
            sp.mu = E.p[0]; sp.om[0] = E.p[1]; sp.om[1] = E.p[2]; sp.om[2] = E.p[3];
            break;
        case B200_EFF_GRAVITY_EDGES_NEWTON:
        case B200_EFF_GRAVITY_EDGES_SOFTENED:
            if (i != 0 || !Q.gforce || !Q.has_edge) return SIG_GENERIC;
            sig |= SIG_GRAPH;
            break;
        case B200_EFF_GRAVITY_J2:
            if (sig & SIG_J2) return SIG_GENERIC;
            sig |= SIG_J2;
            sp.j2_mu = E.p[0]; sp.j2_k = E.p[1] * E.p[2] * E.p[2];
            break;
        case B200_EFF_WRENCH_WORLD:
            if (!E.col || (sig & SIG_WWORLD)) return SIG_GENERIC;
            sig |= SIG_WWORLD;
            sp.wworld = E.col;
            break;
        case B200_EFF_TORQUE_BODY_FOLD: // the fold overwrites Force: only as the first effector is it a plain torque term
            if (i != 0 || !E.col || E.col_width != 9) return SIG_GENERIC;
            sig |= SIG_WHEELS;
            sp.wheels = E.col;
            break;
        default: return SIG_GENERIC;
        }
    }
    Q.spec = sp;
    return sig;
}

// launch shape of the specialised kernels: (threads per CTA, resident CTAs per SM the register allocation is bounded
// for, bodies per thread).  B200_SPEC_CFG selects among the shapes a tuning build (-DB200_TUNE) instantiates.
template <int INTEG, uint32_t SIG, bool TRAJ, int BLOCK, int MINB, int BPT>
static void launch_spec_shape(const StepParams &Q, cudaStream_t s)
{
    const uint64_t threads = (Q.n_bodies + BPT - 1) / BPT;
    const unsigned grid = (unsigned)((threads + BLOCK - 1) / BLOCK);
    body_fast_spec_kernel<INTEG, SIG, TRAJ, BLOCK, MINB, BPT><<<grid, BLOCK, 0, s>>>(Q);
}

static bool planes_16B_aligned(const StepParams &Q, uint32_t sig)
{
    uintptr_t a = (uintptr_t)Q.pos | (uintptr_t)Q.vel | (uintptr_t)Q.ine | (uintptr_t)Q.acc | (uintptr_t)Q.frc | (uintptr_t)Q.traj;
    if (sig & SIG_THRUST) a |= (uintptr_t)Q.spec.thrust;
    if (sig & SIG_WRENCH) a |= (uintptr_t)Q.spec.wr_t | (uintptr_t)Q.spec.wr_f;
    if (sig & SIG_DRAG) a |= (uintptr_t)Q.spec.drag;
    if (sig & SIG_WHEELS) a |= (uintptr_t)Q.spec.wheels;
    if (sig & SIG_WWORLD) a |= (uintptr_t)Q.spec.wworld;
    return (a & 15u) == 0 && (Q.ld & 1u) == 0;
}

// Default shape (scripts/tune_spec.py sweeps the others in a tuning build): body pairs (BPT = 2, LDG.E.128) at
// 128 threads x 3 CTAs/SM (<= 168 registers) keep every load of the pair in flight under the first body's arithmetic;
// on the H100 the free / rocket / falcon9 signatures move their touched bytes at the device copy rate.  Ranges too small to
// fill the machine with pairs, or whose planes are not 16-byte aligned (odd world-range offsets), take one body
// per thread.
template <int INTEG, uint32_t SIG, bool TRAJ>
static void launch_spec(const StepParams &Q, cudaStream_t s)
{
    const bool vec_ok = planes_16B_aligned(Q, SIG);
#ifdef B200_TUNE
    const int cfg = env_int("B200_SPEC_CFG", -1); // re-read per launch: one tuning process sweeps the shapes
    switch (cfg) {
    case 0: launch_spec_shape<INTEG, SIG, TRAJ, 128, 4, 1>(Q, s); return;
    case 1: launch_spec_shape<INTEG, SIG, TRAJ, 128, 5, 1>(Q, s); return;
    case 2: launch_spec_shape<INTEG, SIG, TRAJ, 128, 6, 1>(Q, s); return;
    case 3: launch_spec_shape<INTEG, SIG, TRAJ, 256, 2, 1>(Q, s); return;
    case 4: if (vec_ok) { launch_spec_shape<INTEG, SIG, TRAJ, 128, 3, 2>(Q, s); return; } break;
    case 5: if (vec_ok) { launch_spec_shape<INTEG, SIG, TRAJ, 128, 4, 2>(Q, s); return; } break;
    case 6: if (vec_ok) { launch_spec_shape<INTEG, SIG, TRAJ, 128, 2, 2>(Q, s); return; } break;
    case 7: if (vec_ok) { launch_spec_shape<INTEG, SIG, TRAJ, 64, 6, 2>(Q, s); return; } break;
    case 8: launch_spec_shape<INTEG, SIG, TRAJ, 64, 10, 1>(Q, s); return;
    default: break;
    }
#endif
    constexpr uint64_t kPairMinBodies = 2ull * 128 * 3 * kNumSMs; // one full wave of body pairs
    if (vec_ok && Q.n_bodies >= kPairMinBodies) launch_spec_shape<INTEG, SIG, TRAJ, 128, 3, 2>(Q, s);
    else launch_spec_shape<INTEG, SIG, TRAJ, 128, 4, 1>(Q, s);
}

// signatures with a compiled kernel; anything else falls back to the interpreter kernel
#ifdef B200_TUNE
#define B200_SPEC_SIGS(X) X(0u) X(SIG_THRUST | SIG_DRAG) X(SIG_FRAME | SIG_WRENCH)
#else
#define B200_SPEC_SIGS(X)                                                                                        \
    X(0u) X(SIG_DRAG) X(SIG_THRUST) X(SIG_WRENCH) X(SIG_FRAME) X(SIG_GRAPH)                                       \
    X(SIG_THRUST | SIG_DRAG) X(SIG_THRUST | SIG_DRAG | SIG_DRAG_PB) X(SIG_THRUST | SIG_WRENCH) X(SIG_FRAME | SIG_WRENCH)     \
    X(SIG_J2) X(SIG_WHEELS | SIG_J2) X(SIG_WWORLD) X(SIG_WHEELS | SIG_WWORLD)
#endif

template <int INTEG>
static bool launch_spec_sig(const StepParams &Q, uint32_t sig, cudaStream_t s)
{
    const bool traj = Q.traj_every != 0;
    switch (sig) {
#define X(SIGV)                                                                \
    case (SIGV):                                                               \
        if (traj) launch_spec<INTEG, (SIGV), true>(Q, s);                      \
        else launch_spec<INTEG, (SIGV), false>(Q, s);                          \
        return true;
        B200_SPEC_SIGS(X)
#undef X
    default: return false;
    }
}

// EXACT effector sequences with a compiled kernel (four bits per effector kind, list order); every other list —
// and any list with an entity mask — runs the interpreter kernel
#define B200_SEQ1(a) ((uint32_t)(a))
#define B200_SEQ2(a, b) ((uint32_t)(a) | ((uint32_t)(b) << 4))
#define B200_SEQ3(a, b, c) ((uint32_t)(a) | ((uint32_t)(b) << 4) | ((uint32_t)(c) << 8))
#define B200_EXACT_SEQS(X)                                                                                              \
    X(0u)                                                                                                               \
    X(B200_SEQ1(B200_EFF_GRAVITY_CONST))                                                                                \
    X(B200_SEQ2(B200_EFF_GRAVITY_CONST, B200_EFF_DRAG_QUADRATIC))                            /* ball/sim.py */          \
    X(B200_SEQ3(B200_EFF_GRAVITY_CONST, B200_EFF_THRUST_BODY, B200_EFF_DRAG_QUADRATIC))      /* rocket Monte-Carlo */   \
    X(B200_SEQ3(B200_EFF_GRAVITY_CONST, B200_EFF_THRUST_BODY, B200_EFF_WRENCH_BODY))         /* rocket/main.py */       \
    X(B200_SEQ2(B200_EFF_GRAVITY_FRAME, B200_EFF_WRENCH_BODY))                               /* falcon9/sim.py */       \
    X(B200_SEQ1(B200_EFF_GRAVITY_EDGES_NEWTON)) X(B200_SEQ1(B200_EFF_GRAVITY_EDGES_SOFTENED))                         \
    X(B200_SEQ2(B200_EFF_TORQUE_BODY_FOLD, B200_EFF_WRENCH_WORLD))                           /* cube-sat replay */

static uint32_t exact_sequence(const StepParams &P)
{
    if (P.n_eff > 5) return SEQ_INTERPRET;
    uint32_t seq = 0;
    for (uint32_t i = 0; i < P.n_eff; ++i) {
        if (P.eff[i].mask || P.eff[i].kind == 0 || P.eff[i].kind > 15) return SEQ_INTERPRET;
        seq |= P.eff[i].kind << (4 * i);
    }
    return seq;
}

template <int INTEG, int BLOCK, int MINB>
static bool launch_exact_seq(const StepParams &P, uint32_t seq, cudaStream_t s)
{
    const unsigned grid = (unsigned)((P.n_bodies + BLOCK - 1) / BLOCK);
    switch (seq) {
#define X(SEQV)                                                                            \
    case (SEQV):                                                                           \
        body_exact_kernel<INTEG, BLOCK, MINB, false, (SEQV)><<<grid, BLOCK, 0, s>>>(P);    \
        return true;
        B200_EXACT_SEQS(X)
#undef X
    default: return false;
    }
}

cudaError_t launch_body_step(const StepParams &P, int integrator, int math_mode, cudaStream_t s)
{
    if (P.n_bodies == 0) return cudaSuccess;
    const bool rk4 = integrator == B200_INTEGRATOR_RK4;
    if (math_mode == B200_MATH_EXACT) {
#ifdef B200_TUNE
        const int xcfg = env_int("B200_EXACT_CFG", 3);
#else
        static const int xcfg = env_int("B200_EXACT_CFG", 3);
#endif
        auto g = [&](int blk) { return (unsigned)((P.n_bodies + blk - 1) / blk); };
        // default: the kernel compiled for this effector sequence (no run-time interpreter in the tick); the interpreter
        // kernel for every other list
        if (xcfg == 3) {
            const uint32_t seq = exact_sequence(P);
#ifdef B200_TUNE
            if (seq != SEQ_INTERPRET && rk4) switch (env_int("B200_EXACT_SEQ_CFG", 0)) { // registers vs warps for the compiled sequences
            case 1: if (launch_exact_seq<B200_INTEGRATOR_RK4, 128, 3>(P, seq, s)) return cudaGetLastError(); break;
            case 2: if (launch_exact_seq<B200_INTEGRATOR_RK4, 128, 2>(P, seq, s)) return cudaGetLastError(); break;
            case 3: if (launch_exact_seq<B200_INTEGRATOR_RK4, 64, 6>(P, seq, s)) return cudaGetLastError(); break;
            case 4: if (launch_exact_seq<B200_INTEGRATOR_RK4, 128, 5>(P, seq, s)) return cudaGetLastError(); break;
            default: break;
            }
#endif
            if (seq != SEQ_INTERPRET &&
                (rk4 ? launch_exact_seq<B200_INTEGRATOR_RK4, 128, 4>(P, seq, s) : launch_exact_seq<B200_INTEGRATOR_SEMI_IMPLICIT, 256, 1>(P, seq, s)))
                return cudaGetLastError();
        }
        if (!rk4) body_exact_kernel<B200_INTEGRATOR_SEMI_IMPLICIT, 256, 1><<<g(256), 256, 0, s>>>(P);
        else switch (xcfg) {
        case 1: body_exact_kernel<B200_INTEGRATOR_RK4, 256, 2><<<g(256), 256, 0, s>>>(P); break;
        case 0: body_exact_kernel<B200_INTEGRATOR_RK4, 256, 1><<<g(256), 256, 0, s>>>(P); break;
#ifdef B200_TUNE
        case 4: body_exact_kernel<B200_INTEGRATOR_RK4, 128, 5><<<g(128), 128, 0, s>>>(P); break;
        case 5: body_exact_kernel<B200_INTEGRATOR_RK4, 128, 6><<<g(128), 128, 0, s>>>(P); break;
        case 6: body_exact_kernel<B200_INTEGRATOR_RK4, 64, 12><<<g(64), 64, 0, s>>>(P); break;
        case 7: body_exact_kernel<B200_INTEGRATOR_RK4, 128, 3, true><<<g(128), 128, 0, s>>>(P); break;
        case 8: body_exact_kernel<B200_INTEGRATOR_RK4, 128, 2, true><<<g(128), 128, 0, s>>>(P); break;
        case 9: body_exact_kernel<B200_INTEGRATOR_RK4, 128, 4, true><<<g(128), 128, 0, s>>>(P); break;
        case 10: body_exact_kernel<B200_INTEGRATOR_RK4, 128, 3, true, 0u><<<g(128), 128, 0, s>>>(P); break;
        case 11: body_exact_kernel<B200_INTEGRATOR_RK4, 128, 5, false, 0u><<<g(128), 128, 0, s>>>(P); break;
#endif
        default: body_exact_kernel<B200_INTEGRATOR_RK4, 128, 4><<<g(128), 128, 0, s>>>(P); break; // 12: interpreter kept
        }
        return cudaGetLastError();
    }
    auto g = [&](int blk) { return (unsigned)((P.n_bodies + blk - 1) / blk); };
    // default: the kernel compiled for this effector signature; the interpreter kernel for the lists none covers
#ifdef B200_TUNE
    const int no_spec = env_int("B200_NO_SPEC", 0);
#else
    static const int no_spec = env_int("B200_NO_SPEC", 0);
#endif
    StepParams Q = P;
    static const int snake = env_int("B200_SNAKE", 1);
    if (!snake) Q.reverse = 0; // A/B switch: always walk forward
    const uint32_t sig = no_spec ? (uint32_t)SIG_GENERIC : spec_signature(Q);
    // the mass-class summary stands in for the mass only where its one use is (0 m + 0) rcp_nr(m): signature 0 with a
    // +0 gravity, no Force (write_fa) and no full trajectory sample (both form m a); the one-body-per-thread kernels
    // never read it.  B200_MASS_CLASS=0 reads every mass (A/B switch).
    static const int mass_class = env_int("B200_MASS_CLASS", 1);
    static const double pos_zero[3] = {0.0, 0.0, 0.0};
    const bool g_pos_zero = std::memcmp(Q.spec.g, pos_zero, sizeof pos_zero) == 0;
    if (!mass_class || sig != 0u || !g_pos_zero || Q.write_fa || (Q.traj_every && Q.traj_planes == 25)) Q.mass_class = nullptr;
    bool done = false;
    if (sig != SIG_GENERIC) done = rk4 ? launch_spec_sig<B200_INTEGRATOR_RK4>(Q, sig, s)
                                       : launch_spec_sig<B200_INTEGRATOR_SEMI_IMPLICIT>(Q, sig, s);
    if (!done) {
        // 128 threads x 4 CTAs/SM = 16 warps/SM at <= 128 registers
        if (rk4) BODY_FAST(B200_INTEGRATOR_RK4, 128, 4);
        else BODY_FAST(B200_INTEGRATOR_SEMI_IMPLICIT, 128, 4);
    }
    return cudaGetLastError();
}

} // namespace b200
