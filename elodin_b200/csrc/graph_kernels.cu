// sm_90a kernels of GraphQuery.edge_fold gravity (K3 of SURVEY §2.4) and the kernels that fuse it with the
// body tick (nbody_tick_fused_kernel, small_world_kernel).
//
// Why one launch per tick suffices even with body-body coupling: in the reference's RK4
// (libs/nox-py/src/integrator/rk4.rs:85-111) every stage position is x0 (+) (dt*f)*v0 — it never
// depends on a stage acceleration — so the gravity at all four stages (three distinct positions,
// f = 0, .5, 1) is a function of the tick's input state alone and needs no grid-wide synchronisation.
#include <algorithm>

#include "sixdof_tick.cuh"
#include "egm08_field.cuh"
#include "sixdof_launch.h"

namespace b200 {

// ================================================================== edge_fold gravity

// stage position of a body for slot 0/1/2 (f = 0, .5, 1): x (+) (dt*f)*v, linear part
template <bool EXACT>
__device__ __forceinline__ Vec3 stage_pos(const Vec3 &x, const Vec3 &v, double dtf)
{
    if (EXACT) return Vec3{ex::add(x.x, ex::mul(dtf, v.x)), ex::add(x.y, ex::mul(dtf, v.y)), ex::add(x.z, ex::mul(dtf, v.z))};
    return Vec3{fma(dtf, v.x, x.x), fma(dtf, v.y, x.y), fma(dtf, v.z, x.z)};
}

// Dense all-pairs (every body's out-edges are all other bodies, ascending): block =
// kBlockG source bodies of one world, targets streamed through shared memory in
// tiles; each thread folds its targets sequentially in ascending order, which is
// the reference's fold order (graph.rs:177-236) — so EXACT stays bit-exact.
static constexpr int kBlockG = 64;

// blockDim = (kBlockG, NS): thread (x, y) folds source x over all targets for stage slot y,
// so the three stage positions of a tick proceed in parallel while every fold stays sequential.
template <bool EXACT, bool RK4>
__global__ void __launch_bounds__(kBlockG * 3) graph_dense_kernel(const __grid_constant__ GraphParams G)
{
    constexpr int NS = RK4 ? 3 : 1;
    __shared__ double sx[NS][3][kBlockG];
    __shared__ double sm[kBlockG];

    const uint32_t N = G.n_entities;
    const uint32_t s0 = G.src_n ? G.src0 : 0u, sn = G.src_n ? G.src_n : N; // source rows this launch folds
    const uint32_t tiles = (sn + kBlockG - 1) / kBlockG;
    const uint32_t world = blockIdx.x / tiles;
    const uint32_t tile = blockIdx.x % tiles;
    const uint32_t tx = threadIdx.x, sl = threadIdx.y; // sl = stage slot
    const uint32_t i = s0 + tile * kBlockG + tx;
    const uint64_t wbase = (uint64_t)world * N;
    const bool active = i < s0 + sn;
    const bool newton = G.kind == B200_EFF_GRAVITY_EDGES_NEWTON;

    const double fac = sl == 0 ? 0.0 : (sl == 1 ? 0.5 : 1.0);
    const double dtf = EXACT ? ex::mul(G.dt_stage, fac) : fac * G.dt_stage;

    Vec3 xi = {0, 0, 0}, acc = {0, 0, 0};
    double mi = 0.0;
    if (active) {
        const uint64_t b = wbase + i;
        const Vec3 x = {ldp(G.pos, G.ld, 4, b), ldp(G.pos, G.ld, 5, b), ldp(G.pos, G.ld, 6, b)};
        const Vec3 v = {ldp(G.vel, G.ld, 3, b), ldp(G.vel, G.ld, 4, b), ldp(G.vel, G.ld, 5, b)};
        mi = ldp(G.ine, G.ld, 6, b);
        xi = RK4 ? stage_pos<EXACT>(x, v, dtf) : x;
    }

    for (uint32_t j0 = 0; j0 < N; j0 += kBlockG) {
        const uint32_t j = j0 + tx;
        __syncthreads();
        if (j < N) {
            const uint64_t b = wbase + j;
            const Vec3 x = {ldp(G.pos, G.ld, 4, b), ldp(G.pos, G.ld, 5, b), ldp(G.pos, G.ld, 6, b)};
            const Vec3 v = {ldp(G.vel, G.ld, 3, b), ldp(G.vel, G.ld, 4, b), ldp(G.vel, G.ld, 5, b)};
            const Vec3 p = RK4 ? stage_pos<EXACT>(x, v, dtf) : x;
            sx[sl][0][tx] = p.x; sx[sl][1][tx] = p.y; sx[sl][2][tx] = p.z;
            if (sl == 0) sm[tx] = ldp(G.ine, G.ld, 6, b);
        }
        __syncthreads();
        const uint32_t jn = min((uint32_t)kBlockG, N - j0);
        if (active) {
            for (uint32_t jj = 0; jj < jn; ++jj) {
                if (j0 + jj == i) continue;
                const double mj = sm[jj];
                const Vec3 xj = {sx[sl][0][jj], sx[sl][1][jj], sx[sl][2][jj]};
                if (EXACT) {
                    if (newton) ex::fold_newton(G.p0, xi, mi, xj, mj, acc);
                    else ex::fold_softened(G.p0, G.p1, xi, mi, xj, mj, acc);
                } else {
                    // common factor (G|K^2)*m_i applied after the loop
                    const Vec3 r = {xj.x - xi.x, xj.y - xi.y, xj.z - xi.z};
                    const double d2 = r.x * r.x + r.y * r.y + r.z * r.z + (newton ? 0.0 : G.p1);
                    const double inv = fa::rsqrt_nr(d2);
                    const double w = mj * inv * inv * inv;
                    acc.x = fma(w, r.x, acc.x); acc.y = fma(w, r.y, acc.y); acc.z = fma(w, r.z, acc.z);
                }
            }
        }
    }
    if (active) {
        const uint64_t b = wbase + i;
        const double k = EXACT ? 1.0 : G.p0 * mi;
        stp(G.gforce, G.ld, sl * 3 + 0, b, EXACT ? acc.x : k * acc.x);
        stp(G.gforce, G.ld, sl * 3 + 1, b, EXACT ? acc.y : k * acc.y);
        stp(G.gforce, G.ld, sl * 3 + 2, b, EXACT ? acc.z : k * acc.z);
    }
}

// FAST all-pairs: one warp per (source body, stage slot); lanes stride over the targets of a
// tile and keep private partial sums, a fixed xor-butterfly of warp shuffles combines them
// (summation order differs from the reference's sequential fold -> tolerance, not bit
// parity; EXACT uses graph_dense_kernel).  blockDim = (32, kFastSrc, NS): the 8 sources x 3
// slots of a CTA share one shared-memory tile of stage positions, and N = 1024, M = 1 still
// spreads over 128 CTAs x 24 warps.
static constexpr int kFastSrc = 8;

// SPLIT = true : blockDim (32, kFastSrc, NS), one warp per (source, slot)  — small batches
// SPLIT = false: blockDim (32, kFastSrc, 1),  one warp per source, NS slots — large batches
// TJ = targets per shared-memory tile: 256 (3 CTAs/SM) for big grids; 1024 for small grids, where
// the whole world of an N <= 1024 system is staged in ONE load phase instead of four dependent ones.
template <bool RK4, bool SPLIT, int TJ>
__global__ void __launch_bounds__(32 * kFastSrc * ((RK4 && SPLIT) ? 3 : 1)) graph_dense_fast_kernel(const __grid_constant__ GraphParams G)
{
    constexpr int NS = RK4 ? 3 : 1;       // stage slots of a tick
    constexpr int NW = SPLIT ? 1 : NS;    // slots folded by one warp
    constexpr int NT = 32 * kFastSrc * (SPLIT ? NS : 1);
    constexpr int kFastTJ = TJ;
    extern __shared__ double dsm[];
    double(*sx)[3][TJ] = reinterpret_cast<double(*)[3][TJ]>(dsm);
    double *sm = dsm + NS * 3 * TJ;

    const uint32_t N = G.n_entities;
    const uint32_t s0 = G.src_n ? G.src0 : 0u, sn = G.src_n ? G.src_n : N; // source rows this launch folds
    const uint32_t groups = (sn + kFastSrc - 1) / kFastSrc;
    const uint32_t world = blockIdx.x / groups;
    const uint32_t grp = blockIdx.x % groups;
    const uint32_t lane = threadIdx.x, src = threadIdx.y, sl0 = SPLIT ? threadIdx.z : 0;
    const uint32_t flat = (threadIdx.z * kFastSrc + src) * 32 + lane;
    const uint32_t i = s0 + grp * kFastSrc + src;
    const uint64_t wbase = (uint64_t)world * N;
    const bool active = i < s0 + sn;
    const bool newton = G.kind == B200_EFF_GRAVITY_EDGES_NEWTON;
    const double soft = (newton || !(G.p1 > 0.0)) ? fa::kNewtonSelfSoft : G.p1;
    auto dtf_of = [&](uint32_t sl) { return sl == 0 ? 0.0 : (sl == 1 ? 0.5 * G.dt_stage : G.dt_stage); };

    Vec3 xi[NW], acc[NW];
    double mi = 0.0;
#pragma unroll
    for (int s = 0; s < NW; ++s) { xi[s] = Vec3{0, 0, 0}; acc[s] = Vec3{0, 0, 0}; }
    if (active) {
        const uint64_t b = wbase + i;
        const Vec3 x = {ldp(G.pos, G.ld, 4, b), ldp(G.pos, G.ld, 5, b), ldp(G.pos, G.ld, 6, b)};
        const Vec3 v = {ldp(G.vel, G.ld, 3, b), ldp(G.vel, G.ld, 4, b), ldp(G.vel, G.ld, 5, b)};
        mi = ldp(G.ine, G.ld, 6, b);
#pragma unroll
        for (int s = 0; s < NW; ++s) xi[s] = RK4 ? stage_pos<false>(x, v, dtf_of(sl0 + s)) : x;
    }
    for (uint32_t j0 = 0; j0 < N; j0 += kFastTJ) {
        __syncthreads();
        // NT threads fill the (kFastTJ x NS) tile: element t -> target t % TJ, slot t / TJ
        for (uint32_t t = flat; t < kFastTJ * NS; t += NT) {
            const uint32_t jt = t % kFastTJ, st = t / kFastTJ;
            const uint32_t j = j0 + jt;
            if (j < N) {
                const uint64_t b = wbase + j;
                const Vec3 x = {ldp(G.pos, G.ld, 4, b), ldp(G.pos, G.ld, 5, b), ldp(G.pos, G.ld, 6, b)};
                Vec3 pnt = x;
                if (RK4) {
                    const Vec3 v = {ldp(G.vel, G.ld, 3, b), ldp(G.vel, G.ld, 4, b), ldp(G.vel, G.ld, 5, b)};
                    pnt = stage_pos<false>(x, v, dtf_of(st));
                }
                sx[st][0][jt] = pnt.x; sx[st][1][jt] = pnt.y; sx[st][2][jt] = pnt.z;
                if (st == 0) sm[jt] = ldp(G.ine, G.ld, 6, b);
            }
        }
        __syncthreads();
        const uint32_t jn = min((uint32_t)kFastTJ, N - j0);
        if (active) {
#pragma unroll 4
            for (uint32_t jj = lane; jj < jn; jj += 32) {
                const double mj = sm[jj]; // the self pair contributes exactly 0: r = 0 and soft > 0 (pair_fold)
#pragma unroll
                for (int s = 0; s < NW; ++s)
                    fa::pair_fold(xi[s], sx[sl0 + s][0][jj], sx[sl0 + s][1][jj], sx[sl0 + s][2][jj], mj, soft, acc[s]);
            }
        }
    }
#pragma unroll
    for (int s = 0; s < NW; ++s) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            acc[s].x += __shfl_xor_sync(0xffffffffu, acc[s].x, off);
            acc[s].y += __shfl_xor_sync(0xffffffffu, acc[s].y, off);
            acc[s].z += __shfl_xor_sync(0xffffffffu, acc[s].z, off);
        }
    }
    if (active && lane == 0) {
        const uint64_t b = wbase + i;
        const double k = G.p0 * mi;
#pragma unroll
        for (int s = 0; s < NW; ++s) {
            stp(G.gforce, G.ld, (sl0 + s) * 3 + 0, b, k * acc[s].x);
            stp(G.gforce, G.ld, (sl0 + s) * 3 + 1, b, k * acc[s].y);
            stp(G.gforce, G.ld, (sl0 + s) * 3 + 2, b, k * acc[s].z);
        }
    }
}

// FAST all-pairs for worlds of N <= TJ bodies, persistent: a CTA keeps ONE world's three stage-position tiles and
// masses in shared memory (80 KB at TJ = 1024) and folds many sources against them — the round-1 kernel re-staged
// the world for every 8 sources and its grid (one CTA per 8 sources) quantised badly against the SM count (M = 8:
// 1024 CTAs on 3 x 132 = 396 slots = 2.6 waves).  A work item is (SRC sources, one stage slot), one warp each, lanes striding
// the targets TGT at a time (SRC x TGT independent chains for the FP64 pipe); with fewer worlds than CTAs a world's
// sources are split over grid/M CTAs, otherwise a CTA walks whole worlds.  No self test (pair_fold), one third-order
// rsqrt step: 18 FP64-pipe slots per pair evaluation.
//
// FUSE: the CTA also integrates the sources it folded (all three stage slots of a source belong to one CTA), reading
// their gravity straight back after a block barrier: one launch per tick for any batch size.  Other CTAs may still be
// staging this tick's positions, so the new pose / velocity go to the second plane set (ping-pong, swapped by the host).
template <bool RK4, int TJ, int NT, int MINB, int SRC, int TGT, bool FUSE = false, uint32_t FSIG = SIG_GENERIC>
__global__ void __launch_bounds__(NT, MINB) graph_dense_world_kernel(const __grid_constant__ GraphParams G,
                                                                     const __grid_constant__ StepParams P,
                                                                     double *__restrict__ pos_out, double *__restrict__ vel_out)
{
    constexpr int NS = RK4 ? 3 : 1;
    constexpr int NWARP = NT / 32;
    extern __shared__ double dsm[];
    double(*sx)[3][TJ] = reinterpret_cast<double(*)[3][TJ]>(dsm);
    double *sm = dsm + NS * 3 * TJ;

    const uint32_t N = G.n_entities, M = G.n_worlds;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const double soft = (G.kind == B200_EFF_GRAVITY_EDGES_NEWTON || !(G.p1 > 0.0)) ? fa::kNewtonSelfSoft : G.p1;
    // CTAs per world (cpw >= 1) when the grid outnumbers the worlds; otherwise worlds stride the grid
    const uint32_t cpw = gridDim.x > M ? gridDim.x / M : 1u;
    const uint32_t part = cpw > 1 ? blockIdx.x % cpw : 0u;
    uint32_t world = cpw > 1 ? blockIdx.x / cpw : blockIdx.x;
    const uint32_t wstep = cpw > 1 ? M : gridDim.x; // cpw > 1: one world per CTA (CTAs beyond M * cpw idle)
    auto dtf_of = [&](uint32_t sl) { return sl == 0 ? 0.0 : (sl == 1 ? 0.5 * G.dt_stage : G.dt_stage); };

    for (; world < M; world += wstep) {
        const uint64_t wbase = (uint64_t)world * N;
        __syncthreads(); // the previous world's folds are done with the tiles
        for (uint32_t j = threadIdx.x; j < N; j += NT) {
            const uint64_t b = wbase + j;
            const Vec3 x = {ldp(G.pos, G.ld, 4, b), ldp(G.pos, G.ld, 5, b), ldp(G.pos, G.ld, 6, b)};
            if (RK4) {
                const Vec3 v = {ldp(G.vel, G.ld, 3, b), ldp(G.vel, G.ld, 4, b), ldp(G.vel, G.ld, 5, b)};
#pragma unroll
                for (int st = 0; st < NS; ++st) {
                    const Vec3 pnt = stage_pos<false>(x, v, dtf_of(st));
                    sx[st][0][j] = pnt.x; sx[st][1][j] = pnt.y; sx[st][2][j] = pnt.z;
                }
            } else {
                sx[0][0][j] = x.x; sx[0][1][j] = x.y; sx[0][2][j] = x.z;
            }
            sm[j] = ldp(G.ine, G.ld, 6, b);
        }
        __syncthreads();
        const uint32_t s0 = G.src_n ? G.src0 : 0u, sn = G.src_n ? G.src_n : N; // source rows this launch folds
        const uint32_t i0 = s0 + (uint32_t)((uint64_t)sn * part / cpw), i1 = s0 + (uint32_t)((uint64_t)sn * (part + 1) / cpw);
        const uint32_t n_grp = (i1 - i0 + SRC - 1) / SRC;
        const uint32_t items = n_grp * NS;
        for (uint32_t it = warp; it < items; it += NWARP) {
            const uint32_t gr = it / NS, sl = it - gr * NS;
            uint32_t is[SRC];
            Vec3 xi[SRC], acc[SRC][TGT];
#pragma unroll
            for (int a = 0; a < SRC; ++a) {
                is[a] = min(i0 + SRC * gr + a, i1 - 1u); // ragged tail: the last source again, written once
                xi[a] = Vec3{sx[sl][0][is[a]], sx[sl][1][is[a]], sx[sl][2][is[a]]};
#pragma unroll
                for (int t = 0; t < TGT; ++t) acc[a][t] = Vec3{0.0, 0.0, 0.0};
            }
            uint32_t jj = lane;
            for (; jj + 32u * (TGT - 1) < N; jj += 32u * TGT) {
#pragma unroll
                for (int t = 0; t < TGT; ++t) {
                    const uint32_t j = jj + 32u * t;
                    const double xj = sx[sl][0][j], yj = sx[sl][1][j], zj = sx[sl][2][j], mj = sm[j];
#pragma unroll
                    for (int a = 0; a < SRC; ++a) fa::pair_fold(xi[a], xj, yj, zj, mj, soft, acc[a][t]);
                }
            }
            for (; jj < N; jj += 32) {
                const double xj = sx[sl][0][jj], yj = sx[sl][1][jj], zj = sx[sl][2][jj], mj = sm[jj];
#pragma unroll
                for (int a = 0; a < SRC; ++a) fa::pair_fold(xi[a], xj, yj, zj, mj, soft, acc[a][0]);
            }
#pragma unroll
            for (int a = 0; a < SRC; ++a) {
                Vec3 r = acc[a][0];
#pragma unroll
                for (int t = 1; t < TGT; ++t) r = Vec3{r.x + acc[a][t].x, r.y + acc[a][t].y, r.z + acc[a][t].z};
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) {
                    r.x += __shfl_xor_sync(0xffffffffu, r.x, off);
                    r.y += __shfl_xor_sync(0xffffffffu, r.y, off);
                    r.z += __shfl_xor_sync(0xffffffffu, r.z, off);
                }
                if (lane == 0 && (a == 0 || is[a] != is[a - 1 < 0 ? 0 : a - 1])) {
                    const double k = G.p0 * sm[is[a]];
                    stp(G.gforce, G.ld, sl * 3 + 0, wbase + is[a], k * r.x);
                    stp(G.gforce, G.ld, sl * 3 + 1, wbase + is[a], k * r.y);
                    stp(G.gforce, G.ld, sl * 3 + 2, wbase + is[a], k * r.z);
                }
            }
        }
        if (FUSE) {
            __syncthreads(); // this CTA's gravity planes are complete and visible to its integrating threads
            for (uint32_t t = threadIdx.x; t < i1 - i0; t += NT) {
                const uint64_t b = wbase + i0 + t;
                Pose x0 = load_pose(P.pos, P.ld, b);
                Motion v0 = load_motion(P.vel, P.ld, b);
                const Inertia I = load_inertia(P.ine, P.ld, b);
                Motion a_last, f_last;
                fast_ticks<B200_INTEGRATOR_RK4, true, false, FSIG>(P, b, x0, v0, I, a_last, f_last, P.n_ticks, P.tick0, P.write_fa != 0, GravReg{});
                store_pose(pos_out, P.ld, b, x0);
                store_motion(vel_out, P.ld, b, v0);
                if (P.write_fa) {
                    store_motion(P.acc, P.ld, b, a_last);
                    store_motion(P.frc, P.ld, b, f_last);
                }
            }
        }
    }
}

// Small grids (one or a few worlds): gravity AND the body tick in ONE launch.  The CTA computes the
// three stage-slot forces of its 8 sources exactly like graph_dense_fast_kernel<RK4, SPLIT>, then 8 of
// its threads integrate those sources.  Other CTAs are still reading this tick's positions, so the
// new pose / velocity go to a second set of planes (ping-pong, swapped by the host after the launch).
// Saves the dependent second launch (~7 us of pure latency per tick at N = 1024, M = 1).
template <int TJ>
__global__ void __launch_bounds__(32 * kFastSrc * 3) nbody_tick_fused_kernel(const __grid_constant__ GraphParams G,
                                                                              const __grid_constant__ StepParams P,
                                                                              double *__restrict__ pos_out,
                                                                              double *__restrict__ vel_out)
{
    constexpr int NS = 3;
    constexpr int NT = 32 * kFastSrc * NS;
    extern __shared__ double dsm[];
    double(*sx)[3][TJ] = reinterpret_cast<double(*)[3][TJ]>(dsm);
    double *sm = dsm + NS * 3 * TJ;

    const uint32_t N = G.n_entities;
    const uint32_t groups = (N + kFastSrc - 1) / kFastSrc;
    const uint32_t world = blockIdx.x / groups;
    const uint32_t grp = blockIdx.x % groups;
    const uint32_t lane = threadIdx.x, src = threadIdx.y, sl = threadIdx.z;
    const uint32_t flat = (sl * kFastSrc + src) * 32 + lane;
    const uint32_t i = grp * kFastSrc + src;
    const uint64_t wbase = (uint64_t)world * N;
    const bool active = i < N;
    const bool newton = G.kind == B200_EFF_GRAVITY_EDGES_NEWTON;
    const double soft = (newton || !(G.p1 > 0.0)) ? fa::kNewtonSelfSoft : G.p1;
    auto dtf_of = [&](uint32_t k) { return k == 0 ? 0.0 : (k == 1 ? 0.5 * G.dt_stage : G.dt_stage); };

    Vec3 xi = {0, 0, 0}, acc = {0, 0, 0};
    double mi = 0.0;
    if (active) {
        const uint64_t b = wbase + i;
        const Vec3 x = {ldp(G.pos, G.ld, 4, b), ldp(G.pos, G.ld, 5, b), ldp(G.pos, G.ld, 6, b)};
        const Vec3 v = {ldp(G.vel, G.ld, 3, b), ldp(G.vel, G.ld, 4, b), ldp(G.vel, G.ld, 5, b)};
        mi = ldp(G.ine, G.ld, 6, b);
        xi = stage_pos<false>(x, v, dtf_of(sl));
    }
    for (uint32_t j0 = 0; j0 < N; j0 += TJ) {
        __syncthreads();
        for (uint32_t t = flat; t < TJ * NS; t += NT) {
            const uint32_t jt = t % TJ, st = t / TJ;
            const uint32_t j = j0 + jt;
            if (j < N) {
                const uint64_t b = wbase + j;
                const Vec3 x = {ldp(G.pos, G.ld, 4, b), ldp(G.pos, G.ld, 5, b), ldp(G.pos, G.ld, 6, b)};
                const Vec3 v = {ldp(G.vel, G.ld, 3, b), ldp(G.vel, G.ld, 4, b), ldp(G.vel, G.ld, 5, b)};
                const Vec3 pnt = stage_pos<false>(x, v, dtf_of(st));
                sx[st][0][jt] = pnt.x; sx[st][1][jt] = pnt.y; sx[st][2][jt] = pnt.z;
                if (st == 0) sm[jt] = ldp(G.ine, G.ld, 6, b);
            }
        }
        __syncthreads();
        const uint32_t jn = min((uint32_t)TJ, N - j0);
        if (active) {
#pragma unroll 4
            for (uint32_t jj = lane; jj < jn; jj += 32)
                fa::pair_fold(xi, sx[sl][0][jj], sx[sl][1][jj], sx[sl][2][jj], sm[jj], soft, acc);
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        acc.x += __shfl_xor_sync(0xffffffffu, acc.x, off);
        acc.y += __shfl_xor_sync(0xffffffffu, acc.y, off);
        acc.z += __shfl_xor_sync(0xffffffffu, acc.z, off);
    }
    if (active && lane == 0) {
        const uint64_t b = wbase + i;
        const double k = G.p0 * mi;
        stp(G.gforce, G.ld, sl * 3 + 0, b, k * acc.x);
        stp(G.gforce, G.ld, sl * 3 + 1, b, k * acc.y);
        stp(G.gforce, G.ld, sl * 3 + 2, b, k * acc.z);
    }
    __syncthreads(); // the CTA's gforce entries are visible to its integrating threads
    if (active && lane == 0 && sl == 0) {
        const uint64_t b = wbase + i;
        Pose x0 = load_pose(P.pos, P.ld, b);
        Motion v0 = load_motion(P.vel, P.ld, b);
        const Inertia I = load_inertia(P.ine, P.ld, b);
        Motion a_last, f_last;
        fast_ticks<B200_INTEGRATOR_RK4, true>(P, b, x0, v0, I, a_last, f_last, P.n_ticks, P.tick0, P.write_fa != 0, GravReg{});
        store_pose(pos_out, P.ld, b, x0);
        store_motion(vel_out, P.ld, b, v0);
        if (P.write_fa) {
            store_motion(P.acc, P.ld, b, a_last);
            store_motion(P.frc, P.ld, b, f_last);
        }
    }
}

// General edge list (CSR by source, spawn order inside a row): one thread per
// (world, source) gathers its targets.  Used for sparse / irregular graphs.
template <bool EXACT, bool RK4>
__global__ void __launch_bounds__(kBlockG) graph_csr_kernel(const __grid_constant__ GraphParams G)
{
    constexpr int NS = RK4 ? 3 : 1;
    const uint64_t t = (uint64_t)blockIdx.x * kBlockG + threadIdx.x;
    const uint64_t total = (uint64_t)G.n_entities * G.n_worlds;
    if (t >= total) return;
    const uint32_t i = (uint32_t)(t % G.n_entities);
    const uint64_t wbase = t - i;
    const bool newton = G.kind == B200_EFF_GRAVITY_EDGES_NEWTON;
    double dtf[3];
    dtf[0] = EXACT ? ex::mul(G.dt_stage, 0.0) : 0.0;
    dtf[1] = EXACT ? ex::mul(G.dt_stage, 0.5) : 0.5 * G.dt_stage;
    dtf[2] = EXACT ? ex::mul(G.dt_stage, 1.0) : G.dt_stage;

    const Vec3 x = {ldp(G.pos, G.ld, 4, t), ldp(G.pos, G.ld, 5, t), ldp(G.pos, G.ld, 6, t)};
    const Vec3 v = {ldp(G.vel, G.ld, 3, t), ldp(G.vel, G.ld, 4, t), ldp(G.vel, G.ld, 5, t)};
    const double mi = ldp(G.ine, G.ld, 6, t);
    Vec3 xi[NS], acc[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) { xi[s] = RK4 ? stage_pos<EXACT>(x, v, dtf[s]) : x; acc[s] = Vec3{0, 0, 0}; }

    for (uint32_t e = G.row_ptr[i]; e < G.row_ptr[i + 1]; ++e) {
        const uint64_t bj = wbase + G.col_idx[e];
        const Vec3 xj0 = {ldp(G.pos, G.ld, 4, bj), ldp(G.pos, G.ld, 5, bj), ldp(G.pos, G.ld, 6, bj)};
        const Vec3 vj = {ldp(G.vel, G.ld, 3, bj), ldp(G.vel, G.ld, 4, bj), ldp(G.vel, G.ld, 5, bj)};
        const double mj = ldp(G.ine, G.ld, 6, bj);
#pragma unroll
        for (int s = 0; s < NS; ++s) {
            const Vec3 xj = RK4 ? stage_pos<EXACT>(xj0, vj, dtf[s]) : xj0;
            if (EXACT) {
                if (newton) ex::fold_newton(G.p0, xi[s], mi, xj, mj, acc[s]);
                else ex::fold_softened(G.p0, G.p1, xi[s], mi, xj, mj, acc[s]);
            } else {
                const Vec3 r = {xj.x - xi[s].x, xj.y - xi[s].y, xj.z - xi[s].z};
                const double d2 = r.x * r.x + r.y * r.y + r.z * r.z + (newton ? 0.0 : G.p1);
                const double inv = fa::rsqrt_nr(d2);
                const double w = mj * inv * inv * inv;
                acc[s].x = fma(w, r.x, acc[s].x); acc[s].y = fma(w, r.y, acc[s].y); acc[s].z = fma(w, r.z, acc[s].z);
            }
        }
    }
    const double k = EXACT ? 1.0 : G.p0 * mi;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
        stp(G.gforce, G.ld, s * 3 + 0, t, EXACT ? acc[s].x : k * acc[s].x);
        stp(G.gforce, G.ld, s * 3 + 1, t, EXACT ? acc[s].y : k * acc[s].y);
        stp(G.gforce, G.ld, s * 3 + 2, t, EXACT ? acc[s].z : k * acc[s].z);
    }
}

// ================================================================== EGM08 stage forces
//
// GRAVITY_EGM08 (python/elodin/egm08.py) is a ~30 k-instruction series per evaluation at degree 64.  Like the edge_fold
// gravity it depends on the stage POSITION only, and the stage positions of a tick depend on (x0, v0) only, so it runs
// in its own launch before the body kernel: thread = (body, stage slot), result = 9 planes of additive stage forces the
// body kernels add where the effector sits in the list.  One arithmetic (the oracle's, IEEE operation by operation) in
// both math modes: EXACT stays bit-identical, FAST inherits it.
template <bool EXACT, bool RK4>
__global__ void __launch_bounds__(128) egm08_force_kernel(const __grid_constant__ EgmParams E)
{
    constexpr int NS = RK4 ? 3 : 1;
    const uint64_t t = (uint64_t)blockIdx.x * 128 + threadIdx.x;
    if (t >= E.n_bodies * NS) return;
    const uint64_t b = t % E.n_bodies; // slot-major: the threads of a warp share a stage slot
    const int sl = (int)(t / E.n_bodies);
    if (E.mask && !E.mask[(b + E.ent0) % E.n_entities]) return; // not a member: the body kernel skips the effector too
    const Vec3 x = {ldp(E.pos, E.ld, 4, b), ldp(E.pos, E.ld, 5, b), ldp(E.pos, E.ld, 6, b)};
    Vec3 p = x;
    if (RK4) {
        const Vec3 v = {ldp(E.vel, E.ld, 3, b), ldp(E.vel, E.ld, 4, b), ldp(E.vel, E.ld, 5, b)};
        const double fac = sl == 0 ? 0.0 : (sl == 1 ? 0.5 : 1.0);
        // the stage position exactly as the body kernel of the same math mode forms it
        p = stage_pos<EXACT>(x, v, EXACT ? ex::mul(E.dt_stage, fac) : fac * E.dt_stage);
    }
    const Vec3 g = egm08_field(E.table, (int)E.L, E.mu, E.r_ref, p, ldp(E.ine, E.ld, 6, b));
    stp(E.aforce, E.ld, sl * 3 + 0, b, g.x);
    stp(E.aforce, E.ld, sl * 3 + 1, b, g.y);
    stp(E.aforce, E.ld, sl * 3 + 2, b, g.z);
}

// ================================================================== small graph worlds: whole ticks in one warp
//
// A world of N <= 32 bodies fits in a warp: lane = body, floor(32/N) whole worlds per warp.  The edge_fold
// gravity of a tick needs the other bodies' three stage positions — functions of (x0, v0) only — which the
// lanes exchange with warp shuffles, so the state never leaves registers between ticks: one launch integrates
// n_ticks ticks (the generic route is two launches and a round trip of the 9 gravity planes through HBM per
// tick).  Every lane folds its out-edges sequentially in CSR (= spawn) order with the same ex:: functions as
// graph_dense_kernel / graph_csr_kernel, then runs the same tick function as body_exact_kernel — EXACT stays
// bit-identical to the oracle.  FAST folds sequentially too (no tree), with the FAST kernels' arithmetic.
// SIG: SIG_GRAPH when the edge_fold gravity is the only effector (the FAST tick is then compiled for exactly that),
// SIG_GENERIC otherwise (the run-time interpreter)
template <bool EXACT, int INTEG, int MINB, uint32_t SIG = SIG_GENERIC>
__global__ void __launch_bounds__(128, MINB) small_world_kernel(const __grid_constant__ GraphParams G,
                                                          const __grid_constant__ StepParams P)
{
    constexpr bool RK4 = INTEG == B200_INTEGRATOR_RK4;
    constexpr int NS = RK4 ? 3 : 1;
    constexpr unsigned FULL = 0xffffffffu;
    const uint32_t N = G.n_entities;
    const uint32_t wpw = 32u / N; // worlds per warp
    const uint32_t lane = threadIdx.x & 31u;
    const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t wl = lane / N, ent = lane - wl * N;
    const uint64_t world = warp * wpw + wl;
    const bool live = wl < wpw && world < G.n_worlds;
    const uint64_t b = live ? world * N + ent : 0;
    const uint32_t lane0 = lane - ent; // first lane of this lane's world
    const bool newton = G.kind == B200_EFF_GRAVITY_EDGES_NEWTON;

    Pose x0 = {{0.0, 0.0, 0.0, 1.0}, {0.0, 0.0, 0.0}};
    Motion v0 = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}}, a_out = v0, f_out = v0;
    Inertia I = {{1.0, 1.0, 1.0}, 1.0};
    uint32_t e0 = 0, deg = 0;
    if (live) {
        x0 = load_pose(P.pos, P.ld, b);
        v0 = load_motion(P.vel, P.ld, b);
        if (EXACT) a_out = load_motion(P.acc, P.ld, b);
        I = load_inertia(P.ine, P.ld, b);
        e0 = G.row_ptr[ent];
        deg = G.row_ptr[ent + 1] - e0;
    }
    GravReg g;
    g.g0 = g.g1 = g.g2 = Vec3{0.0, 0.0, 0.0};
    g.has = deg != 0;

    for (uint32_t t = 0; t < P.n_ticks; ++t) {
        // stage positions of this body and the running folds, one per distinct stage position
        Vec3 p[NS], acc[NS];
#pragma unroll
        for (int s = 0; s < NS; ++s) {
            const double fac = s == 0 ? 0.0 : (s == 1 ? 0.5 : 1.0);
            const double dtf = EXACT ? ex::mul(G.dt_stage, fac) : fac * G.dt_stage;
            p[s] = RK4 ? stage_pos<EXACT>(x0.x, v0.lin, dtf) : x0.x;
            acc[s] = Vec3{0.0, 0.0, 0.0};
        }
        for (uint32_t k = 0; k < G.max_deg; ++k) { // warp-uniform trip count: every lane takes part in the shuffles
            const bool on = k < deg;
            const uint32_t src = lane0 + (on ? G.col_idx[e0 + k] : ent);
            const double mj = __shfl_sync(FULL, I.m, src);
#pragma unroll
            for (int s = 0; s < NS; ++s) {
                const Vec3 xj = {__shfl_sync(FULL, p[s].x, src), __shfl_sync(FULL, p[s].y, src), __shfl_sync(FULL, p[s].z, src)};
                if (!on) continue;
                if (EXACT) {
                    if (newton) ex::fold_newton(G.p0, p[s], I.m, xj, mj, acc[s]);
                    else ex::fold_softened(G.p0, G.p1, p[s], I.m, xj, mj, acc[s]);
                } else {
                    const Vec3 r = {xj.x - p[s].x, xj.y - p[s].y, xj.z - p[s].z};
                    const double d2 = fma(r.x, r.x, fma(r.y, r.y, fma(r.z, r.z, newton ? 0.0 : G.p1)));
                    const double inv = fa::rsqrt_nr(d2);
                    const double w = mj * inv * inv * inv;
                    acc[s].x = fma(w, r.x, acc[s].x); acc[s].y = fma(w, r.y, acc[s].y); acc[s].z = fma(w, r.z, acc[s].z);
                }
            }
        }
        const double kf = EXACT ? 1.0 : G.p0 * I.m; // FAST: common factor (G | K^2) * m_i applied once
        g.g0 = EXACT ? acc[0] : Vec3{kf * acc[0].x, kf * acc[0].y, kf * acc[0].z};
        if (RK4) {
            g.g1 = EXACT ? acc[NS - 2] : Vec3{kf * acc[NS - 2].x, kf * acc[NS - 2].y, kf * acc[NS - 2].z};
            g.g2 = EXACT ? acc[NS - 1] : Vec3{kf * acc[NS - 1].x, kf * acc[NS - 1].y, kf * acc[NS - 1].z};
        }
        if (!live) continue;
        if (EXACT) {
            exact_tick<INTEG, true>(P, b, x0, v0, a_out, f_out, I, g);
            uint64_t slot;
            if (traj_due(P, P.tick0 + t + 1, slot)) {
                traj_store_state(P, b, slot, x0, v0);
                if (P.traj_planes == 25) traj_store_af(P, b, slot, a_out, f_out);
            }
        } else {
            fast_ticks<INTEG, true, true, SIG>(P, b, x0, v0, I, a_out, f_out, 1u, P.tick0 + t, P.write_fa && t + 1 == P.n_ticks, g);
        }
    }
    if (!live) return;
    store_pose(P.pos, P.ld, b, x0);
    store_motion(P.vel, P.ld, b, v0);
    if (P.write_fa) {
        store_motion(P.acc, P.ld, b, a_out);
        store_motion(P.frc, P.ld, b, f_out);
    }
}

// ================================================================== launchers

cudaError_t launch_graph_force(const GraphParams &G, int math_mode, bool dense, cudaStream_t s)
{
    const bool exact = math_mode == B200_MATH_EXACT;
    const bool rk4 = G.integrator == B200_INTEGRATOR_RK4;
    if (G.n_entities == 0 || G.n_worlds == 0) return cudaSuccess;
    if (dense) {
        const unsigned n_src = G.src_n ? G.src_n : G.n_entities; // sources folded by this launch
        const unsigned tiles = (n_src + kBlockG - 1) / kBlockG;
        const unsigned grid = tiles * G.n_worlds;
        static const int gcfg = [] { const char *e = getenv("B200_GRAPH_CFG"); return e ? atoi(e) : 1; }();
        const dim3 blk3(kBlockG, 3), blk1(kBlockG, 1);
        if (exact) { if (rk4) graph_dense_kernel<true, true><<<grid, blk3, 0, s>>>(G); else graph_dense_kernel<true, false><<<grid, blk1, 0, s>>>(G); }
        else if (gcfg == 0) { if (rk4) graph_dense_kernel<false, true><<<grid, blk3, 0, s>>>(G); else graph_dense_kernel<false, false><<<grid, blk1, 0, s>>>(G); }
        else {
            if (gcfg == 1 && G.n_entities <= 1024 && G.n_entities >= 64) {
                // worlds that fit one shared-memory tile set: persistent world-resident kernel
                int dev = 0, sms = (int)kNumSMs;
                cudaGetDevice(&dev);
                cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
                auto launch_world = [&](auto kern, int nt, int minb, int src) -> cudaError_t {
                    const unsigned slots = (unsigned)minb * (unsigned)sms;
                    unsigned grid_w;
                    if (G.n_worlds >= slots) grid_w = slots;
                    else {
                        // few worlds: as many CTAs per world as the SMs allow, down to four busy warps per CTA (latency,
                        // not throughput, is the price of a tick then)
                        const unsigned items = (n_src + src - 1) / src * (rk4 ? 3u : 1u), warps = (unsigned)nt / 32u;
                        const unsigned busy = std::min(warps, 4u); // one busy warp per FP64 pipe when there is room to spread
                        const unsigned cpw = std::max(1u, std::min(slots / G.n_worlds, (items + busy - 1) / busy));
                        grid_w = cpw * G.n_worlds;
                    }
                    const size_t smem = ((rk4 ? 3 : 1) * 3 + 1) * 1024 * sizeof(double);
                    const cudaError_t e = ensure_dynamic_smem(kern, smem);
                    if (e != cudaSuccess) return e;
                    kern<<<grid_w, nt, smem, s>>>(G, StepParams{}, nullptr, nullptr);
                    return cudaGetLastError();
                };
#ifdef B200_TUNE
                if (rk4) switch (env_int("B200_WORLD_CFG", 0)) {
                case 1: return launch_world(graph_dense_world_kernel<true, 1024, 256, 2, 2, 2>, 256, 2, 2);
                case 2: return launch_world(graph_dense_world_kernel<true, 1024, 256, 2, 1, 2>, 256, 2, 1);
                case 3: return launch_world(graph_dense_world_kernel<true, 1024, 256, 2, 1, 8>, 256, 2, 1);
                case 4: return launch_world(graph_dense_world_kernel<true, 1024, 512, 1, 1, 4>, 512, 1, 1);
                case 5: return launch_world(graph_dense_world_kernel<true, 1024, 384, 2, 1, 4>, 384, 2, 1);
                case 6: return launch_world(graph_dense_world_kernel<true, 1024, 256, 2, 3, 2>, 256, 2, 3);
                case 7: return launch_world(graph_dense_world_kernel<true, 1024, 128, 2, 1, 4>, 128, 2, 1);
                case 8: return launch_world(graph_dense_world_kernel<true, 1024, 256, 2, 1, 4>, 256, 2, 1);
                case 9: return launch_world(graph_dense_world_kernel<true, 1024, 512, 1, 3, 2>, 512, 1, 3);
                case 10: return launch_world(graph_dense_world_kernel<true, 1024, 512, 1, 4, 1>, 512, 1, 4);
                case 11: return launch_world(graph_dense_world_kernel<true, 1024, 1024, 1, 2, 1>, 1024, 1, 2);
                case 12: return launch_world(graph_dense_world_kernel<true, 1024, 768, 1, 2, 2>, 768, 1, 2);
                case 13: return launch_world(graph_dense_world_kernel<true, 1024, 512, 1, 2, 4>, 512, 1, 2);
                case 14: return launch_world(graph_dense_world_kernel<true, 1024, 1024, 1, 1, 2>, 1024, 1, 1);
                default: break;
                }
#endif
                // default shapes: one 512-thread CTA per SM stages each world
                // once per SM.  Big batches (>= 8 rounds of four-source items per resident warp) fold four sources per
                // item — four chains that share every target load: 0.81 of the DFMA issue rate; small batches keep
                // two sources x two targets so that the item count still divides over the warps (M = 8: 0.55)
                const unsigned long long items4 = (unsigned long long)((n_src + 3) / 4) * (rk4 ? 3u : 1u) * G.n_worlds;
                const bool big = items4 >= 8ull * 16ull * (unsigned)sms;
                if (rk4) return big ? launch_world(graph_dense_world_kernel<true, 1024, 512, 1, 4, 1>, 512, 1, 4)
                                    : launch_world(graph_dense_world_kernel<true, 1024, 512, 1, 2, 2>, 512, 1, 2);
                return big ? launch_world(graph_dense_world_kernel<false, 1024, 512, 1, 4, 1>, 512, 1, 4)
                           : launch_world(graph_dense_world_kernel<false, 1024, 512, 1, 2, 2>, 512, 1, 2);
            }
            const unsigned gridf = ((n_src + kFastSrc - 1) / kFastSrc) * G.n_worlds;
            // few CTAs: split the stage slots over warps to fill the machine; many CTAs: keep
            // 3 slots per warp (more ILP per lane, 3 CTAs/SM) — measured on N = 1024, M = 1 / 8
            const bool split = gcfg == 2 || (gcfg == 1 && gridf < 3u * kNumSMs);
            constexpr size_t smem256 = (3 * 3 + 1) * 256 * sizeof(double), smem1024 = (3 * 3 + 1) * 1024 * sizeof(double);
            if (!rk4) graph_dense_fast_kernel<false, false, 256><<<gridf, dim3(32, kFastSrc, 1), smem256, s>>>(G);
            else if (split) {
                const cudaError_t e = ensure_dynamic_smem(graph_dense_fast_kernel<true, true, 1024>, smem1024);
                if (e != cudaSuccess) return e;
                graph_dense_fast_kernel<true, true, 1024><<<gridf, dim3(32, kFastSrc, 3), smem1024, s>>>(G);
            } else graph_dense_fast_kernel<true, false, 256><<<gridf, dim3(32, kFastSrc, 1), smem256, s>>>(G);
        }
    } else {
        const uint64_t total = (uint64_t)G.n_entities * G.n_worlds;
        const unsigned grid = (unsigned)((total + kBlockG - 1) / kBlockG);
        if (exact) { if (rk4) graph_csr_kernel<true, true><<<grid, kBlockG, 0, s>>>(G); else graph_csr_kernel<true, false><<<grid, kBlockG, 0, s>>>(G); }
        else { if (rk4) graph_csr_kernel<false, true><<<grid, kBlockG, 0, s>>>(G); else graph_csr_kernel<false, false><<<grid, kBlockG, 0, s>>>(G); }
    }
    return cudaGetLastError();
}

cudaError_t launch_egm08_force(const EgmParams &E, int math_mode, cudaStream_t s)
{
    if (E.n_bodies == 0) return cudaSuccess;
    const bool rk4 = E.integrator == B200_INTEGRATOR_RK4;
    const uint64_t threads = E.n_bodies * (rk4 ? 3u : 1u);
    const unsigned grid = (unsigned)((threads + 127) / 128);
    if (math_mode == B200_MATH_EXACT) {
        if (rk4) egm08_force_kernel<true, true><<<grid, 128, 0, s>>>(E);
        else egm08_force_kernel<true, false><<<grid, 128, 0, s>>>(E);
    } else {
        if (rk4) egm08_force_kernel<false, true><<<grid, 128, 0, s>>>(E);
        else egm08_force_kernel<false, false><<<grid, 128, 0, s>>>(E);
    }
    return cudaGetLastError();
}

bool nbody_fused_applicable(const GraphParams &G, int math_mode, bool dense)
{
    if (math_mode != B200_MATH_FAST || !dense || G.integrator != B200_INTEGRATOR_RK4) return false;
    static const int fcfg = [] { const char *e = getenv("B200_NBODY_FUSED"); return e ? atoi(e) : 1; }();
    if (fcfg == 0) return false;
    const unsigned gridf = ((G.n_entities + kFastSrc - 1) / kFastSrc) * G.n_worlds;
    if (gridf < 3u * kNumSMs) return true; // small grids: one launch per tick (pair kernel for 64..1024 bodies, nbody_tick_fused_kernel otherwise)
    // worlds that fit the persistent kernel's tile set: fused at any batch size (one launch per tick instead of two,
    // identical bits; B200_NBODY_FUSED=2 keeps the two-launch route)
    return fcfg != 2 && G.n_entities >= 64 && G.n_entities <= 1024;
}

cudaError_t launch_nbody_tick_fused(const GraphParams &G, const StepParams &P, double *pos_out, double *vel_out, cudaStream_t s)
{
    constexpr size_t smem = (3 * 3 + 1) * 1024 * sizeof(double);
    const unsigned gridf = ((G.n_entities + kFastSrc - 1) / kFastSrc) * G.n_worlds;
    // One to three worlds too: a world's (source pair, slot) items spread over as many CTAs as give every warp one item
    // (scripts/tune_nbody_small.py compares the routes; same bits); B200_NBODY_WORLD_MIN=396 restores the small-grid kernel below 3 x 132 split-kernel CTAs
    static const unsigned world_min = (unsigned)env_int("B200_NBODY_WORLD_MIN", 0);
    static const unsigned world_rounds = (unsigned)std::max(1, env_int("B200_NBODY_WORLD_ROUNDS", 1));
    if (gridf >= world_min && G.n_entities >= 64 && G.n_entities <= 1024) {
        // the persistent world-resident kernel with the integration fused in (same shapes as launch_graph_force picks)
        int dev = 0, sms = (int)kNumSMs;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        const unsigned long long items4 = (unsigned long long)((G.n_entities + 3) / 4) * 3u * G.n_worlds;
        const bool big = items4 >= 8ull * 16ull * (unsigned)sms;
        const unsigned src = big ? 4u : 2u, slots = (unsigned)sms, warps = 16u;
        unsigned grid_w;
        if (G.n_worlds >= slots) grid_w = slots;
        else {
            const unsigned items = (G.n_entities + src - 1) / src * 3u;
            // few worlds: spread a world's items over the SMs until a CTA keeps only four warps busy — one per FP64 pipe
            static const unsigned spread = (unsigned)std::max(1, env_int("B200_NBODY_WORLD_SPREAD", 4));
            const unsigned per_cta = world_rounds * std::min(warps, spread);
            grid_w = std::max(1u, std::min(slots / G.n_worlds, (items + per_cta - 1) / per_cta)) * G.n_worlds;
        }
        // gravity is usually the whole effector list (n-body): the integration is then compiled for that signature
        const bool only_graph = P.n_eff == 1 && !P.eff[0].mask;
        auto kern = big ? (only_graph ? graph_dense_world_kernel<true, 1024, 512, 1, 4, 1, true, SIG_GRAPH>
                                      : graph_dense_world_kernel<true, 1024, 512, 1, 4, 1, true, SIG_GENERIC>)
                        : (only_graph ? graph_dense_world_kernel<true, 1024, 512, 1, 2, 2, true, SIG_GRAPH>
                                      : graph_dense_world_kernel<true, 1024, 512, 1, 2, 2, true, SIG_GENERIC>);
        const cudaError_t e = ensure_dynamic_smem(kern, smem);
        if (e != cudaSuccess) return e;
        kern<<<grid_w, 512, smem, s>>>(G, P, pos_out, vel_out);
        return cudaGetLastError();
    }
    const cudaError_t e = ensure_dynamic_smem(nbody_tick_fused_kernel<1024>, smem);
    if (e != cudaSuccess) return e;
    nbody_tick_fused_kernel<1024><<<gridf, dim3(32, kFastSrc, 3), smem, s>>>(G, P, pos_out, vel_out);
    return cudaGetLastError();
}

bool small_world_applicable(const GraphParams &G, int math_mode)
{
    // faster than the two-launch route over the whole range a warp can
    // hold, in both arithmetic modes (N = 3: 53x FAST / 4.4x EXACT; N = 32: 3.6x / 1.35x)
    (void)math_mode;
    static const int cfg = [] { const char *e = getenv("B200_SMALL_WORLD"); return e ? atoi(e) : 1; }();
    return cfg != 0 && G.n_entities >= 1 && G.n_entities <= 32;
}

template <int MINB>
static void launch_small_world_cfg(const GraphParams &G, const StepParams &P, int math_mode, unsigned grid, cudaStream_t s)
{
    const bool rk4 = G.integrator == B200_INTEGRATOR_RK4;
    if (math_mode == B200_MATH_EXACT) {
        if (rk4) small_world_kernel<true, B200_INTEGRATOR_RK4, MINB><<<grid, 128, 0, s>>>(G, P);
        else small_world_kernel<true, B200_INTEGRATOR_SEMI_IMPLICIT, MINB><<<grid, 128, 0, s>>>(G, P);
    } else {
        const bool only_graph = P.n_eff == 1 && !P.eff[0].mask; // three-body / n-body: gravity is the whole effector list
        if (only_graph) {
            if (rk4) small_world_kernel<false, B200_INTEGRATOR_RK4, MINB, SIG_GRAPH><<<grid, 128, 0, s>>>(G, P);
            else small_world_kernel<false, B200_INTEGRATOR_SEMI_IMPLICIT, MINB, SIG_GRAPH><<<grid, 128, 0, s>>>(G, P);
        } else if (rk4) small_world_kernel<false, B200_INTEGRATOR_RK4, MINB><<<grid, 128, 0, s>>>(G, P);
        else small_world_kernel<false, B200_INTEGRATOR_SEMI_IMPLICIT, MINB><<<grid, 128, 0, s>>>(G, P);
    }
}

cudaError_t launch_small_world(const GraphParams &G, const StepParams &P, int math_mode, cudaStream_t s)
{
    if (G.n_entities == 0 || G.n_worlds == 0) return cudaSuccess;
    const uint32_t wpw = 32u / G.n_entities;
    const uint64_t warps = ((uint64_t)G.n_worlds + wpw - 1) / wpw;
    const unsigned grid = (unsigned)((warps + 3) / 4); // 4 warps per CTA
    // resident CTAs per SM the register allocation is bounded for (B200_SMALL_WORLD_CFG = 2 | 3 | 4): the kernel
    // is latency-bound, 16 warps/SM at 128 registers (a few spilled doubles) beat 8 warps at 196 by 1.3-1.45x
    static const int cfg = [] { const char *e = getenv("B200_SMALL_WORLD_CFG"); return e ? atoi(e) : 4; }();
    switch (cfg) {
    case 2: launch_small_world_cfg<2>(G, P, math_mode, grid, s); break;
    case 3: launch_small_world_cfg<3>(G, P, math_mode, grid, s); break;
    default: launch_small_world_cfg<4>(G, P, math_mode, grid, s); break;
    }
    return cudaGetLastError();
}


} // namespace b200
