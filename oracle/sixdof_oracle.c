/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.  See sixdof_oracle.h for the parity
 * status ("pinned" for the free-body / three-body / rocket / ball paths).
 *
 * Plain-C restatement of the reference arithmetic, one IEEE operation per
 * source operation, in the reference's evaluation order.  Build with
 *   gcc -O2 -ffp-contract=off -fno-fast-math      (oracle/Makefile)
 * so no multiply-add is ever contracted.
 */
#define _GNU_SOURCE /* sched_getaffinity / CPU_COUNT for orc_max_threads */
#include "sixdof_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <sched.h>
#include <stdio.h>
#include <unistd.h>

/* ---- libs/nox/src/quaternion.rs:268-281 — Mul for &Quaternion; storage [i,j,k,w]
 * (quaternion.rs:100,134-138).  Rust `a + b + c - d` associates left to right. */
void orc_qmul(const double l[4], const double r[4], double out[4])
{
    const double li = l[0], lj = l[1], lk = l[2], lw = l[3];
    const double ri = r[0], rj = r[1], rk = r[2], rw = r[3];
    const double i = ((lw * ri + li * rw) + lj * rk) - lk * rj;
    const double j = ((lw * rj - li * rk) + lj * rw) + lk * ri;
    const double k = ((lw * rk + li * rj) - lj * ri) + lk * rw;
    const double w = ((lw * rw - li * ri) - lj * rj) - lk * rk;
    out[0] = i; out[1] = j; out[2] = k; out[3] = w;
}

/* 4-element dot.  dot_general of two rank-1 tensors is a left fold from 0.0
 * (libs/cranelift-mlir/src/lower.rs:9357-9366): ((a0*b0 + a1*b1) + a2*b2) + a3*b3. */
static double dot4_plain(const double a[4], const double b[4])
{
    return ((a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]) + a[3] * b[3];
}

/* The same fold as the reference JIT's *pointer-ABI* runtime evaluates it:
 * tensor_matmul_f64 (libs/cranelift-mlir/src/tensor_rt.rs:1141-1163) uses
 * `d.algebraic_add(a.algebraic_mul(b))`, which the Rust compiler contracts to a
 * fused multiply-add on hosts that have one.  The reference's golden rocket
 * telemetry was produced that way (see orc_set_dot_mode). */
static double dot4_fused(const double a[4], const double b[4])
{
    double d = a[0] * b[0];
    d = fma(a[1], b[1], d);
    d = fma(a[2], b[2], d);
    d = fma(a[3], b[3], d);
    return d;
}

/* 0 = ORC_DOT_PLAIN (canonical: no contraction anywhere).
 * 1 = ORC_DOT_GOLDEN_HOST: quaternion norm_squared inside the Rust-defined
 *     systems that nox inlines into `main` (the (+) of spatial.rs:530-549 and
 *     calc_accel, six_dof.rs:137-146) is FMA-contracted, while Python @el.map
 *     effectors (private scalar-ABI functions) stay plain.  With this mode the
 *     oracle reproduces scripts/ci/baseline/rocket-csv bit for bit (100/100
 *     one-step predictions); plain mode differs from it by <= 1e-15 relative. */
static int g_dot_mode = 0;
void orc_set_dot_mode(int mode) { g_dot_mode = mode; }
int orc_get_dot_mode(void) { return g_dot_mode; }

static double dot4_sys(const double a[4], const double b[4])
{
    return g_dot_mode ? dot4_fused(a, b) : dot4_plain(a, b);
}

static double dot3(const double a[3], const double b[3])
{
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2];
}

typedef double (*dot4_fn)(const double *, const double *);

/* libs/nox/src/quaternion.rs:141-155 — conjugate() / norm_squared(); no unit-norm assumption */
static void qinv_with(dot4_fn dot, const double q[4], double out[4])
{
    const double n2 = dot(q, q);
    out[0] = -q[0] / n2;
    out[1] = -q[1] / n2;
    out[2] = -q[2] / n2;
    out[3] = q[3] / n2;
}

/* libs/nox/src/quaternion.rs:283-305 — Quaternion * Vector3: (q * [v,0]) * q.inverse(),
 * the inverse is recomputed on every call. */
static void qrot_with(dot4_fn dot, const double q[4], const double v[3], double out[3])
{
    const double vq[4] = {v[0], v[1], v[2], 0.0};
    double inv[4], t[4], r[4];
    qinv_with(dot, q, inv);
    orc_qmul(q, vq, t);
    orc_qmul(t, inv, r);
    out[0] = r[0]; out[1] = r[1]; out[2] = r[2];
}

/* libs/nox/src/quaternion.rs:147-149 + vector.rs:115-122 — q / sqrt(dot(q,q)) */
static void qnormalize_with(dot4_fn dot, const double q[4], double out[4])
{
    const double n = sqrt(dot(q, q));
    out[0] = q[0] / n; out[1] = q[1] / n; out[2] = q[2] / n; out[3] = q[3] / n;
}

/* public primitives: canonical (plain) arithmetic */
void orc_qinv(const double q[4], double out[4]) { qinv_with(dot4_plain, q, out); }
void orc_qrot(const double q[4], const double v[3], double out[3]) { qrot_with(dot4_plain, q, v, out); }
void orc_qnormalize(const double q[4], double out[4]) { qnormalize_with(dot4_plain, q, out); }

/* libs/nox/src/spatial.rs:530-549 — SpatialTransform + SpatialMotion:
 * h = [omega/2, 0]; q' = normalize(q + h*q); x' = x + v */
void orc_transform_add_motion(const double pos[7], const double m[6], double out[7])
{
    const double h[4] = {m[0] / 2.0, m[1] / 2.0, m[2] / 2.0, 0.0};
    double hq[4], s[4];
    orc_qmul(h, pos, hq);
    s[0] = pos[0] + hq[0]; s[1] = pos[1] + hq[1]; s[2] = pos[2] + hq[2]; s[3] = pos[3] + hq[3];
    qnormalize_with(dot4_sys, s, out);
    out[4] = pos[4] + m[3];
    out[5] = pos[5] + m[4];
    out[6] = pos[6] + m[5];
}

/* libs/nox-py/src/six_dof.rs:137-146 calc_accel, with
 * Quaternion * SpatialForce (spatial.rs:587-593), SpatialForce / SpatialInertia
 * (spatial.rs:353-361) and Quaternion * SpatialMotion (spatial.rs:571-577). */
void orc_calc_accel(const double pos[7], const double force[6], const double inertia[7], double accel[6])
{
    double qi[4], tb[3], fb[3], ab_ang[3], ab_lin[3];
    qinv_with(dot4_sys, pos, qi);              /* q.inverse() */
    qrot_with(dot4_sys, qi, force, tb);        /* body-frame torque */
    qrot_with(dot4_sys, qi, force + 3, fb);    /* body-frame force  */
    ab_lin[0] = fb[0] / inertia[6]; ab_lin[1] = fb[1] / inertia[6]; ab_lin[2] = fb[2] / inertia[6];
    ab_ang[0] = tb[0] / inertia[0]; ab_ang[1] = tb[1] / inertia[1]; ab_ang[2] = tb[2] / inertia[2];
    qrot_with(dot4_sys, pos, ab_ang, accel);
    qrot_with(dot4_sys, pos, ab_lin, accel + 3);
}

/* ------------------------------------------------------------------ effectors */

static void cross3(const double a[3], const double b[3], double o[3])
{
    /* jnp.cross / libs/nox/src/vector.rs:84-91 */
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

/* examples/ball/sim.py:56-58, examples/rocket/main.py:292-294:
 *   f + SpatialForce(linear=g * inertia.mass())   (torque part adds +0.0) */
static void eff_gravity_const(const orc_effector *e, const double inertia[7], double F[6])
{
    const double m = inertia[6];
    F[0] = F[0] + 0.0; F[1] = F[1] + 0.0; F[2] = F[2] + 0.0;
    F[3] = F[3] + e->p[0] * m;
    F[4] = F[4] + e->p[1] * m;
    F[5] = F[5] + e->p[2] * m;
}

/* examples/ball/sim.py:99-116 apply_drag; calculate_drag = 0.5*(Cd*r*V**2*A).
 * Cd*r is a Python constant (p[0]); returns SpatialForce(linear=...) => torque 0. */
static void eff_drag_quadratic(const orc_effector *e, const double *wind, const double vel[6], double F[6])
{
    double fl[3];
    const double w0 = wind ? wind[0] : 0.0, w1 = wind ? wind[1] : 0.0, w2 = wind ? wind[2] : 0.0;
    fl[0] = w0 - vel[3]; fl[1] = w1 - vel[4]; fl[2] = w2 - vel[5];
    const double speed = sqrt(dot3(fl, fl));
    /* width-5 column: [wind(3), Cd*rho, area] per body (Monte-Carlo worlds with their own drag) */
    const double cd_rho = (wind && e->column_width == 5) ? wind[3] : e->p[0];
    const double area = (wind && e->column_width == 5) ? wind[4] : e->p[1];
    const double drag = 0.5 * ((cd_rho * (speed * speed)) * area);
    const double d0 = fl[0] / speed, d1 = fl[1] / speed, d2 = fl[2] / speed;
    F[0] = 0.0; F[1] = 0.0; F[2] = 0.0;
    F[3] = F[3] + drag * d0;
    F[4] = F[4] + drag * d1;
    F[5] = F[5] + drag * d2;
}

/* examples/rocket/main.py:429-431: f + SpatialForce(linear=p.angular() @ axis * thrust) */
static void eff_thrust_body(const orc_effector *e, const double *thrust, const double pos[7], double F[6])
{
    double d[3];
    const double t = thrust ? thrust[0] : 0.0;
    orc_qrot(pos, e->p, d);
    F[0] = F[0] + 0.0; F[1] = F[1] + 0.0; F[2] = F[2] + 0.0;
    F[3] = F[3] + d[0] * t;
    F[4] = F[4] + d[1] * t;
    F[5] = F[5] + d[2] * t;
}

/* examples/rocket/main.py:407-413: f + p.angular() @ f_aero   (column [tau, f])
 * examples/falcon9/sim.py:659-672: force + SpatialForce(linear=q@total[:3], torque=q@total[3:]) */
static void eff_wrench_body(const orc_effector *e, const double *wr, const double pos[7], double F[6])
{
    double tw[3], fw[3];
    const double zero[6] = {0, 0, 0, 0, 0, 0};
    if (!wr) wr = zero;
    if (e->flags & ORC_FLAG_WRENCH_LINEAR_FIRST) {
        orc_qrot(pos, wr + 3, tw);
        orc_qrot(pos, wr, fw);
    } else {
        orc_qrot(pos, wr, tw);
        orc_qrot(pos, wr + 3, fw);
    }
    F[0] = F[0] + tw[0]; F[1] = F[1] + tw[1]; F[2] = F[2] + tw[2];
    F[3] = F[3] + fw[0]; F[4] = F[4] + fw[1]; F[5] = F[5] + fw[2];
}

/* World-frame wrench column [tau(3), f(3)] added to Force: `force + SpatialForce(...)` of effectors whose value is
 * computed outside six_dof — examples/cube-sat/main.py:516-527 (gravity_effector: force + SpatialForce(linear=f)),
 * examples/drone/sim.py:99-103 (f + SpatialForce(linear=drag)). */
static void eff_wrench_world(const double *wr, double F[6])
{
    if (!wr) return;
    for (int k = 0; k < 6; ++k) F[k] = F[k] + wr[k];
}

/* Reaction-wheel edge fold, examples/cube-sat/main.py:492-505:
 *   rw_force.edge_fold(.., el.SpatialForce(), lambda f, pos, force: f + SpatialForce(torque=pos.angular() @ force.torque()))
 * per body, over its out-edges in spawn order; the column carries the K wheel torques of the body, [tau_1 .. tau_K]. */
static void eff_torque_body_fold(const orc_effector *e, const double *col, const double pos[7], double F[6])
{
    if (!col) return;
    double acc[6] = {0, 0, 0, 0, 0, 0}; /* edge_fold init: SpatialForce() */
    const uint32_t K = e->column_width / 3;
    for (uint32_t k = 0; k < K; ++k) {
        double t[3];
        orc_qrot(pos, col + 3 * k, t);
        acc[0] = acc[0] + t[0]; acc[1] = acc[1] + t[1]; acc[2] = acc[2] + t[2];
        acc[3] = acc[3] + 0.0; acc[4] = acc[4] + 0.0; acc[5] = acc[5] + 0.0;
    }
    /* the fold's result IS the Force column of the bodies that own an edge (edge_fold writes el.Force) */
    for (int k = 0; k < 6; ++k) F[k] = acc[k];
}

/* x^6, correctly rounded but for results within ~2^-100 of a rounding boundary: x^2, x^4 and x^6 as double-double
 * products (FMA error terms), rounded once.  pow() is not correctly rounded, and libm implementations (the host's, the
 * GPU's) round differently; the EXACT kernel (sixdof_tick.cuh:pow6_exact) runs this same operation sequence. */
static double pow6(double x)
{
    const double s = x * x, se = fma(x, x, -s);
    const double q = s * s, qe = fma(s, s, -q) + (2.0 * s) * se;
    const double p = q * s;
    if (!isfinite(p)) return p;
    const double pe = fma(q, s, -p) + ((q * se) + (qe * s));
    return p + pe;
}

/* libs/nox-py/python/elodin/j2.py:5-29 (J2.compute_field), applied as `force + SpatialForce(linear=field)`.
 * p = [mu, J2, r_ref].  Integer powers follow lax.integer_pow's square-and-multiply (x**5 = x * (x^2)^2,
 * x**4 = (x^2)^2); `norm**6.0` has a float exponent and lowers to pow(), evaluated here correctly rounded (pow6).
 * Parity unpinned: no golden uses J2. */
static void eff_gravity_j2(const orc_effector *e, const double pos[7], const double inertia[7], double F[6])
{
    const double mu = e->p[0], J2 = e->p[1], r_ref = e->p[2];
    const double *r = pos + 4;
    const double m = inertia[6], z = r[2];
    const double norm = sqrt(dot3(r, r));
    const double e_r[3] = {r[0] / norm, r[1] / norm, r[2] / norm};
    const double n3 = (norm * norm) * norm;
    const double c0 = (-mu) * m;
    const double n2 = norm * norm, n4 = n2 * n2, n5 = norm * n4;
    const double n6 = pow6(norm);
    const double kz = (3.0 * z) / n5;
    const double kr = 3.0 / (2.0 * n4) - (15.0 * (z * z)) / (2.0 * n6);
    const double c1 = ((c0 * J2) * (r_ref * r_ref));
    const double e_z[3] = {0.0, 0.0, 1.0};
    for (int k = 0; k < 3; ++k) {
        const double f = (c0 * r[k]) / n3;
        const double j2 = c1 * (kz * e_z[k] + kr * e_r[k]);
        F[3 + k] = F[3 + k] + (f + j2);
    }
    F[0] = F[0] + 0.0; F[1] = F[1] + 0.0; F[2] = F[2] + 0.0;
}

/* ------------------------------------------------------------------ EGM08 spherical-harmonic gravity
 * libs/nox-py/python/elodin/egm08.py (EGM08.compute_field), applied as force + SpatialForce(linear=field)
 * (examples/cube-sat/main.py:516-527).  p = [mu, r_ref, L]; table0 / table1 = the normalised C / S coefficients
 * the reference loads from C_normal.npy / S_normal.npy (a download: not in its tree, so no golden can be recomputed;
 * with C20 alone the field equals j2.py's to rounding, which is what pins the zonal path — tests/test_oracle_golden.py).
 *
 * The restatement keeps the reference's formulas, including `m = roll(self.m, -1)` (every term carries m+1, :153),
 * and fixes two things the source leaves to XLA: the double sum runs column by column (m outer, l = m..L inner; terms
 * with l < m vanish because a_bar is lower triangular) with one running accumulator per component, and
 * rho_l = (mu/r) (r_ref/r)^l is built by repeated multiplication instead of pow(). */
static double kdelta(int d) { return d == 0 ? 1.0 : 2.0; }

void orc_egm08_tables(int L, double *out)
{
    const int n = L + 1;
    double *n1 = out, *n2 = n1 + n * n, *nq1 = n2 + n * n, *nq2 = nq1 + n * n, *diag = nq2 + n * n, *offc = diag + n;
    for (int l = 0; l <= L; ++l)
        for (int m = 0; m <= L; ++m) {
            double v1 = 0.0, v2 = 0.0;
            if (l >= m + 2) { /* compute_n1 / compute_n2, :98-108 */
                v1 = sqrt((double)((2 * l + 1) * (2 * l - 1)) / (double)((l + m) * (l - m)));
                v2 = sqrt((double)((l + m - 1) * (l - m - 1) * (2 * l + 1)) / (double)((2 * l - 3) * (l + m) * (l - m)));
            }
            n1[l * n + m] = v1;
            n2[l * n + m] = v2;
            const double num1 = (double)(l - m) * kdelta(m) * (double)(l + m + 1);          /* compute_nq1, :126-134 */
            nq1[l * n + m] = num1 < 0.0 ? 0.0 : sqrt(num1 / kdelta(m + 1));
            const double num2 = (double)(l + m + 2) * (double)(l + m + 1) * (double)(2 * l + 1) * kdelta(m); /* :136-144 */
            nq2[l * n + m] = num2 < 0.0 ? 0.0 : sqrt(num2 / ((double)(2 * l + 3) * kdelta(m + 1)));
        }
    double cur = 1.0; /* a_0_0 */
    for (int l = 0; l <= L; ++l) { /* compute_a_bar_diagonal, :84-89 */
        if (l > 0) cur = cur * sqrt(((double)(2 * l + 1) * kdelta(l)) / ((double)(2 * l) * kdelta(l - 1)));
        diag[l] = cur;
        offc[l] = l == 0 ? 0.0 : diag[l] * sqrt(((double)(2 * l) * kdelta(l - 1)) / kdelta(l)); /* :91-96, times u at run time */
    }
}

static void eff_gravity_egm08(const orc_effector *e, const double pos[7], const double inertia[7], double F[6])
{
    const double mu = e->p[0], r_ref = e->p[1];
    const int L = (int)e->p[2], n = L + 1;
    if (!e->table0 || !e->table1 || L < 0 || L > 128 || e->table_len != (uint64_t)n * (uint64_t)n) return;
    double *tab = (double *)malloc((size_t)(4 * n * n + 2 * n + n + 2) * sizeof(double));
    orc_egm08_tables(L, tab);
    const double *n1 = tab, *n2 = n1 + n * n, *nq1 = n2 + n * n, *nq2 = nq1 + n * n, *diag = nq2 + n * n, *offc = diag + n;
    double *rho = tab + 4 * n * n + 2 * n; /* rho[0 .. L+1], rho[L+1] = 0 (rho_l_1's last entry, :150) */
    const double *C = e->table0, *S = e->table1;
    const double x = pos[4], y = pos[5], z = pos[6], mass = inertia[6];
    const double r = sqrt((x * x + y * y) + z * z);
    const double s = x / r, t = y / r, u = z / r;
    rho[0] = mu / r;
    const double q = r_ref / r;
    for (int l = 1; l <= L; ++l) rho[l] = rho[l - 1] * q;
    rho[L + 1] = 0.0;
    double a1 = 0.0, a2 = 0.0, a3 = 0.0, a4 = 0.0;
    double im_prev = 0.0, rm_prev = 0.0, im = 0.0, rm = 1.0; /* (i_0, r_0) = (0, 1), :110-114 */
    for (int m = 0; m <= L; ++m) {
        if (m > 0) {
            const double i_new = s * im + t * rm, r_new = s * rm - t * im;
            im_prev = im; rm_prev = rm; im = i_new; rm = r_new;
        }
        const double rm1 = m == 0 ? 0.0 : rm_prev, im1 = m == 0 ? 0.0 : im_prev; /* roll(.., 1).at[0].set(0), :151-152 */
        const double mp = m == L ? 0.0 : (double)(m + 1);                          /* roll(self.m, -1).at[-1].set(0), :154 */
        /* column m (A) and column m+1 (B) of a_bar by the same three-term recursion (:116-124) */
        double A0 = 0.0, A1 = 0.0; /* a[l-1][m], a[l-2][m] */
        double B0 = 0.0, B1 = 0.0; /* a[l][m+1] (one step ahead), a[l-1][m+1]  */
        /* B runs one degree ahead of A: prime it with a[m][m+1] = 0 */
        for (int l = m; l <= L; ++l) {
            double Al;
            if (l == m) Al = diag[m];
            else if (l == m + 1) Al = offc[l] * u;
            else Al = (u * n1[l * n + m]) * A0 - n2[l * n + m] * A1;
            A1 = A0; A0 = Al;
            /* a[l][m+1] */
            double Bl = 0.0;
            if (m + 1 <= L) {
                if (l == m + 1) Bl = diag[m + 1];
                else if (l == m + 2) Bl = offc[l] * u;
                else if (l > m + 2) Bl = (u * n1[l * n + m + 1]) * B0 - n2[l * n + m + 1] * B1;
            }
            /* a[l+1][m+1] */
            double Bn = 0.0;
            if (m + 1 <= L && l + 1 <= L) {
                const int l1 = l + 1;
                if (l1 == m + 1) Bn = diag[m + 1];
                else if (l1 == m + 2) Bn = offc[l1] * u;
                else Bn = (u * n1[l1 * n + m + 1]) * Bl - n2[l1 * n + m + 1] * B0;
            }
            B1 = B0; B0 = Bl;
            const double w = rho[l + 1] / r_ref;
            const double c = C[l * n + m], sv = S[l * n + m];
            const double ee = c * rm1 + sv * im1, ff = sv * rm1 - c * im1, dd = c * rm + sv * im;
            a1 = a1 + ((w * Al) * mp) * ee;
            a2 = a2 + ((w * Al) * mp) * ff;
            a3 = a3 + (((w * Bl) * mp) * nq1[l * n + m]) * dd;
            a4 = a4 + ((((w * Bn) * mp) * nq2[l * n + m]) * dd) * (-1.0);
        }
    }
    free(tab);
    F[3] = F[3] + mass * (a1 + s * a4);
    F[4] = F[4] + mass * (a2 + t * a4);
    F[5] = F[5] + mass * (a3 + u * a4);
    F[0] = F[0] + 0.0; F[1] = F[1] + 0.0; F[2] = F[2] + 0.0;
}

/* examples/falcon9/sim.py:350-361 + frames.py:91-109 (parity unpinned: no golden) */
static void eff_gravity_frame(const orc_effector *e, const double pos[7], const double vel[6],
                              const double inertia[7], double F[6])
{
    const double mu = e->p[0];
    const double *om = e->p + 1;
    const double *r = pos + 4, *v = vel + 3;
    const double rn = sqrt(dot3(r, r));
    const double rn3 = (rn * rn) * rn;
    double g[3], c[3], cr[3], c2[3], acc[3];
    g[0] = ((-mu) * r[0]) / rn3; g[1] = ((-mu) * r[1]) / rn3; g[2] = ((-mu) * r[2]) / rn3;
    cross3(om, v, c);
    cross3(om, r, cr);
    cross3(om, cr, c2);
    for (int k = 0; k < 3; ++k) {
        const double cor = -2.0 * c[k];
        const double cen = -c2[k];
        const double frame = cor + cen;
        acc[k] = g[k] + frame;
    }
    const double m = inertia[6];
    F[0] = F[0] + 0.0; F[1] = F[1] + 0.0; F[2] = F[2] + 0.0;
    F[3] = F[3] + acc[0] * m; F[4] = F[4] + acc[1] * m; F[5] = F[5] + acc[2] * m;
}

/* examples/three-body/main.py:63-70 gravity_fn (fold accumulator in, out) */
static void fold_newton(double G, const double *a_pos, const double *a_in, const double *b_pos,
                        const double *b_in, double acc[6])
{
    double r[3];
    r[0] = a_pos[4] - b_pos[4]; r[1] = a_pos[5] - b_pos[5]; r[2] = a_pos[6] - b_pos[6];
    const double m = a_in[6], M = b_in[6];
    const double norm = sqrt(dot3(r, r));
    const double s = (G * M) * m;
    const double d = (norm * norm) * norm;
    acc[0] = 0.0; acc[1] = 0.0; acc[2] = 0.0;       /* el.Force(linear=...) => zero torque */
    acc[3] = acc[3] - (s * r[0]) / d;
    acc[4] = acc[4] - (s * r[1]) / d;
    acc[5] = acc[5] - (s * r[2]) / d;
}

/* examples/n-body/sim.py:349-361 gravity_fn (parity unpinned above N=3: no golden) */
static void fold_softened(double K2, double soft, const double *a_pos, const double *a_in,
                          const double *b_pos, const double *b_in, double acc[6])
{
    double r[3];
    r[0] = b_pos[4] - a_pos[4]; r[1] = b_pos[5] - a_pos[5]; r[2] = b_pos[6] - a_pos[6];
    const double dist_sq = dot3(r, r) + soft;
    const double inv = 1.0 / sqrt(dist_sq);
    const double inv3 = (inv * inv) * inv;
    const double scalar = ((K2 * a_in[6]) * b_in[6]) * inv3;
    acc[0] = acc[0] + 0.0; acc[1] = acc[1] + 0.0; acc[2] = acc[2] + 0.0;
    acc[3] = acc[3] + scalar * r[0];
    acc[4] = acc[4] + scalar * r[1];
    acc[5] = acc[5] + scalar * r[2];
}

/* GraphQuery.edge_fold: per source entity, sequential left fold over its
 * out-edges in spawn order, init = zero Force; the result REPLACES that
 * entity's Force (libs/nox-py/src/graph.rs:177-236, __init__.py:454-557). */
static void eff_gravity_edges(const orc_effector *e, uint64_t n, const double *pos,
                              const double *inertia, double *F, unsigned char *has_edge)
{
    memset(has_edge, 0, n);
    for (uint64_t k = 0; k < e->n_edges; ++k)
        if (e->edge_from[k] < n) has_edge[e->edge_from[k]] = 1;
    for (uint64_t i = 0; i < n; ++i)
        if (has_edge[i]) memset(F + 6 * i, 0, 6 * sizeof(double));
    for (uint64_t k = 0; k < e->n_edges; ++k) {
        const uint64_t a = e->edge_from[k], b = e->edge_to[k];
        if (a >= n || b >= n) continue;
        if (e->kind == ORC_EFF_GRAVITY_EDGES_NEWTON)
            fold_newton(e->p[0], pos + 7 * a, inertia + 7 * a, pos + 7 * b, inertia + 7 * b, F + 6 * a);
        else
            fold_softened(e->p[0], e->p[1], pos + 7 * a, inertia + 7 * a, pos + 7 * b, inertia + 7 * b,
                          F + 6 * a);
    }
}

/* clear_forces | effectors | calc_accel  (six_dof.rs:195) on one world's stage state */
static void eval_pipe(uint64_t n, uint64_t world, const double *inertia, uint32_t n_eff,
                      const orc_effector *effs, const double *pos, const double *vel, double *F,
                      double *A, unsigned char *scratch)
{
    for (uint64_t i = 0; i < 6 * n; ++i) F[i] = 0.0; /* clear_forces, six_dof.rs:148-150 */
    for (uint32_t k = 0; k < n_eff; ++k) {
        const orc_effector *e = &effs[k];
        if (e->kind == ORC_EFF_GRAVITY_EDGES_NEWTON || e->kind == ORC_EFF_GRAVITY_EDGES_SOFTENED) {
            eff_gravity_edges(e, n, pos, inertia, F, scratch);
            continue;
        }
        for (uint64_t i = 0; i < n; ++i) {
            if (e->entity_mask && !e->entity_mask[i]) continue; /* entity lacks one of the effector's components */
            const double *col = e->column ? e->column + (world * n + i) * e->column_width : 0;
            switch (e->kind) {
            case ORC_EFF_GRAVITY_CONST: eff_gravity_const(e, inertia + 7 * i, F + 6 * i); break;
            case ORC_EFF_DRAG_QUADRATIC: eff_drag_quadratic(e, col, vel + 6 * i, F + 6 * i); break;
            case ORC_EFF_THRUST_BODY: eff_thrust_body(e, col, pos + 7 * i, F + 6 * i); break;
            case ORC_EFF_WRENCH_BODY: eff_wrench_body(e, col, pos + 7 * i, F + 6 * i); break;
            case ORC_EFF_GRAVITY_FRAME:
                eff_gravity_frame(e, pos + 7 * i, vel + 6 * i, inertia + 7 * i, F + 6 * i);
                break;
            case ORC_EFF_WRENCH_WORLD: eff_wrench_world(col, F + 6 * i); break;
            case ORC_EFF_TORQUE_BODY_FOLD: eff_torque_body_fold(e, col, pos + 7 * i, F + 6 * i); break;
            case ORC_EFF_GRAVITY_J2: eff_gravity_j2(e, pos + 7 * i, inertia + 7 * i, F + 6 * i); break;
            case ORC_EFF_GRAVITY_EGM08: eff_gravity_egm08(e, pos + 7 * i, inertia + 7 * i, F + 6 * i); break;
            default: break;
            }
        }
    }
    for (uint64_t i = 0; i < n; ++i) orc_calc_accel(pos + 7 * i, F + 6 * i, inertia + 7 * i, A + 6 * i);
}

void orc_eval_stage(const orc_world *w, uint64_t world, uint32_t n_eff, const orc_effector *effs,
                    const double *pos, const double *vel, double *force, double *accel)
{
    unsigned char *scratch = (unsigned char *)malloc(w->n ? w->n : 1);
    eval_pipe(w->n, world, w->inertia + world * w->n * 7, n_eff, effs, pos, vel, force, accel, scratch);
    free(scratch);
}

/* ------------------------------------------------------------------ RK4
 * libs/nox-py/src/integrator/rk4.rs:77-125.  `init_u.insert_into_builder`
 * (rk4.rs:105,107,109) restores WorldPos/WorldVel to (x0, v0) before each
 * `step` binds `du = (vars[WorldVel], vars[WorldAccel])`, so every stage
 * position is advanced with v0 and every stage velocity with the previous
 * stage's acceleration (stage 1: the WorldAccel column, times 0):
 *   a_s = A(x0 (+) (dt*f_s)*v0 ,  v0 + (dt*f_s)*a_{s-1}),   f = 0, .5, .5, 1
 *   k_s = (stage velocity, a_s)
 *   u1  = u0 + (dt_final*(1/6)) * (((k1 + 2.0*k2) + 2.0*k3) + k4)
 * Force and WorldAccel leave the tick holding their stage-4 values. */
static void rk4_world_tick(uint64_t n, uint64_t world, double *pos, double *vel, double *accel,
                           double *force, const double *inertia, uint32_t n_eff,
                           const orc_effector *effs, double dt_stage, double dt_final, double *tmp,
                           unsigned char *scratch)
{
    double *sx = tmp;            /* [n,7] stage position  */
    double *sv = sx + 7 * n;     /* [n,6] stage velocity  */
    double *sa = sv + 6 * n;     /* [n,6] stage accel     */
    double *sf = sa + 6 * n;     /* [n,6] stage force     */
    double *kv = sf + 6 * n;     /* [n,6] running sum of k.v */
    double *ka = kv + 6 * n;     /* [n,6] running sum of k.a */
    static const double fac[4] = {0.0, 0.5, 0.5, 1.0};

    memcpy(sa, accel, 6 * n * sizeof(double)); /* du.a before stage 1 = WorldAccel column */
    for (int s = 0; s < 4; ++s) {
        const double dtf = dt_stage * fac[s]; /* rk4.rs:90 */
        for (uint64_t i = 0; i < n; ++i) {
            double mv[6];
            for (int k = 0; k < 6; ++k) mv[k] = dtf * vel[6 * i + k];           /* dt*du.v (six_dof.rs:62-70) */
            orc_transform_add_motion(pos + 7 * i, mv, sx + 7 * i);               /* U+DU: x (+) v (six_dof.rs:40-49) */
            for (int k = 0; k < 6; ++k) sv[6 * i + k] = vel[6 * i + k] + dtf * sa[6 * i + k];
        }
        eval_pipe(n, world, inertia, n_eff, effs, sx, sv, sf, sa, scratch);
        for (uint64_t i = 0; i < 6 * n; ++i) {
            if (s == 0) { kv[i] = sv[i]; ka[i] = sa[i]; }
            else if (s == 3) { kv[i] = kv[i] + sv[i]; ka[i] = ka[i] + sa[i]; }
            else { kv[i] = kv[i] + 2.0 * sv[i]; ka[i] = ka[i] + 2.0 * sa[i]; }
        }
    }
    const double c = dt_final * (1.0 / 6.0); /* rk4.rs:119 */
    for (uint64_t i = 0; i < n; ++i) {
        double mv[6], nx[7];
        for (int k = 0; k < 6; ++k) mv[k] = c * kv[6 * i + k];
        orc_transform_add_motion(pos + 7 * i, mv, nx);
        memcpy(pos + 7 * i, nx, sizeof nx);
        for (int k = 0; k < 6; ++k) vel[6 * i + k] = vel[6 * i + k] + c * ka[6 * i + k];
    }
    memcpy(accel, sa, 6 * n * sizeof(double));
    memcpy(force, sf, 6 * n * sizeof(double));
}

/* libs/nox-py/src/integrator/semi_implicit.rs:42-62: v' = v + dt*a ; x' = x (+) dt*v' */
static void semi_world_tick(uint64_t n, uint64_t world, double *pos, double *vel, double *accel,
                            double *force, const double *inertia, uint32_t n_eff,
                            const orc_effector *effs, double dt, unsigned char *scratch)
{
    eval_pipe(n, world, inertia, n_eff, effs, pos, vel, force, accel, scratch);
    for (uint64_t i = 0; i < n; ++i) {
        double mv[6], nx[7];
        for (int k = 0; k < 6; ++k) vel[6 * i + k] = vel[6 * i + k] + dt * accel[6 * i + k];
        for (int k = 0; k < 6; ++k) mv[k] = dt * vel[6 * i + k];
        orc_transform_add_motion(pos + 7 * i, mv, nx);
        memcpy(pos + 7 * i, nx, sizeof nx);
    }
}

/* ---- world-parallel driver (bench baseline only): static partition of the
 * world axis over pthreads, mirroring `elodin monte-carlo` workers = logical
 * cores (libs/monte-carlo/src/lib.rs:2530-2538). ---- */
/* CPUs this process may actually run on: the scheduler affinity set, clipped by the cgroup CPU quota
 * (cpu.max = "<quota> <period>") — not the number of CPUs the machine has online. */
int orc_max_threads(void)
{
    long n = sysconf(_SC_NPROCESSORS_ONLN);
    cpu_set_t set;
    CPU_ZERO(&set);
    if (sched_getaffinity(0, sizeof set, &set) == 0 && CPU_COUNT(&set) > 0) n = CPU_COUNT(&set);
    FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r");
    if (f) {
        char q[32] = {0};
        long period = 0;
        if (fscanf(f, "%31s %ld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) {
            long quota = atol(q);
            long cpus = (quota + period - 1) / period;
            if (cpus > 0 && cpus < n) n = cpus;
        }
        fclose(f);
    }
    return n > 0 ? (int)n : 1;
}

typedef struct orc_job {
    orc_world *w;
    uint32_t n_eff;
    const orc_effector *effs;
    double dt_stage, dt_final;
    uint64_t n_ticks;
    uint64_t m0, m1;
    int semi;
} orc_job;

static void *orc_worker(void *arg)
{
    orc_job *j = (orc_job *)arg;
    orc_world *w = j->w;
    const uint64_t n = w->n;
    double *tmp = (double *)malloc((37 * n + 1) * sizeof(double));
    unsigned char *scratch = (unsigned char *)malloc(n ? n : 1);
    for (uint64_t m = j->m0; m < j->m1; ++m) {
        for (uint64_t t = 0; t < j->n_ticks; ++t) {
            if (j->semi)
                semi_world_tick(n, m, w->pos + m * n * 7, w->vel + m * n * 6, w->accel + m * n * 6,
                                w->force + m * n * 6, w->inertia + m * n * 7, j->n_eff, j->effs,
                                j->dt_stage, scratch);
            else
                rk4_world_tick(n, m, w->pos + m * n * 7, w->vel + m * n * 6, w->accel + m * n * 6,
                               w->force + m * n * 6, w->inertia + m * n * 7, j->n_eff, j->effs,
                               j->dt_stage, j->dt_final, tmp, scratch);
        }
    }
    free(tmp);
    free(scratch);
    return 0;
}

static void orc_run(orc_world *w, uint32_t n_eff, const orc_effector *effs, double dt_stage,
                    double dt_final, uint64_t n_ticks, int n_threads, int semi)
{
    const uint64_t M = w->n_worlds;
    if (n_threads < 1) n_threads = 1;
    if ((uint64_t)n_threads > M) n_threads = (int)(M ? M : 1);
    orc_job *jobs = (orc_job *)calloc((size_t)n_threads, sizeof(orc_job));
    pthread_t *th = (pthread_t *)calloc((size_t)n_threads, sizeof(pthread_t));
    for (int t = 0; t < n_threads; ++t) {
        jobs[t].w = w; jobs[t].n_eff = n_eff; jobs[t].effs = effs;
        jobs[t].dt_stage = dt_stage; jobs[t].dt_final = dt_final; jobs[t].n_ticks = n_ticks;
        jobs[t].m0 = M * (uint64_t)t / (uint64_t)n_threads;
        jobs[t].m1 = M * (uint64_t)(t + 1) / (uint64_t)n_threads;
        jobs[t].semi = semi;
    }
    if (n_threads == 1) {
        orc_worker(&jobs[0]);
    } else {
        for (int t = 0; t < n_threads; ++t) pthread_create(&th[t], 0, orc_worker, &jobs[t]);
        for (int t = 0; t < n_threads; ++t) pthread_join(th[t], 0);
    }
    free(jobs);
    free(th);
}

void orc_rk4_ticks(orc_world *w, uint32_t n_eff, const orc_effector *effs, double dt_stage,
                   double dt_final, uint64_t n_ticks, int n_threads)
{
    orc_run(w, n_eff, effs, dt_stage, dt_final, n_ticks, n_threads, 0);
}

void orc_semi_implicit_ticks(orc_world *w, uint32_t n_eff, const orc_effector *effs, double dt,
                             uint64_t n_ticks, int n_threads)
{
    orc_run(w, n_eff, effs, dt, dt, n_ticks, n_threads, 1);
}
