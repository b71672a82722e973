"""The EGM08 field kernel (egm08_force_kernel evaluating egm08_field.cuh) against a high-precision reference of
python/elodin/egm08.py, at every degree the C ABI accepts, on the polar axis and at the edges of the f64 range.

The reference (`ref_field`) evaluates the series with constants built from integers and the sums in 400-bit fixed
point; the radius, the radial factors and the final combination are mpmath at 256 bits.  It keeps the source's quirks:
every term carries m + 1 (0 at m = L), rho_{L+1} = 0 so degree L drops out, and the a4 term is subtracted.  Beside the
field it returns a per-component scale S_k: the same double sum with every term replaced by its magnitude.  An f64
evaluation of the series rounds within

    |got - ref| <= (3 L + 16) 2^-53 S_k        (bound_factor)

per component and per body, wherever every radial factor and the scale are normal doubles.  The per-degree share is
the radial factor: rho_{l+1} is l + 1 chained products of q = r_ref / r, itself formed from a rounded r, so its error
grows with the degree (at most about 2.75 ulps per degree) and is the same for every term of that degree.  Where the
top degrees carry the sum (EGM-like coefficients at r = 1e3 m) the oracle lands at 121 x 2^-53 S_k at degree 64, past
L + 16 = 80; everywhere else it stays below L + 16.  The CPU tests prove the
reference against the array form of the source, the oracle and the J2 closed form, and prove the bound sensitive: a
plain-f64 restatement of egm08_field (which reproduces the oracle bit for bit) with one fault injected must fail it.

The GPU tests read the field out of one tick with v0 = 0 (every RK4 stage slot and the semi-implicit stage sit at x0):
EXACT bit for bit with the oracle at every degree 0..128, FAST within a few ulps, both within the bound; then a tick at
orbital speed, invoke_batch over ragged world ranges with an entity mask, the launched kernels, and the refusals of
degrees and table lengths the ABI does not accept.
"""

import functools
import math
import os
from concurrent.futures import ProcessPoolExecutor
from dataclasses import dataclass
from multiprocessing import get_context
from typing import Optional

import mpmath
import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200.executor import FORCE, INERTIA, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from tests.ensemble_util import need_gpu
from tests.test_oracle_golden import _egm08_array_form, _egm08_random_tables
from tests.util import (MU_EARTH, R_EARTH, assert_body_close, assert_route, body_effectors, body_scales,
                        launched_kernels, orbit_world)

BOUND_PER_DEGREE, BOUND_TERMS = 3, 16
FRAC = 400  # fraction bits of the reference's fixed-point sums
MAX_DEGREE = 128
DT = 1.0
INTEGRATORS = ("rk4", "semi_implicit")
_I = {"rk4": 0, "semi_implicit": 1}
TINY = 2.0 ** -1022


def bound_factor(L):
    """The bound in units of 2^-53 S_k at degree L (module docstring)."""
    return BOUND_PER_DEGREE * L + BOUND_TERMS

# --------------------------------------------------------------------------- the geometry catalogue

M_WORLDS, N_BODIES = 3, 67  # 201 bodies: not a multiple of the kernel's 128-thread blocks


@functools.lru_cache(maxsize=None)
def catalogue():
    """(pos [M, N, 7], ine [M, N, 7], labels [M*N]) of the bodies where the series is fragile, then random directions
    at 0.98..1.1 r_ref up to M*N bodies; attitude identity, unit inertia diagonal, masses U(0.5, 50) except the
    irregular ones."""
    R = R_EARTH * 1.01
    d = 1e-12 * R
    rng = np.random.default_rng(2024)
    bodies = [("+z pole", (0.0, 0.0, R)), ("-z pole", (0.0, 0.0, -R)), ("+z pole -0", (-0.0, -0.0, R)),
              ("-z pole -0", (-0.0, -0.0, -R)), ("off +z pole", (d, 0.0, R)), ("off -z pole", (0.0, -d, -R)),
              ("off +z pole xy", (d, d, R)), ("+x axis", (R, 0.0, 0.0)), ("-x axis", (-R, 0.0, 0.0)),
              ("+y axis", (0.0, R, 0.0)), ("-y axis", (0.0, -R, 0.0))]
    for k in range(4):
        a = 2 * np.pi * rng.random()
        bodies.append((f"equator +0 #{k}", (R * np.cos(a), R * np.sin(a), 0.0)))
        bodies.append((f"equator -0 #{k}", (R * np.cos(a), R * np.sin(a), -0.0)))

    def shell(name, radius, n):
        for k in range(n):
            v = rng.normal(size=3)
            bodies.append((f"{name} #{k}", tuple(v / np.linalg.norm(v) * radius)))

    shell("0.6 r_ref", 0.6 * R_EARTH, 8)
    shell("3 r_ref", 3.0 * R_EARTH, 8)
    shell("1e9 m", 1e9, 8)
    shell("1e12 m", 1e12, 8)
    shell("1e3 m", 1e3, 6)
    bodies += [("r = 0", (0.0, 0.0, 0.0)), ("r = -0", (-0.0, -0.0, -0.0)), ("NaN x", (np.nan, 1e6, 7e6)),
               ("+inf y", (1e6, np.inf, 7e6)), ("-inf z", (1e6, 1e6, -np.inf))]
    n_special = len(bodies)
    while len(bodies) < M_WORLDS * N_BODIES:
        v = rng.normal(size=3)
        bodies.append((f"random #{len(bodies) - n_special}", tuple(v / np.linalg.norm(v) * R_EARTH * rng.uniform(0.98, 1.1))))
    mass = rng.uniform(0.5, 50.0, len(bodies))
    irregular = {n_special + 0: 0.0, n_special + 1: -2.0, n_special + 2: 5e-324, n_special + 3: 1e300, 0: -2.0}
    for i, m in irregular.items():
        mass[i] = m
    pos = np.zeros((M_WORLDS * N_BODIES, 7))
    pos[:, 3] = 1.0
    pos[:, 4:] = np.array([b[1] for b in bodies])
    ine = np.zeros((M_WORLDS * N_BODIES, 7))
    ine[:, :3] = 1.0
    ine[:, 6] = mass
    shape = (M_WORLDS, N_BODIES, 7)
    return pos.reshape(shape), ine.reshape(shape), [b[0] for b in bodies]


def regular_mass(ine):
    """FAST turns a mass of 0, a subnormal, an infinity or NaN into NaN by design (DESIGN.md, mass-class summary)."""
    m = np.abs(ine[..., 6])
    return np.isfinite(m) & (m >= TINY)


@functools.lru_cache(maxsize=None)
def tables(L, kind):
    """(C, S) of degree L: "kaula" (EGM-like, _egm08_random_tables), "dense" (N(0, 1): every term visible) or "unit"
    (one unit S coefficient at (L-1, L-1): an error in the last live column is full size; L >= 2)."""
    rng = np.random.default_rng(1000 + 7 * L + {"kaula": 0, "dense": 1, "unit": 2}[kind])
    if kind == "kaula":  # (C20 needs degree 2: cut the degree-2 tables below it)
        c, s = _egm08_random_tables(max(L, 2), rng)
        return np.ascontiguousarray(c[:L + 1, :L + 1]), np.ascontiguousarray(s[:L + 1, :L + 1])
    c, s = np.zeros((L + 1, L + 1)), np.zeros((L + 1, L + 1))
    if kind == "dense":
        c = np.tril(rng.normal(0, 1, (L + 1, L + 1)))
        s = np.tril(rng.normal(0, 1, (L + 1, L + 1)), -1)
    else:
        assert L >= 2
        s[L - 1, L - 1] = 1.0
    return c, s


def table_kinds(L):
    return ("dense", "kaula", "unit") if L >= 2 else ("dense", "kaula")


# --------------------------------------------------------------------------- the high-precision reference


def _kd(d):
    return 1 if d == 0 else 2


def _fix_sqrt(num, den):
    """floor(sqrt(num / den) 2^FRAC), from integers."""
    return math.isqrt((num << (2 * FRAC)) // den)


def _fix(v):
    """An f64 in fixed point (exact for |v| >= 2^(53 - FRAC))."""
    n, d = float(v).as_integer_ratio()
    return (n << FRAC) // d


@functools.lru_cache(maxsize=4)
def _ref_constants(L):
    """diag, offc, n1, n2, nq1, nq2 of egm08.py in fixed point, each from integers (diag_l^2 is a product of rationals)."""
    diag, offc = [1 << FRAC], [0]
    num, den = 1, 1
    for l in range(1, L + 2):
        num, den = num * (2 * l + 1) * _kd(l), den * 2 * l * _kd(l - 1)
        diag.append(_fix_sqrt(num, den))
        offc.append(_fix_sqrt(num * 2 * l * _kd(l - 1), den * _kd(l)))
    n1 = [[0] * (L + 2) for _ in range(L + 1)]
    n2 = [[0] * (L + 2) for _ in range(L + 1)]
    nq1 = [[0] * (L + 1) for _ in range(L + 1)]
    nq2 = [[0] * (L + 1) for _ in range(L + 1)]
    for l in range(L + 1):
        for m in range(L + 2):
            if l >= m + 2:
                n1[l][m] = _fix_sqrt((2 * l + 1) * (2 * l - 1), (l + m) * (l - m))
                n2[l][m] = _fix_sqrt((l + m - 1) * (l - m - 1) * (2 * l + 1), (2 * l - 3) * (l + m) * (l - m))
        for m in range(l + 1):
            nq1[l][m] = _fix_sqrt((l - m) * _kd(m) * (l + m + 1), _kd(m + 1))
            nq2[l][m] = _fix_sqrt((l + m + 2) * (l + m + 1) * (2 * l + 1) * _kd(m), (2 * l + 3) * _kd(m + 1))
    return diag, offc, n1, n2, nq1, nq2


def ref_field(x, y, z, mass, C, S, L, mu=MU_EARTH, r_ref=R_EARTH):
    """egm08.py's field times the mass at the exact f64 inputs: (field [3], scale S_k [3], largest intermediate), as
    mpmath numbers, or None where the field is undefined (a non-finite input, r = 0).  S_k sums the magnitudes of the
    terms with the true |A_lm| and |B_lm|, plus the |s| |a4| share.  The largest intermediate is the largest
    |w_l A_lm (m+1)|, |w_l B_lm (m+1) nq1| or |w_l B_l+1,m (m+1) nq2| an f64 evaluation forms."""
    if not all(math.isfinite(v) for v in (x, y, z, mass, mu, r_ref)) or (x, y, z) == (0.0, 0.0, 0.0):
        return None
    F = FRAC
    diag, offc, n1, n2, nq1, nq2 = _ref_constants(L)
    with mpmath.workprec(F + 64):
        X, Y, Z = mpmath.mpf(x), mpmath.mpf(y), mpmath.mpf(z)
        r = mpmath.sqrt(X * X + Y * Y + Z * Z)
        s, t, u = X / r, Y / r, Z / r
        fx = lambda v: int(mpmath.floor(mpmath.ldexp(v, F)))
        si, ti, ui = fx(s), fx(t), fx(u)
    rm, im = [1 << F], [0]
    for m in range(1, L + 1):
        r0, i0 = rm[-1], im[-1]
        rm.append((si * r0 - ti * i0) >> F)
        im.append((si * i0 + ti * r0) >> F)

    def column(m):  # a_bar[l][m], l = 0..L (0 for l < m)
        a = [0] * (L + 1)
        if m > L:
            return a
        a[m] = diag[m]
        if m + 1 <= L:
            a[m + 1] = (offc[m + 1] * ui) >> F
        for l in range(m + 2, L + 1):
            a[l] = (((ui * n1[l][m]) >> F) * a[l - 1] >> F) - ((n2[l][m] * a[l - 2]) >> F)
        return a

    # per degree l: the sums over m of the four components (units 2^-3F for a1, a2; 2^-4F for a3, a4), their
    # magnitudes, and the largest |A (m+1)| (2^-F) and |B (m+1) nq| (2^-2F)
    o = [[0] * 4 for _ in range(L + 1)]
    g = [[0] * 4 for _ in range(L + 1)]
    amax, bmax = [0] * (L + 1), [0] * (L + 1)
    Cf = [[_fix(C[l, m]) for m in range(l + 1)] for l in range(L + 1)]
    Sf = [[_fix(S[l, m]) for m in range(l + 1)] for l in range(L + 1)]
    B = column(0)
    for m in range(L):  # column L carries m + 1 = 0 (roll(m, -1)); degree L carries rho_{L+1} = 0
        A, B = B, column(m + 1)
        mp = m + 1
        rm1, im1 = (rm[m - 1], im[m - 1]) if m else (0, 0)
        for l in range(m, L):
            c, sv = Cf[l][m], Sf[l][m]
            p1, p2, p3, p4, q1, q2 = c * rm1, sv * im1, sv * rm1, c * im1, c * rm[m], sv * im[m]
            a, b, bn = A[l] * mp, B[l] * mp, B[l + 1] * mp
            b1, b2 = b * nq1[l][m], bn * nq2[l][m]
            ol, gl = o[l], g[l]
            ol[0] += a * (p1 + p2)
            ol[1] += a * (p3 - p4)
            ol[2] += b1 * (q1 + q2)
            ol[3] -= b2 * (q1 + q2)
            aa, dd = abs(a), abs(q1) + abs(q2)
            gl[0] += aa * (abs(p1) + abs(p2))
            gl[1] += aa * (abs(p3) + abs(p4))
            gl[2] += abs(b1) * dd
            gl[3] += abs(b2) * dd
            amax[l] = max(amax[l], aa)
            bmax[l] = max(bmax[l], abs(b1), abs(b2))
    with mpmath.workprec(256):
        X, Y, Z, Mu, Rr = (mpmath.mpf(v) for v in (x, y, z, mu, r_ref))
        r = mpmath.sqrt(X * X + Y * Y + Z * Z)
        s, t, u = X / r, Y / r, Z / r
        q = Rr / r
        w = [Mu / r * q ** (l + 1) / Rr for l in range(L)]
        units = [mpmath.ldexp(1, -3 * F)] * 2 + [mpmath.ldexp(1, -4 * F)] * 2
        a = [mpmath.fsum(w[l] * o[l][k] for l in range(L)) * units[k] for k in range(4)]
        sc = [mpmath.fsum(abs(w[l]) * g[l][k] for l in range(L)) * units[k] for k in range(4)]
        mx = max([abs(w[l]) * max(amax[l] * mpmath.ldexp(1, -F), bmax[l] * mpmath.ldexp(1, -2 * F)) for l in range(L)],
                 default=mpmath.mpf(0))
        Ms = mpmath.mpf(mass)
        field = [Ms * (a[0] + s * a[3]), Ms * (a[1] + t * a[3]), Ms * (a[2] + u * a[3])]
        scale = [abs(Ms) * (sc[0] + abs(s) * sc[3]), abs(Ms) * (sc[1] + abs(t) * sc[3]), abs(Ms) * (sc[2] + abs(u) * sc[3])]
    return field, scale, mx


def in_range(x, y, z, mass, L, ref, mu=MU_EARTH, r_ref=R_EARTH):
    """Whether the bound applies to this body: a defined reference, every f64 radial factor w_l (l < L) a normal
    double, the field, the scale and every intermediate finite with room to spare, and the mass a normal double."""
    if ref is None or not (TINY <= abs(mass) < math.inf):
        return False
    field, scale, mx = ref
    r = math.sqrt((x * x + y * y) + z * z)
    rho, q = mu / r, r_ref / r
    for _ in range(L):
        rho *= q
        if not TINY <= abs(rho / r_ref) < 2.0 ** 1000:
            return False
    big = mpmath.ldexp(1, 1000)
    return all(abs(v) < big for v in field) and all(v < big for v in scale) and mx * abs(mass) < big and mx < big


def bound_ratios(got, ref, L):
    """|got - ref| / (bound_factor(L) 2^-53 S_k) per component; a component with S_k = 0 must be 0, one whose scale is not
    a normal double far from underflow (S_k < 2^-900) is not judged (returns 0)."""
    field, scale, _ = ref
    out = []
    with mpmath.workprec(256):
        for g, f, sk in zip(got, field, scale):
            if sk == 0:
                out.append(0.0 if g == 0 else math.inf)
            elif sk < mpmath.ldexp(1, -900):
                out.append(0.0)
            elif not math.isfinite(g):
                out.append(math.inf)
            else:
                out.append(float(abs(mpmath.mpf(g) - f) / (bound_factor(L) * mpmath.ldexp(sk, -53))))
    return out


def _ref_job(args):
    x, y, z, mass, L, kind = args
    c, s = tables(L, kind)
    return ref_field(x, y, z, mass, c, s, L)


_REFS = {}


def catalogue_refs(L, kind):
    """ref_field of every catalogue body for the tables (L, kind), computed once per module (in a process pool)."""
    key = (L, kind)
    if key not in _REFS:
        pos, ine, _ = catalogue()
        jobs = [(float(p[4]), float(p[5]), float(p[6]), float(m), L, kind)
                for p, m in zip(pos.reshape(-1, 7), ine.reshape(-1, 7)[:, 6])]
        if L >= 32:
            with ProcessPoolExecutor(max_workers=max(1, min(16, os.cpu_count() or 1)), mp_context=get_context("spawn")) as pool:
                _REFS[key] = list(pool.map(_ref_job, jobs, chunksize=4))
        else:
            _REFS[key] = [_ref_job(j) for j in jobs]
    return _REFS[key]


def judged(L, kind):
    """[(flat body index, ref)] of the catalogue bodies the bound applies to."""
    pos, ine, _ = catalogue()
    p, m = pos.reshape(-1, 7), ine.reshape(-1, 7)[:, 6]
    refs = catalogue_refs(L, kind)
    return [(i, ref) for i, ref in enumerate(refs) if in_range(p[i, 4], p[i, 5], p[i, 6], m[i], L, ref)]


def worst_ratio(force, L, kind, bodies=None):
    """(worst ratio to the bound, its body label) of the linear Force [M, N, 3] over the judged bodies."""
    labels = catalogue()[2]
    f = force.reshape(-1, 3)
    worst = (0.0, "")
    for i, ref in judged(L, kind):
        if bodies is not None and not bodies[i]:
            continue
        r = max(bound_ratios(f[i], ref, L))
        worst = max(worst, (r, labels[i]))
    return worst


# --------------------------------------------------------------------------- f64: the oracle and a restatement


def oracle_field(O, pos, ine, L, c, s):
    """The oracle's Force [M, N, 6] of GRAVITY_EGM08 alone at the positions `pos` (oracle.World.eval_stage)."""
    M, N = pos.shape[:2]
    w = O.World(pos, np.zeros((M, N, 6)), ine)
    e = [O.Effector(O.EFF_GRAVITY_EGM08, p=(MU_EARTH, R_EARTH, L), tables=(c, s))]
    return np.stack([w.eval_stage(k, e)[0] for k in range(M)])


def term_stream(L, c, s):
    """The term stream the library builds at create (sixdof_abi.cu:egm08_tables), [terms, 8]."""
    import ctypes as C

    Lb, dp = _lib.lib(), C.POINTER(C.c_double)
    c, s = np.ascontiguousarray(c, dtype=np.float64), np.ascontiguousarray(s, dtype=np.float64)
    out = np.empty(int(Lb.b200_egm08_stream_len(L)))
    _lib.check(Lb.b200_egm08_stream(L, c.ctypes.data_as(dp), s.ctypes.data_as(dp), out.ctypes.data_as(dp), out.size))
    return out.reshape(-1, 8)


def f64_field(pos3, mass, L, c, s, fault=None, mu=MU_EARTH, r_ref=R_EARTH):
    """egm08_field.cuh restated in numpy f64 over a vector of bodies: the term stream, column by column, the carried
    B_{l+1}, every operation in the kernel's (the oracle's) order.  fault = (kind, where) injects one change:
    ("coef", k) scales C[L-1][L-1] by k; ("swap", None) swaps C and S of term (L-1, L-1); ("rho", l) uses rho_l for
    rho_{l+1} at degree l; ("mp", m) carries m instead of m + 1 in column m.  Returns the field times the mass [B, 3]."""
    kind, where = fault or (None, None)
    c, s = np.array(c, dtype=np.float64), np.array(s, dtype=np.float64)
    if kind == "coef":
        c[L - 1, L - 1] *= where
    if kind == "swap":
        c[L - 1, L - 1], s[L - 1, L - 1] = s[L - 1, L - 1], c[L - 1, L - 1]
    tab = term_stream(L, c, s)
    x, y, z = pos3[:, 0], pos3[:, 1], pos3[:, 2]
    with np.errstate(all="ignore"):
        r = np.sqrt((x * x + y * y) + z * z)
        sx, tx, ux = x / r, y / r, z / r
        rhos = [mu / r]
        q = r_ref / r
        for l in range(1, L + 1):
            rhos.append(rhos[-1] * q)
        w = [rhos[l + 1] / r_ref for l in range(L)] + [np.full_like(r, 0.0 / r_ref)]
        if kind == "rho":
            w[where] = rhos[where] / r_ref
        acc = [np.zeros_like(r) for _ in range(4)]
        im_prev = rm_prev = im = np.zeros_like(r)
        rm = np.ones_like(r)
        k = 0
        for m in range(L + 1):
            if m > 0:
                i_new, r_new = sx * im + tx * rm, sx * rm - tx * im
                im_prev, rm_prev, im, rm = im, rm, i_new, r_new
            rm1, im1 = (0.0, 0.0) if m == 0 else (rm_prev, im_prev)
            mp = 0.0 if m == L else float(m + 1)
            if kind == "mp" and m == where:
                mp = float(m)

            def term(Al, Bl, Bn, rc, wl):
                cc, sv, q1, q2 = rc
                ee, ff, dd = cc * rm1 + sv * im1, sv * rm1 - cc * im1, cc * rm + sv * im
                wa = (wl * Al) * mp
                acc[0] = acc[0] + wa * ee
                acc[1] = acc[1] + wa * ff
                acc[2] = acc[2] + (((wl * Bl) * mp) * q1) * dd
                acc[3] = acc[3] - (((wl * Bn) * mp) * q2) * dd

            ra = tab[k]
            A1, A0, Bl, Bn = 0.0, ra[0], 0.0, ra[2] if m < L else 0.0
            term(A0, Bl, Bn, tab[k, 4:], w[m])
            k += 1
            if m == L:
                break
            ra = tab[k]
            A1, A0 = A0, ra[0] * ux
            Bl, Bn = Bn, ra[2] * ux if m + 1 < L else 0.0
            term(A0, Bl, Bn, tab[k, 4:], w[m + 1])
            k += 1
            if m + 1 == L:
                continue
            for l in range(m + 2, L):
                ra = tab[k]
                Al = (ux * ra[0]) * A0 - ra[1] * A1
                A1, A0 = A0, Al
                Bq = (ux * ra[2]) * Bn - ra[3] * Bl
                Bl, Bn = Bn, Bq
                term(Al, Bl, Bn, tab[k, 4:], w[l])
                k += 1
            ra = tab[k]
            Al = (ux * ra[0]) * A0 - ra[1] * A1
            term(Al, Bn, 0.0, tab[k, 4:], w[L])
            k += 1
        a1, a2, a3, a4 = acc  # added to a zero Force, as the oracle and the body kernels do
        return np.stack([0.0 + mass * (a1 + sx * a4), 0.0 + mass * (a2 + tx * a4), 0.0 + mass * (a3 + ux * a4)], -1)


def same_bits(a, b):
    """Equal bit for bit where not NaN (the sign of zero included), NaN where the other is NaN."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a.view(np.uint64)[~na], b.view(np.uint64)[~nb])


def ulp_distance(a, b):
    """|a - b| in units in the last place (ordered integer distance: +0 and -0 are 0 apart); NaNs count 0."""
    ka, kb = (np.asarray(v, dtype=np.float64).view(np.int64).astype(object) for v in (a, b))
    key = np.vectorize(lambda i: i if i >= 0 else -(i & 0x7FFFFFFFFFFFFFFF), otypes=[object])
    d = np.abs(key(ka) - key(kb))
    d[np.isnan(a) | np.isnan(b)] = 0
    return d.astype(np.float64)


# --------------------------------------------------------------------------- CPU: the reference is right


@pytest.mark.parametrize("L", [1, 2, 3, 8, 16, 64, 128])
@pytest.mark.parametrize("kind", ["dense", "kaula"])
def test_reference_agrees_with_the_oracle_and_the_array_form(oracle, L, kind):
    """Within the bound on the catalogue: the oracle's field (every judged body), and the array formulation of the
    source (_egm08_array_form, a second reading of egm08.py with pow() radial factors) at the fragile bodies and a
    few random ones.  The judged bodies cover the poles, the axes, both equators and every finite shell."""
    pos, ine, labels = catalogue()
    c, s = tables(L, kind)
    got = oracle_field(oracle, pos, ine, L, c, s)[..., 3:].reshape(-1, 3)
    judge = judged(L, kind)
    assert len(judge) >= 150, f"only {len(judge)} bodies judged"
    worst_o, worst_a = (0.0, ""), (0.0, "")
    p = pos.reshape(-1, 7)
    m = ine.reshape(-1, 7)[:, 6]
    for i, ref in judge:
        worst_o = max(worst_o, (max(bound_ratios(got[i], ref, L)), labels[i]))
        if not labels[i].startswith("random") or labels[i] in ("random #0", "random #1"):
            with np.errstate(all="ignore"):
                arr = _egm08_array_form(p[i, 4], p[i, 5], p[i, 6], m[i], c, s, L)
            worst_a = max(worst_a, (max(bound_ratios(arr, ref, L)), labels[i]))
    print(f"\nL={L} {kind}: error / bound, oracle {worst_o[0]:.3g} ({worst_o[1]}), array form {worst_a[0]:.3g} "
          f"({worst_a[1]}); worst / 2^-53 S_k: {worst_o[0] * bound_factor(L):.3g}")
    assert worst_o[0] <= 1.0, f"L={L} {kind}: the oracle at {worst_o[1]} is {worst_o[0]:.3g} of the bound"
    assert worst_a[0] <= 1.0, f"L={L} {kind}: the array form at {worst_a[1]} is {worst_a[0]:.3g} of the bound"
    # (at 1e12 m rho_l leaves the normal doubles near degree 57)
    for name in ("+z pole", "-z pole", "off +z pole", "+x axis", "equator -0 #0", "3 r_ref #0", "1e9 m #0") + (("1e12 m #0",) if L <= 32 else ()):
        assert labels.index(name) in dict(judge), f"{name} is not judged"


@pytest.mark.parametrize("L", [3, 4, 16])
def test_reference_with_c20_alone_is_the_j2_closed_form(L):
    """With C00 = 1 and C20 = -J2/sqrt(5) alone the series is j2.py's closed form
    -mu r/n^3 - 3/2 J2 mu R^2/n^5 ((1 - 5 z^2/n^2) r + 2 z e_z), to the reference's own precision."""
    c, s = np.zeros((L + 1, L + 1)), np.zeros((L + 1, L + 1))
    j2 = 1.08262668e-3
    c[0, 0], c[2, 0] = 1.0, -j2 / np.sqrt(5.0)
    pos, ine, labels = catalogue()
    p, mass = pos.reshape(-1, 7)[:, 4:], ine.reshape(-1, 7)[:, 6]
    n = 0
    for i in range(len(p)):
        if not (np.all(np.isfinite(p[i])) and np.any(p[i] != 0) and np.isfinite(mass[i])):
            continue
        f, sc, _ = ref_field(*p[i], mass[i], c, s, L)
        with mpmath.workprec(256):
            X = [mpmath.mpf(v) for v in p[i]]
            nn = mpmath.sqrt(sum(v * v for v in X))
            Mu, R, J2, M = mpmath.mpf(MU_EARTH), mpmath.mpf(R_EARTH), mpmath.mpf(c[2, 0]) * -mpmath.sqrt(5), mpmath.mpf(mass[i])
            k = 1 - 5 * X[2] ** 2 / nn ** 2
            want = [M * (-Mu * X[j] / nn ** 3 - mpmath.mpf(3) / 2 * J2 * Mu * R ** 2 / nn ** 5 * (k * X[j] + (2 * X[2] if j == 2 else 0)))
                    for j in range(3)]
            err = max(abs(a - b) for a, b in zip(f, want))
            size = max(abs(b) for b in want)
            assert err <= mpmath.ldexp(size, -120) or size == 0, f"{labels[i]}: {float(err / size):.3g}"
        n += 1
    assert n >= 190


def test_oracle_tick_force_is_the_field_at_x0(oracle):
    """With v0 = 0 the Force after one tick is mass times the field at x0, for both integrators (the stage positions
    x0 + h v0 are x0): the oracle's semi-implicit and RK4 Force equal eval_stage's, value for value, NaN for NaN."""
    O = oracle
    pos, ine, _ = catalogue()
    for L, kind in ((8, "dense"), (64, "kaula")):
        c, s = tables(L, kind)
        want = oracle_field(O, pos, ine, L, c, s)
        for integ in INTEGRATORS:
            force = _oracle_tick(O, pos, ine, L, c, s, integ)[3]
            assert np.array_equal(force, want, equal_nan=True), f"{integ} L={L}"
            if integ == "semi_implicit":
                assert same_bits(force, want), f"{integ} L={L}: a zero changed sign"


# --------------------------------------------------------------------------- CPU: the bound is sensitive


@pytest.mark.parametrize("L", [0, 1, 2, 3, 8, 64, 128])
def test_f64_restatement_is_the_oracle_bit_for_bit(oracle, L):
    """The numpy restatement of egm08_field reproduces the oracle on the catalogue, bit for bit, for every table kind
    (so the faults below are faults of the kernel's own arithmetic)."""
    pos, ine, _ = catalogue()
    for kind in table_kinds(L):
        c, s = tables(L, kind)
        want = oracle_field(oracle, pos, ine, L, c, s)[..., 3:].reshape(-1, 3)
        got = f64_field(pos.reshape(-1, 7)[:, 4:], ine.reshape(-1, 7)[:, 6], L, c, s)
        assert same_bits(got, want), f"L={L} {kind}"


FAULTS = {"coef": lambda L: ("coef", 1.0 + 1e-6), "swap": lambda L: ("swap", None),
          "rho": lambda L: ("rho", 100 if L > 100 else L - 14), "mp": lambda L: ("mp", L // 2)}


@pytest.mark.parametrize("L", [64, 128])
def test_bound_rejects_faults_and_accepts_the_faithful_restatement(oracle, L):
    """Dense tables: C[L-1][L-1] scaled by 1 + 1e-6, C and S swapped for term (L-1, L-1), rho_l for rho_{l+1} at one
    degree (100 at L = 128), m for m + 1 in column L/2: each fails the bound at some body; the faithful restatement
    passes it."""
    pos, ine, labels = catalogue()
    p, m = pos.reshape(-1, 7)[:, 4:], ine.reshape(-1, 7)[:, 6]
    c, s = tables(L, "dense")
    faithful = worst_ratio(f64_field(p, m, L, c, s), L, "dense")
    print(f"\nL={L} dense: faithful restatement {faithful[0]:.3g} of the bound ({faithful[1]})")
    assert faithful[0] <= 1.0
    for name, fault in FAULTS.items():
        r = worst_ratio(f64_field(p, m, L, c, s, fault(L)), L, "dense")
        print(f"  fault {name} {fault(L)}: worst {r[0]:.3g} of the bound ({r[1]})")
        assert r[0] > 1.0, f"L={L}: the bound accepts the fault {name}"


def test_max_degree_129_is_refused_in_python():
    """GravityEGM08 checks the degree before anything reaches the C ABI."""
    c = np.zeros((130, 130))
    with pytest.raises(ValueError):
        el.B200Exec(1, 1, DT, None, [el.GravityEGM08(c, c, 129)], "rk4", "exact")
    with pytest.raises(ValueError):
        el.GravityEGM08(c, c, -1).lower(None)


# --------------------------------------------------------------------------- GPU: a direct readout of the field


def _oracle_tick(O, pos, ine, L, c, s, integ, vel=None, dt=DT, mask=None):
    M, N = pos.shape[:2]
    w = O.World(pos, np.zeros((M, N, 6)) if vel is None else vel, ine)
    e = [O.Effector(O.EFF_GRAVITY_EGM08, p=(MU_EARTH, R_EARTH, L), tables=(c, s), mask=mask)]
    threads = max(1, min(O.max_threads(), os.cpu_count() or 1))
    (w.rk4 if integ == "rk4" else w.semi_implicit)(dt, 1, e, threads=threads)
    return w.pos, w.vel, w.accel, w.force


def _gpu_tick(effs, math_mode, integ, pos, ine, vel=None, dt=DT):
    M, N = pos.shape[:2]
    with el.B200Exec(N, M, dt, None, effs, integ, math_mode) as ex:
        ex.set_state(pos, np.zeros((M, N, 6)) if vel is None else vel, ine)
        ex.step(1, sync=True)
        return tuple(ex.download(k) for k in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE))


@functools.lru_cache(maxsize=None)
def gpu_readout(L, kind, math_mode, integ, drop=False):
    """One tick of the catalogue with GRAVITY_EGM08 alone (v0 = 0); drop: row L of C and S randomised."""
    pos, ine, _ = catalogue()
    c, s = tables(L, kind)
    if drop:
        rng = np.random.default_rng(L)
        c, s = c.copy(), s.copy()
        c[L, :] = rng.normal(0, 1, L + 1)
        s[L, :] = rng.normal(0, 1, L + 1)
    return _gpu_tick([el.GravityEGM08(c, s, L)], math_mode, integ, pos, ine)


ULP_WORST = {}


@pytest.mark.gpu
@pytest.mark.parametrize("L", range(MAX_DEGREE + 1))
def test_field_readout_at_every_degree(oracle, L):
    """EXACT: pos, vel, accel and Force equal the oracle's bit for bit (NaN-ness and the sign of zeros included), and
    the Force is eval_stage's field at x0 with a zero angular part.  FAST, bodies of regular mass: the linear Force
    within 4 ulps of the oracle's per component, NaN where it is NaN.  Both integrators, every table kind.  Row L of
    C and S drops out: randomising it changes no output bit of a body with a finite field, in either mode."""
    need_gpu()
    pos, ine, labels = catalogue()
    reg = regular_mass(ine)
    flat = lambda a: a.reshape(-1, a.shape[-1])
    for kind in table_kinds(L):
        c, s = tables(L, kind)
        field = oracle_field(oracle, pos, ine, L, c, s)
        for integ in INTEGRATORS:
            want = _oracle_tick(oracle, pos, ine, L, c, s, integ)
            exact = gpu_readout(L, kind, "exact", integ)
            for q, a, b in zip(("pos", "vel", "accel", "force"), exact, want):
                assert same_bits(a, b), f"L={L} {kind} {integ} exact {q}: differs from the oracle"
            assert np.array_equal(exact[3], field, equal_nan=True), f"L={L} {kind} {integ}: Force is not the field at x0"
            assert np.all(exact[3][..., :3] == 0.0), f"L={L} {kind} {integ}: angular Force"
            fast = gpu_readout(L, kind, "fast", integ)[3][..., 3:]
            f, w = fast[reg], want[3][..., 3:][reg]
            bad = np.isnan(f) != np.isnan(w)
            assert not bad.any(), f"L={L} {kind} {integ} fast: NaN-ness differs at {np.argwhere(bad)[:5]}"
            d = ulp_distance(f, w)
            k = int(np.argmax(d)) // 3
            ULP_WORST[L] = max(ULP_WORST.get(L, 0.0), float(d.max()))
            assert d.max() <= 4, f"L={L} {kind} {integ} fast: {d.max():.0f} ulps at {np.array(labels)[reg.reshape(-1)][k]}"
    for math_mode in ("exact", "fast"):
        base, drop = gpu_readout(L, "dense", math_mode, "rk4"), gpu_readout(L, "dense", math_mode, "rk4", drop=True)
        finite = np.all(np.isfinite(base[3]), -1)
        for q, a, b in zip(("pos", "vel", "accel", "force"), base, drop):
            assert same_bits(a[finite], b[finite]), f"L={L} {math_mode}: row L of the tables changed {q}"
    print(f"\nL={L}: worst FAST Force distance {ULP_WORST[L]:.0f} ulps")


BOUND_DEGREES = (16, 64, 100, 127, 128)


@pytest.mark.gpu
@pytest.mark.parametrize("L", BOUND_DEGREES)
@pytest.mark.parametrize("kind", ["dense", "kaula"])
def test_gpu_field_within_the_high_precision_bound(L, kind):
    """The Force of every judged body (finite in-range reference) within (L + 16) 2^-53 S_k of ref_field, per
    component, in both modes and for both integrators (FAST: bodies of regular mass)."""
    need_gpu()
    _, ine, _ = catalogue()
    reg = regular_mass(ine).reshape(-1)
    for math_mode in ("exact", "fast"):
        for integ in INTEGRATORS:
            force = gpu_readout(L, kind, math_mode, integ)[3][..., 3:]
            r = worst_ratio(force, L, kind, bodies=reg if math_mode == "fast" else None)
            print(f"\nL={L} {kind} {math_mode} {integ}: worst {r[0]:.3g} of the bound ({r[1]}), "
                  f"{r[0] * bound_factor(L):.3g} x 2^-53 S_k")
            assert r[0] <= 1.0, f"L={L} {kind} {math_mode} {integ}: {r[0]:.3g} of the bound at {r[1]}"


# --------------------------------------------------------------------------- GPU: the field inside a real tick


def _orbit(L, kind, M=5, N=41):
    pos, vel, ine, _, dt = orbit_world(300 + L, M, N)
    c, s = tables(L, kind)
    return (pos, vel, ine), [("egm08", {"c_bar": c, "s_bar": s, "L": L})], dt


@pytest.mark.gpu
@pytest.mark.parametrize("L", [32, 128])
@pytest.mark.parametrize("kind", ["dense", "kaula"])
def test_rk4_tick_at_orbital_speed(oracle, L, kind):
    """One RK4 tick with v != 0 (three distinct stage positions): EXACT bit for bit, FAST per body."""
    need_gpu()
    start, spec, dt = _orbit(L, kind)
    oe, ge, _ = body_effectors(oracle, spec)
    w = oracle.World(*start).rk4(dt, 1, oe, threads=4)
    want = (w.pos, w.vel, w.accel, w.force)
    got = _gpu_tick(ge, "exact", "rk4", start[0], start[2], start[1], dt)
    for q, a, b in zip(("pos", "vel", "accel", "force"), got, want):
        assert same_bits(a, b), f"L={L} {kind} exact {q}"
    fast = _gpu_tick(ge, "fast", "rk4", start[0], start[2], start[1], dt)
    worst = assert_body_close(fast, want, start, dt, 1, body_scales(spec, *start), what=f"L={L} {kind} fast")
    print(f"\nL={L} {kind} fast: worst error / bound " + ", ".join(f"{q} {r:.3g}" for q, r in worst.items()))


@pytest.mark.gpu
@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
def test_invoke_batch_ragged_ranges_with_a_mask(oracle, math_mode, integ):
    """invoke_batch over world ranges of 2 worlds out of 5 (2, 2, 1) with the field masked to some entities."""
    need_gpu()
    L = 128
    start, spec, dt = _orbit(L, "dense")
    pos, vel, ine = start
    M, N = pos.shape[:2]
    mask = (np.random.default_rng(9).random(N) < 0.6).astype(np.uint8)
    mask[0], mask[1] = 1, 0
    spec = [("egm08", {**spec[0][1], "mask": mask})]
    oe, ge, _ = body_effectors(oracle, spec)
    w = oracle.World(*start)
    (w.rk4 if integ == "rk4" else w.semi_implicit)(dt, 1, oe, threads=4)
    want = (w.pos, w.vel, w.accel, w.force)
    with el.B200Exec(N, M, dt, None, ge, integ, math_mode, invoke_chunk_bodies=2 * N) as ex:
        table = {el.component_id("tick"): np.array([0], dtype=np.uint64), FORCE: np.zeros((M, N, 6)), INERTIA: ine,
                 WORLD_POS: pos, WORLD_ACCEL: np.zeros((M, N, 6)), el.component_id("simulation_time_step"): np.array([dt]),
                 WORLD_VEL: vel}
        out = dict(zip(ex.output_ids, ex.invoke_batch([table[k] for k in ex.input_ids], 1)))
    got = (out[WORLD_POS], out[WORLD_VEL], out[WORLD_ACCEL], out[FORCE])
    if math_mode == "exact":
        for q, a, b in zip(("pos", "vel", "accel", "force"), got, want):
            assert same_bits(a, b), f"{integ} exact {q}"
    else:
        assert_body_close(got, want, start, dt, 1, body_scales(spec, *start), what=f"{integ} fast masked")
    assert np.all(got[3][:, mask == 0] == 0.0), "an unmasked entity felt the field"


@pytest.mark.gpu
@pytest.mark.parametrize("integ", INTEGRATORS)
@pytest.mark.parametrize("math_mode", ["exact", "fast"])
def test_one_field_launch_per_tick(math_mode, integ):
    """Each tick runs one egm08_force_kernel<EXACT, RK4> of the handle's instance, then the body kernel."""
    need_gpu()
    start, spec, dt = _orbit(16, "kaula", M=3, N=41)
    _, ge, _ = body_effectors(None, spec)
    exact, r, i = math_mode == "exact", "true" if integ == "rk4" else "false", _I[integ]
    field = f"egm08_force_kernel<{'true' if exact else 'false'}, {r}>"
    body = f"body_exact_kernel<{i}, " if exact else f"body_fast_kernel<{i}, 128, 4, false>"
    ticks = 3
    for _ in range(3):  # the profiler can lose the records of a short window
        with el.B200Exec(start[0].shape[1], start[0].shape[0], dt, None, ge, integ, math_mode) as ex:
            ex.set_state(*start)
            n0 = ex.timings()["kernel_launches"]
            _, names = launched_kernels(lambda: ex.step(ticks, sync=True))
            launches = ex.timings()["kernel_launches"] - n0
        names = [n for n in names if not n.startswith(("Memcpy", "Memset"))]
        if len(names) == launches:
            break
    assert len(names) == launches, f"the profiler saw {len(names)} of {launches} launches: {names}"
    ran = assert_route(names, [field, body], f"{math_mode} {integ}")
    assert sum(n.startswith("egm08_force_kernel<") for n in ran) == ticks, ran
    assert sum(n.startswith(body) for n in ran) == ticks, ran


# --------------------------------------------------------------------------- GPU: refusals


@dataclass
class _BentEGM08(el.GravityEGM08):
    """GravityEGM08 whose lowered struct carries a degree or table length the Python check would not let through."""

    bad_degree: Optional[float] = None
    bad_len: Optional[int] = None

    def lower(self, world):
        e = super().lower(world)
        if self.bad_degree is not None:
            e.p[2] = self.bad_degree
        if self.bad_len is not None:
            e.table_len = self.bad_len
        return e


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [("degree", 129.0), ("degree", 2.5), ("degree", -1.0), ("degree", float("nan")),
                                 ("len", 80), ("len", 0), ("len", 82)], ids=str)
def test_abi_refuses_bad_degrees_and_table_lengths(bad):
    """b200_sixdof_create refuses a max_degree outside 0..128 or not an integer (B200_ERR_INVALID_ARGUMENT) and a table
    length other than (L+1)^2 (B200_ERR_VALUE_SIZE_MISMATCH); the same effector corrected then runs a tick."""
    need_gpu()
    what, value = bad
    L = 128 if what == "degree" and value > 128 else 8
    c, s = tables(L, "kaula")
    eff = _BentEGM08(c, s, L, bad_degree=value if what == "degree" else None, bad_len=value if what == "len" else None)
    pos, vel, ine, _, dt = orbit_world(5, 2, 3)
    with pytest.raises(el.B200Error) as ei:
        el.B200Exec(3, 2, dt, None, [eff], "rk4", "exact")
    want = _lib.ERR_INVALID_ARGUMENT if what == "degree" else _lib.ERR_VALUE_SIZE_MISMATCH
    assert ei.value.code == want, f"{bad}: code {ei.value.code}, expected {want}"
    eff.bad_degree = eff.bad_len = None
    with el.B200Exec(3, 2, dt, None, [eff], "rk4", "exact") as ex:
        ex.set_state(pos, vel, ine)
        ex.step(1, sync=True)
        assert np.all(np.isfinite(ex.download(FORCE)))
