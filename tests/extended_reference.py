"""A numpy restatement of one tick of the oracle, written once and parametrised by dtype.

At np.float64 it computes what oracle/sixdof_oracle.c computes (default dot mode, no contraction), bit for bit: every
sum and dot product is written term by term in the oracle's source order (no np.dot, np.sum or @, whose summation
order is not the oracle's), the edge folds run per source over its out-edges in edge-list order, and J2's sixth
power is the oracle's pow6 (a double-double product, with Dekker's exact product errors in place of fma).  The CPU
tests of tests/test_fast_long_horizon.py hold it to that over 1000 ticks.

At np.longdouble (x87 extended: 64-bit significand, 11 bits more than f64) it is the truth that the f64 runs are
judged against: the same operations, each rounded about 2000 times more finely, with 1/6 and the sixth power of J2
taken at that precision.  The inputs are the f64 inputs, exactly.

Covered: RK4 with the reference's stage quirk (DESIGN §2) and semi-implicit Euler; quaternion product, rotation and
normalisation, transform_add_motion and calc_accel; const gravity, quadratic drag (3- and 5-wide wind), body thrust,
body wrench (both layouts), world wrench, the wheel torque fold (1..8 wheels), frame gravity, J2, and edge gravity
(newton and softened, all-pairs or any edge list); entity masks.  EGM08 is left out: its stage-force kernel is the
oracle's arithmetic in both math modes (DESIGN §9), and the body-kernel half of an EGM08 list is the interpreter,
which the other interpreted lists exercise.

`Perturb` injects faults into named operations of an f64 run (each result scaled by a factor, or moved by a random
+-1 ulp): the tests use it to prove that the long-horizon bound rejects a systematic bias and tolerates noise.
"""

import numpy as np

from oracle import oracle as O

assert np.finfo(np.longdouble).nmant >= 63, "np.longdouble is not x87 extended precision (64-bit significand)"

# the named operations a Perturb can act on
# (the first nine can carry a bias; "rotate" and "normalize" are the results of every quaternion rotation and
# normalisation, which the noise model perturbs as well)
FAULTABLE = ("g", "thrust", "drag", "frame", "j2", "pair", "inv_mass", "inv_inertia", "rk4_weights")
OPERATIONS = FAULTABLE + ("rotate", "normalize")


class Perturb:
    """Faults of an f64 run: `scale` {operation: factor} multiplies each listed operation's result; `noise` (a seed)
    moves every result of the operations in `noisy` by +-1 ulp, the sign drawn per element and evaluation."""

    def __init__(self, scale=None, noise=None, noisy=OPERATIONS):
        self.scale = dict(scale or {})
        self.rng = None if noise is None else np.random.default_rng(noise)
        self.noisy = set(noisy) if noise is not None else set()

    def __call__(self, name, x):
        if name in self.scale:
            x = x * self.scale[name]
        if name in self.noisy:
            up = self.rng.random(np.shape(x)) < 0.5
            x = np.where(up, np.nextafter(x, np.inf), np.nextafter(x, -np.inf))
        return x


def _none(name, x):
    return x


# --------------------------------------------------------------------------- quaternions (components as [M, N] arrays)


def dot3(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def dot4(a, b):
    return ((a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]) + a[3] * b[3]


def qmul(l, r):
    li, lj, lk, lw = l
    ri, rj, rk, rw = r
    return (((lw * ri + li * rw) + lj * rk) - lk * rj,
            ((lw * rj - li * rk) + lj * rw) + lk * ri,
            ((lw * rk + li * rj) - lj * ri) + lk * rw,
            ((lw * rw - li * ri) - lj * rj) - lk * rk)


def qinv(q):
    n2 = dot4(q, q)
    return (-q[0] / n2, -q[1] / n2, -q[2] / n2, q[3] / n2)


def qrot(q, v, zero, pt=_none):
    """(q * [v, 0]) * q.inverse(), the inverse recomputed on every call."""
    r = qmul(qmul(q, (v[0], v[1], v[2], zero)), qinv(q))
    return tuple(pt("rotate", c) for c in r[:3])


def qnormalize(q):
    n = np.sqrt(dot4(q, q))
    return tuple(c / n for c in q)


def transform_add_motion(pos, m, zero, pt=_none):
    """q' = normalize(q + [omega/2, 0] q), x' = x + v."""
    h = (m[0] / 2.0, m[1] / 2.0, m[2] / 2.0, zero)
    hq = qmul(h, pos[:4])
    q = tuple(pt("normalize", c) for c in qnormalize(tuple(pos[k] + hq[k] for k in range(4))))
    return q + (pos[4] + m[3], pos[5] + m[4], pos[6] + m[5])


def cross3(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


# --------------------------------------------------------------------------- J2's sixth power


def _prod_err(a, b, p):
    """a * b - p exactly, for p = fl(a * b) (Dekker's product; what fma(a, b, -p) returns without over/underflow)."""
    c = 134217729.0 * a
    ah = c - (c - a)
    al = a - ah
    c = 134217729.0 * b
    bh = c - (c - b)
    bl = b - bh
    return ((ah * bh - p) + ah * bl + al * bh) + al * bl


def pow6_f64(x):
    """The oracle's pow6: x^2, x^4 and x^6 as double-double products, rounded once."""
    s = x * x
    se = _prod_err(x, x, s)
    q = s * s
    qe = _prod_err(s, s, q) + (2.0 * s) * se
    p = q * s
    pe = _prod_err(q, s, p) + ((q * se) + (qe * s))
    return p + pe


# --------------------------------------------------------------------------- the model


def _split(a, dtype):
    """[M, N, k] -> tuple of k contiguous [M, N] arrays of dtype."""
    a = np.asarray(a)
    return tuple(np.ascontiguousarray(a[..., k], dtype=dtype) for k in range(a.shape[-1]))


class _Edges:
    """Per source, its out-edges in edge-list order, padded: targets [N, D], valid [N, D]."""

    def __init__(self, edges, N):
        e = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
        e = e[(e[:, 0] < N) & (e[:, 1] < N)]
        e = e[np.argsort(e[:, 0], kind="stable")]  # grouped by source, each source's edges in list order
        count = np.bincount(e[:, 0], minlength=N)
        slot = np.arange(len(e)) - (np.cumsum(count) - count)[e[:, 0]]
        self.D = D = max(int(count.max(initial=0)), 1)
        self.target = np.zeros((N, D), dtype=np.int64)
        self.valid = np.zeros((N, D), dtype=bool)
        self.target[e[:, 0], slot] = e[:, 1]
        self.valid[e[:, 0], slot] = True
        self.has_edge = count > 0


class Model:
    """One world batch's effector list and inertia at a dtype.  effs: oracle Effector objects (tests.util
    body_effectors(None, spec)[0]), their columns [M, N, width]; ine [M, N, 7]."""

    def __init__(self, effs, ine, dtype=np.float64, perturb=None):
        self.dtype = np.dtype(dtype)
        self.f64 = self.dtype == np.float64
        self.pt = perturb or _none
        self.ine = _split(ine, dtype)
        self.M, self.N = self.ine[0].shape
        self.zero = np.zeros((self.M, self.N), dtype=dtype)
        dt = dtype
        self.effs = []
        for e in effs:
            d = {"kind": e.kind, "flags": e.flags, "p": tuple(dt(float(v)) for v in e.p),
                 "col": None if e.column is None else _split(e.column, dtype),
                 "mask": None if e.mask is None else np.asarray(e.mask, dtype=bool)[None, :]}
            if e.kind in (O.EFF_GRAVITY_EDGES_NEWTON, O.EFF_GRAVITY_EDGES_SOFTENED):
                d["edges"] = _Edges(e.edges, self.N)
            assert e.kind != O.EFF_GRAVITY_EGM08, "EGM08 is not restated (see the module docstring)"
            self.effs.append(d)

    # ---- effectors: each returns the new Force (6 arrays)

    def _gravity_const(self, e, F):
        m, pt = self.ine[6], self.pt
        return F[:3] + tuple(F[3 + k] + pt("g", e["p"][k] * m) for k in range(3))

    def _drag(self, e, vel, F):
        col, pt = e["col"], self.pt
        w = col[:3] if col is not None else (self.zero,) * 3
        fl = (w[0] - vel[3], w[1] - vel[4], w[2] - vel[5])
        speed = np.sqrt(dot3(fl, fl))
        wide = col is not None and len(col) == 5
        cd_rho, area = (col[3], col[4]) if wide else (e["p"][0], e["p"][1])
        drag = 0.5 * ((cd_rho * (speed * speed)) * area)
        d = (fl[0] / speed, fl[1] / speed, fl[2] / speed)
        z = self.zero
        return (z, z, z) + tuple(F[3 + k] + pt("drag", drag * d[k]) for k in range(3))

    def _thrust(self, e, pos, F):
        t = e["col"][0] if e["col"] is not None else self.zero
        d = qrot(pos[:4], e["p"][:3], self.zero, self.pt)
        return F[:3] + tuple(F[3 + k] + self.pt("thrust", d[k] * t) for k in range(3))

    def _wrench_body(self, e, pos, F):
        wr = e["col"] if e["col"] is not None else (self.zero,) * 6
        q = pos[:4]
        if e["flags"] & O.FLAG_WRENCH_LINEAR_FIRST:
            tw, fw = qrot(q, wr[3:6], self.zero, self.pt), qrot(q, wr[0:3], self.zero, self.pt)
        else:
            tw, fw = qrot(q, wr[0:3], self.zero, self.pt), qrot(q, wr[3:6], self.zero, self.pt)
        return tuple(F[k] + tw[k] for k in range(3)) + tuple(F[3 + k] + fw[k] for k in range(3))

    def _wrench_world(self, e, F):
        if e["col"] is None:
            return F
        return tuple(F[k] + e["col"][k] for k in range(6))

    def _torque_fold(self, e, pos, F):
        col = e["col"]
        if col is None:
            return F
        z = self.zero
        acc = (z, z, z)
        for k in range(len(col) // 3):
            t = qrot(pos[:4], col[3 * k:3 * k + 3], z, self.pt)
            acc = (acc[0] + t[0], acc[1] + t[1], acc[2] + t[2])
        return acc + (z + 0.0, z + 0.0, z + 0.0)

    def _gravity_frame(self, e, pos, vel, F):
        mu, om = e["p"][0], e["p"][1:4]
        r, v, m = pos[4:7], vel[3:6], self.ine[6]
        rn = np.sqrt(dot3(r, r))
        rn3 = (rn * rn) * rn
        g = tuple(((-mu) * r[k]) / rn3 for k in range(3))
        c = cross3(om, v)
        c2 = cross3(om, cross3(om, r))
        acc = tuple(g[k] + (-2.0 * c[k] + (-c2[k])) for k in range(3))
        return F[:3] + tuple(F[3 + k] + self.pt("frame", acc[k] * m) for k in range(3))

    def _gravity_j2(self, e, pos, F):
        mu, J2, r_ref = e["p"][:3]
        r, m = pos[4:7], self.ine[6]
        z = r[2]
        norm = np.sqrt(dot3(r, r))
        e_r = (r[0] / norm, r[1] / norm, r[2] / norm)
        n3 = (norm * norm) * norm
        c0 = (-mu) * m
        n2 = norm * norm
        n4 = n2 * n2
        n5 = norm * n4
        n6 = pow6_f64(norm) if self.f64 else np.power(norm, self.dtype.type(6))
        kz = (3.0 * z) / n5
        kr = 3.0 / (2.0 * n4) - (15.0 * (z * z)) / (2.0 * n6)
        c1 = (c0 * J2) * (r_ref * r_ref)
        e_z = (0.0, 0.0, 1.0)
        out = []
        for k in range(3):
            f = (c0 * r[k]) / n3
            j2 = c1 * (kz * e_z[k] + kr * e_r[k])
            out.append(F[3 + k] + self.pt("j2", f + j2))
        return F[:3] + tuple(out)

    def _gravity_edges(self, e, pos, F):
        """Per source, the left fold over its out-edges from a zero Force; the result replaces the source's Force."""
        ed, pt = e["edges"], self.pt
        x, m = pos[4:7], self.ine[6]
        if "term" not in e:  # [3, D, M, N]: edge j of every source, reused by every stage
            e["term"] = np.empty((3, ed.D, self.M, self.N), dtype=self.dtype)
        term = e["term"]
        B = max(1, (1 << 15) // (ed.D * self.M))  # sources per block: a block's temporaries stay in cache
        for a0 in range(0, self.N, B):
            a1 = min(self.N, a0 + B)
            tg = ed.target[a0:a1]  # [b, D]
            xa = [c[:, a0:a1, None] for c in x]
            xb = [c[:, tg] for c in x]  # [M, b, D]
            ma, mb = m[:, a0:a1, None], m[:, tg]
            with np.errstate(divide="ignore", invalid="ignore"):  # padding (and a newton self-edge) divide 0 by 0
                if e["kind"] == O.EFF_GRAVITY_EDGES_SOFTENED:
                    K2, soft = e["p"][:2]
                    r = [xb[k] - xa[k] for k in range(3)]
                    dist_sq = dot3(r, r) + soft
                    inv = 1.0 / np.sqrt(dist_sq)
                    inv3 = (inv * inv) * inv
                    scalar = ((K2 * ma) * mb) * inv3
                    t = [pt("pair", scalar * r[k]) for k in range(3)]
                else:
                    G = e["p"][0]
                    r = [xa[k] - xb[k] for k in range(3)]
                    norm = np.sqrt(dot3(r, r))
                    s = (G * mb) * ma
                    d = (norm * norm) * norm
                    t = [-pt("pair", (s * r[k]) / d) for k in range(3)]  # acc - t == acc + (-t)
            for k in range(3):
                tk = np.where(ed.valid[a0:a1], t[k], 0.0)  # a padded edge adds +0
                term[k, :, :, a0:a1] = np.moveaxis(tk, 2, 0)
        acc = [self.zero.copy() for _ in range(3)]
        for j in range(ed.D):
            for k in range(3):
                acc[k] = acc[k] + term[k, j]
        he = ed.has_edge[None, :]
        z = self.zero
        return tuple(np.where(he, z, F[k]) for k in range(3)) + tuple(np.where(he, acc[k], F[3 + k]) for k in range(3))

    def forces(self, pos, vel):
        """clear_forces, then the effectors in list order: the Force (6 arrays)."""
        z = self.zero
        F = (z,) * 6
        for e in self.effs:
            kind = e["kind"]
            if kind in (O.EFF_GRAVITY_EDGES_NEWTON, O.EFF_GRAVITY_EDGES_SOFTENED):
                F = self._gravity_edges(e, pos, F)
                continue
            if kind == O.EFF_GRAVITY_CONST:
                new = self._gravity_const(e, F)
            elif kind == O.EFF_DRAG_QUADRATIC:
                new = self._drag(e, vel, F)
            elif kind == O.EFF_THRUST_BODY:
                new = self._thrust(e, pos, F)
            elif kind == O.EFF_WRENCH_BODY:
                new = self._wrench_body(e, pos, F)
            elif kind == O.EFF_GRAVITY_FRAME:
                new = self._gravity_frame(e, pos, vel, F)
            elif kind == O.EFF_WRENCH_WORLD:
                new = self._wrench_world(e, F)
            elif kind == O.EFF_TORQUE_BODY_FOLD:
                new = self._torque_fold(e, pos, F)
            elif kind == O.EFF_GRAVITY_J2:
                new = self._gravity_j2(e, pos, F)
            else:
                raise KeyError(kind)
            if e["mask"] is not None:
                new = tuple(np.where(e["mask"], a, b) for a, b in zip(new, F))
            F = new
        return F

    def calc_accel(self, pos, F):
        q, ine, pt, z = pos[:4], self.ine, self.pt, self.zero
        qi = qinv(q)
        tb = qrot(qi, F[:3], z, self.pt)
        fb = qrot(qi, F[3:], z, self.pt)
        ab_lin = tuple(pt("inv_mass", fb[k] / ine[6]) for k in range(3))
        ab_ang = tuple(pt("inv_inertia", tb[k] / ine[k]) for k in range(3))
        return qrot(q, ab_ang, z, self.pt) + qrot(q, ab_lin, z, self.pt)

    def stage(self, pos, vel):
        F = self.forces(pos, vel)
        return F, self.calc_accel(pos, F)

    # ---- integrators: state = (pos 7, vel 6, accel 6, force 6), tuples of [M, N] arrays

    def rk4(self, state, dt_stage, dt_final):
        pos, vel, accel, _ = state
        t = self.dtype.type
        dt_stage, dt_final = t(dt_stage), t(dt_final)
        sa, sf = accel, None
        kv = ka = None
        for s, fac in enumerate((0.0, 0.5, 0.5, 1.0)):
            dtf = dt_stage * fac
            sx = transform_add_motion(pos, tuple(dtf * c for c in vel), self.zero, self.pt)
            sv = tuple(vel[k] + dtf * sa[k] for k in range(6))
            sf, sa = self.stage(sx, sv)
            if s == 0:
                kv, ka = sv, sa
            elif s == 3:
                kv = tuple(kv[k] + sv[k] for k in range(6))
                ka = tuple(ka[k] + sa[k] for k in range(6))
            else:
                kv = tuple(kv[k] + 2.0 * sv[k] for k in range(6))
                ka = tuple(ka[k] + 2.0 * sa[k] for k in range(6))
        c = dt_final * (t(1) / t(6))
        kv = tuple(self.pt("rk4_weights", a) for a in kv)
        ka = tuple(self.pt("rk4_weights", a) for a in ka)
        pos = transform_add_motion(pos, tuple(c * a for a in kv), self.zero, self.pt)
        vel = tuple(vel[k] + c * ka[k] for k in range(6))
        return pos, vel, sa, sf

    def semi_implicit(self, state, dt):
        pos, vel, _, _ = state
        dt = self.dtype.type(dt)
        F, A = self.stage(pos, vel)
        vel = tuple(vel[k] + dt * A[k] for k in range(6))
        pos = transform_add_motion(pos, tuple(dt * c for c in vel), self.zero, self.pt)
        return pos, vel, A, F


def stack(state):
    """A state of component tuples as [M, N, 7 | 6] arrays (pos, vel, accel, force)."""
    return tuple(np.stack(part, -1) for part in state)


def run(start, effs, integ, dt, ticks, dtype=np.float64, every=None, perturb=None, accel=None):
    """(pos, vel, accel, force) [M, N, k] arrays after `ticks` ticks from start = (pos, vel, ine) (accel: the
    WorldAccel column before the first tick, default zero); with `every`, the list of states after every `every`
    ticks instead."""
    pos, vel, ine = start
    model = Model(effs, ine, dtype, perturb)
    M, N = model.M, model.N
    z6 = np.zeros((M, N, 6)) if accel is None else accel
    state = (_split(pos, dtype), _split(vel, dtype), _split(z6, dtype), _split(np.zeros((M, N, 6)), dtype))
    out = []
    for t in range(1, ticks + 1):
        state = model.rk4(state, dt, dt) if integ == "rk4" else model.semi_implicit(state, dt)
        if every and t % every == 0:
            out.append(stack(state))
    return out if every else stack(state)
