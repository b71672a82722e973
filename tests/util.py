"""Shared helpers for the parity tests: seeded synthetic worlds (SURVEY §8d) and
the oracle <-> C-ABI effector translation."""

import re

import numpy as np

import elodin_b200 as el


def random_world(seed, M, N, unit_q=True):
    """q ~ normalised N(0,1)^4, x ~ U(-1e3,1e3), omega ~ N(0,.5), v ~ N(0,10),
    inertia diag ~ U(.1,10), m ~ U(.5,50)  (SURVEY §8d synthetic inputs)."""
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(M, N, 4))
    if unit_q:
        q /= np.linalg.norm(q, axis=-1, keepdims=True)
    pos = np.concatenate([q, rng.uniform(-1e3, 1e3, (M, N, 3))], -1)
    vel = np.concatenate([rng.normal(0, 0.5, (M, N, 3)), rng.normal(0, 10, (M, N, 3))], -1)
    ine = np.concatenate([rng.uniform(0.1, 10, (M, N, 3)), np.zeros((M, N, 3)), rng.uniform(0.5, 50, (M, N, 1))], -1)
    return np.ascontiguousarray(pos), np.ascontiguousarray(vel), np.ascontiguousarray(ine)


def effector_pair(O, kind, **kw):
    """(oracle effector, elodin_b200 effector, {column name: array}) for one built-in kind."""
    if kind == "gravity":
        g = kw.get("g", (0.0, 0.0, -9.81))
        return O.Effector(O.EFF_GRAVITY_CONST, p=g), el.GravityConst(g), {}
    if kind == "drag":  # a wind column of width 5 carries per-body [Cd*rho, area] after the wind
        wind = kw["wind"]
        cd, area = kw.get("cd_rho", 0.6125), kw.get("area", 0.25)
        return (O.Effector(O.EFF_DRAG_QUADRATIC, p=(cd, area), column=wind),
                el.DragQuadratic(cd, area, "wind", per_body_params=wind.shape[-1] == 5), {"wind": wind})
    if kind == "thrust":
        thrust, name = kw["thrust"], kw.get("name", "thrust")
        axis = kw.get("axis", (-1.0, 0.0, 0.0))
        return (O.Effector(O.EFF_THRUST_BODY, p=axis, column=thrust), el.ThrustBody(axis, name), {name: thrust})
    if kind == "wrench":
        wr = kw["wrench"]
        lin_first = kw.get("linear_first", False)
        return (O.Effector(O.EFF_WRENCH_BODY, flags=O.FLAG_WRENCH_LINEAR_FIRST if lin_first else 0, column=wr),
                el.WrenchBody("aero_force", "linear_first" if lin_first else "torque_first"), {"aero_force": wr})
    if kind == "frame":
        mu, om = kw.get("mu", 3.986004418e14), kw.get("omega", (0.0, 0.0, 7.292115e-5))
        return O.Effector(O.EFF_GRAVITY_FRAME, p=(mu, *om)), el.GravityFrame(mu, om), {}
    if kind == "wrench_world":
        wr = kw["wrench"]
        return O.Effector(O.EFF_WRENCH_WORLD, column=wr), el.WrenchWorld("external_force"), {"external_force": wr}
    if kind == "wheels":
        tq = kw["torques"]
        return (O.Effector(O.EFF_TORQUE_BODY_FOLD, column=tq), el.TorqueBodyFold("wheel_torques", tq.shape[-1] // 3),
                {"wheel_torques": tq})
    if kind == "j2":
        mu, j2, rr = kw.get("mu", 3.986004418e14), kw.get("j2", 1.08262668e-3), kw.get("r_ref", 6.378e6)
        return O.Effector(O.EFF_GRAVITY_J2, p=(mu, j2, rr)), el.GravityJ2(mu, j2, rr), {}
    if kind == "egm08":
        c, s, L = kw["c_bar"], kw["s_bar"], kw["L"]
        mu, rr = kw.get("mu", 3.986004418e14), kw.get("r_ref", 6.378e6)
        return O.Effector(O.EFF_GRAVITY_EGM08, p=(mu, rr, L), tables=(c, s)), el.GravityEGM08(c, s, L, mu, rr), {}
    if kind == "newton":
        return (O.Effector(O.EFF_GRAVITY_EDGES_NEWTON, p=(kw.get("G", 6.6743e-11),), edges=kw["edges"]),
                el.GravityEdges("newton", G=kw.get("G", 6.6743e-11), edges=kw["edges"]), {})
    if kind == "softened":
        k2, soft = kw.get("k2", 1e-3), kw.get("soft", 1e-10)
        return (O.Effector(O.EFF_GRAVITY_EDGES_SOFTENED, p=(k2, soft), edges=kw["edges"]),
                el.GravityEdges("softened", k_squared=k2, softening=soft, edges=kw["edges"]), {})
    raise KeyError(kind)


def max_rel(a, b):
    """max |a-b| / max(|b|) per trailing vector block — the vector-scaled relative error."""
    a, b = np.asarray(a), np.asarray(b)
    scale = np.maximum(np.max(np.abs(b), axis=-1, keepdims=True), 1e-300)
    return float(np.max(np.abs(a - b) / scale))


# --------------------------------------------------------------------------- FAST n-body parity, body by body

EPS = np.finfo(np.float64).eps
ULPS_PER_TICK = 8  # rounding of the stored state: a few ulps per tick, whatever the gravity


def nbody_pair_scale(pos, ine, k, soft):
    """S_i = sum_j |a_ij|: the absolute sum of body i's pair accelerations k m_j r_ij / (|r_ij|^2 + soft)^1.5 at the
    positions `pos` [M, N, 7].  It bounds the rounding of a reordered gravity sum and does not collapse when the
    forces on a body cancel.  Returns [M, N]."""
    x, m = pos[..., 4:], ine[..., 6]
    M, N = m.shape
    out = np.empty((M, N))
    step = max(1, (1 << 22) // max(N * N, 1))
    for w0 in range(0, M, step):
        xs, ms = x[w0:w0 + step], m[w0:w0 + step]
        r = xs[:, None, :, :] - xs[:, :, None, :]  # [w, i, j, 3]
        d = np.sqrt(np.sum(r * r, -1))
        with np.errstate(divide="ignore", invalid="ignore"):  # the self pair (soft = 0) is dropped below
            a = k * ms[:, None, :] * d / (d * d + soft) ** 1.5
        a[:, np.arange(N), np.arange(N)] = 0.0
        out[w0:w0 + step] = np.sum(a, -1)
    return out


def graph_pair_scale(pos, ine, edges, kind, k, soft):
    """S_i = sum over body i's out-edges (i, j), with multiplicity, of |a_ij| = k m_j |r_ij| / (|r_ij|^2 + soft)^1.5
    at the positions `pos` [M, N, 7]; kind "newton" has no softening.  A self-edge contributes 0 (softened: r = 0;
    Newton divides 0 by 0, which no bound can cover).  Returns [M, N]."""
    x, m = pos[..., 4:], ine[..., 6]
    out = np.zeros(m.shape)
    e = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
    if len(e) == 0:
        return out
    soft = 0.0 if kind == "newton" else soft
    a, b = e[:, 0], e[:, 1]
    r = x[:, b] - x[:, a]  # [M, E, 3]
    d = np.sqrt(np.sum(r * r, -1))
    with np.errstate(divide="ignore", invalid="ignore"):
        acc = k * m[:, b] * d / (d * d + soft) ** 1.5
    acc[:, a == b] = 0.0
    np.add.at(out, (slice(None), a), acc)
    return out


def nbody_world(seed, M, N, dt, kick=1e-2, size=1.0, speed=1.0, soft=1e-2, edges=None, kind="softened"):
    """A gravity world where a tick's gravity is visible at FAST tolerance: positions in a cube of `size`, linear
    speeds ~ `speed`, and the gravity constant k scaled so that the median body with an out-edge gets a kick of
    `kick` * |v| per tick.  A tick moves a body by dt * speed, which must be at least 1e-5 of the cube, so that
    gravity evaluated at the wrong stage position differs visibly.  The graph is all pairs (softened), or the
    `edges` of `kind` (graph_pair_scale).  Attitude, angular velocity and inertia come from random_world.
    Returns (pos, vel, ine, k, soft, S)."""
    assert dt * speed >= 1e-5 * size
    pos, vel, ine = random_world(seed, M, N)
    rng = np.random.default_rng(seed + 1)
    pos[..., 4:] = rng.uniform(-size, size, (M, N, 3))
    vel[..., 3:] = rng.normal(0, speed / np.sqrt(3), (M, N, 3))
    S1 = nbody_pair_scale(pos, ine, 1.0, soft) if edges is None else graph_pair_scale(pos, ine, edges, kind, 1.0, soft)
    live = S1[S1 > 0]
    k = kick * np.median(np.linalg.norm(vel[..., 3:], axis=-1)) / (dt * np.median(live)) if live.size else 1.0
    return pos, vel, ine, k, soft, k * S1


def assert_nbody_close(got, want, start, dt, n_ticks, S, tol=1e-12, what=""):
    """FAST n-body parity per body, on what the run changed.

    got / want: (WorldPos, WorldVel, WorldAccel, Force) after `n_ticks` ticks of `dt` from start = (pos, vel, ine);
    S: nbody_pair_scale at the start positions.  For every body i, with T = n_ticks:
      * dv = v_T - v_0 (linear): |dv - dv_ref| <= T (tol dt S_i + ulps of |v_T| and of dt |a|)
      * dx = x_T - x_0 - T dt v_0:  |dx - dx_ref| <= T (tol T dt^2 S_i + ulps of |x_T| and of dt |v_T|)
      * the last tick's stage-4 linear accel within tol S_i (+ ulps), Force within tol m_i S_i (+ ulps)
      * the attitude within a few ulps per tick, the angular velocity within T tol of the body's own, and the
        angular parts of accel / Force within tol of the body's own magnitude.
    Returns {quantity: worst error / bound} (every entry <= 1)."""
    pos0, vel0, ine = start
    T = n_ticks
    m = ine[..., 6]
    u = ULPS_PER_TICK * EPS
    inf = lambda a: np.max(np.abs(a), axis=-1)
    (gp, gv, ga, gf), (wp, wv, wa, wf) = got, want
    dv_g, dv_w = gv[..., 3:] - vel0[..., 3:], wv[..., 3:] - vel0[..., 3:]
    lin0 = pos0[..., 4:] + T * dt * vel0[..., 3:]
    dx_g, dx_w = gp[..., 4:] - lin0, wp[..., 4:] - lin0
    checks = {
        "dv": (inf(dv_g - dv_w), T * (tol * dt * S + u * (inf(wv[..., 3:]) + dt * inf(wa[..., 3:])))),
        "dx": (inf(dx_g - dx_w), T * (tol * T * dt * dt * S + u * (inf(wp[..., 4:]) + dt * inf(wv[..., 3:])))),
        "accel": (inf(ga[..., 3:] - wa[..., 3:]), tol * S + u * inf(wa[..., 3:])),
        "force": (inf(gf[..., 3:] - wf[..., 3:]), tol * m * S + u * inf(wf[..., 3:])),
        "q": (inf(gp[..., :4] - wp[..., :4]), np.full(m.shape, T * u)),  # unit quaternion: ulps per tick
        "omega": (inf(gv[..., :3] - wv[..., :3]), T * tol * np.maximum(inf(wv[..., :3]), 1e-300)),
        "accel_ang": (inf(ga[..., :3] - wa[..., :3]), tol * np.maximum(inf(wa[..., :3]), 1e-300)),
        "force_ang": (inf(gf[..., :3] - wf[..., :3]), tol * np.maximum(inf(wf[..., :3]), 1e-300)),
    }
    worst = {}
    for name, (err, bound) in checks.items():
        assert np.all(np.isfinite(err)), f"{what} {name}: non-finite result"
        ratio = err / bound
        i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        worst[name] = float(ratio[i])
        assert ratio[i] <= 1.0, (f"{what} {name}: body (world {i[0]}, entity {i[1]}) error {err[i]:.3e} > bound {bound[i]:.3e} "
                                 f"({ratio[i]:.3g}x); T dt S_i = {T * dt * S[i]:.3e}")
    return worst


# --------------------------------------------------------------------------- FAST body kernels, body by body

# the terms each built-in effector kind adds to a body's acceleration; frame gravity and J2 split into the parts whose
# errors a kernel can make independently
BODY_TERMS = {"gravity": ("g",), "thrust": ("thrust",), "drag": ("drag",), "wrench": ("wrench_force", "wrench_torque"),
              "wrench_world": ("world_force", "world_torque"), "frame": ("central", "coriolis", "centrifugal"),
              "j2": ("j2_central", "j2"), "wheels": ("wheels",), "egm08": ("egm08",),
              "softened": ("graph",), "newton": ("graph",)}
GRAPH_KINDS = ("softened", "newton")
ANGULAR_TERMS = ("wrench_torque", "world_torque", "wheels")
MU_EARTH, OMEGA_EARTH, J2_EARTH, R_EARTH = 3.986004418e14, (0.0, 0.0, 7.292115e-5), 1.08262668e-3, 6.378e6


def body_effectors(O, spec):
    """(oracle effectors, elodin_b200 effectors, columns) of an effector list [(kind, kwargs)], as effector_pair
    builds them; a kwarg `mask` ([N] 0/1) restricts an effector to those entities (query join).  O = None: the
    oracle module's effector descriptions without loading its library."""
    if O is None:
        from oracle import oracle as O
    oe, ge, cols = [], [], {}
    for kind, kw in spec:
        kw = dict(kw)
        mask = kw.pop("mask", None)
        a, b, c = effector_pair(O, kind, **kw)
        if mask is not None:
            a.mask = np.asarray(mask, dtype=np.uint8)
            b = b.with_mask(np.asarray(mask, dtype=np.uint8))
        oe.append(a); ge.append(b); cols.update(c)
    return oe, ge, cols


def body_terms(spec):
    """[(effector index, term)] of the terms of `spec` that reach the Force.  The wheel fold overwrites everything
    accumulated before it, and a drag resets the torque accumulated before it (both as the reference does).  The
    edge-fold gravity overwrites the Force of the bodies with an out-edge; FAST math takes it only first in the list,
    where nothing precedes it, so it is one more additive term there (lists with it later are compared bit for bit)."""
    terms = []
    for i, (kind, _) in enumerate(spec):
        assert kind not in GRAPH_KINDS or i == 0, "the edge-fold gravity must be the first effector of a FAST list"
        if kind == "wheels":
            terms = []
        if kind == "drag":
            terms = [t for t in terms if t[1] not in ANGULAR_TERMS]
        terms += [(i, t) for t in BODY_TERMS[kind]]
    return terms


def _norm(a):
    return np.sqrt(np.sum(a * a, -1))


def _qrot_inv(q, v):
    """R(q)^-1 v for unit quaternions q = (i, j, k, w)."""
    qv, w = -q[..., :3], q[..., 3:4]
    t = 2.0 * np.cross(qv, v)
    return v + w * t + np.cross(qv, t)


def body_term_accels(kind, kw, term, pos, vel, ine):
    """(|linear acceleration|, |angular acceleration|) [M, N] that one term alone gives each body at the state
    (pos, vel).  The angular part is |tau_body .* I^-1|, the torque taken into the body frame."""
    x, v, m, inv_i = pos[..., 4:], vel[..., 3:], ine[..., 6], 1.0 / ine[..., :3]
    zero = np.zeros(m.shape)
    r = _norm(x)
    if term == "g":
        return np.full(m.shape, float(np.linalg.norm(kw.get("g", (0.0, 0.0, -9.81))))), zero
    if term == "thrust":
        return float(np.linalg.norm(kw.get("axis", (-1.0, 0.0, 0.0)))) * np.abs(kw["thrust"][..., 0]) / m, zero
    if term == "drag":
        col = kw["wind"]
        kd = 0.5 * (col[..., 3] * col[..., 4] if col.shape[-1] == 5 else kw.get("cd_rho", 0.6125) * kw.get("area", 0.25))
        rel = col[..., :3] - v
        return kd * np.sum(rel * rel, -1) / m, zero
    if term in ("wrench_force", "wrench_torque"):
        wr, lf = kw["wrench"], kw.get("linear_first", False)
        f, t = (wr[..., :3], wr[..., 3:]) if lf else (wr[..., 3:], wr[..., :3])
        return (_norm(f) / m, zero) if term == "wrench_force" else (zero, _norm(t * inv_i))
    if term == "world_force":
        return _norm(kw["wrench"][..., 3:]) / m, zero
    if term == "world_torque":
        return zero, _norm(_qrot_inv(pos[..., :4], kw["wrench"][..., :3]) * inv_i)
    if term == "wheels":
        tq = kw["torques"]
        return zero, _norm(sum(tq[..., 3 * k:3 * k + 3] for k in range(tq.shape[-1] // 3)) * inv_i)
    if term in ("central", "j2_central"):
        return kw.get("mu", MU_EARTH) / (r * r), zero
    if term in ("coriolis", "centrifugal"):
        om = np.broadcast_to(np.asarray(kw.get("omega", OMEGA_EARTH), dtype=np.float64), x.shape)
        if term == "coriolis":
            return _norm(2.0 * np.cross(om, v)), zero
        return _norm(np.cross(om, np.cross(om, x))), zero
    if term == "j2":  # mu J2 r_ref^2 | 3 z/n^5 e_z + (3/(2 n^4) - 15 z^2/(2 n^6)) r/n |   (j2.py)
        z = x[..., 2]
        k = (1.5 / r ** 4 - 7.5 * z * z / r ** 6) / r
        vec = k[..., None] * x
        vec[..., 2] += 3.0 * z / r ** 5
        return kw.get("mu", MU_EARTH) * kw.get("j2", J2_EARTH) * kw.get("r_ref", R_EARTH) ** 2 * _norm(vec), zero
    if term == "egm08":  # the series sum_n (r_ref/r)^n sum_m |C_nm| + |S_nm|, each term bounded by (n + 1) mu/r^2
        c, s, L = kw["c_bar"], kw["s_bar"], kw["L"]
        ratio = kw.get("r_ref", R_EARTH) / r
        series = sum((n + 1) * ratio ** n * (np.sum(np.abs(c[n, :n + 1])) + np.sum(np.abs(s[n, :n + 1])))
                     for n in range(L + 1))
        return kw.get("mu", MU_EARTH) / (r * r) * series, zero
    if term == "graph":  # sum over the body's out-edges of |a_ij| (graph_pair_scale), at the start positions
        k = kw.get("k2", 1e-3) if kind == "softened" else kw.get("G", 6.6743e-11)
        return graph_pair_scale(pos, ine, kw["edges"], kind, k, kw.get("soft", 1e-10)), zero
    raise KeyError(term)


def _term_torque(kind, kw, term, pos):
    """|tau| [M, N] of a torque term (0 for the others): the rotation-invariant size of the torque it applies."""
    if term == "wrench_torque":
        wr = kw["wrench"]
        return _norm(wr[..., 3:] if kw.get("linear_first", False) else wr[..., :3])
    if term == "world_torque":
        return _norm(kw["wrench"][..., :3])
    if term == "wheels":
        tq = kw["torques"]
        return _norm(sum(tq[..., 3 * k:3 * k + 3] for k in range(tq.shape[-1] // 3)))
    return np.zeros(pos.shape[:2])


def body_scales(spec, pos, vel, ine):
    """(A, B, C) [M, N]: the absolute sums over the terms of `spec` of each term's linear (A) and angular (B)
    acceleration at the start state, and of each torque term's |tau| (C).  They scale the FAST tolerance body by
    body: a reordered or fused sum of the terms rounds relative to A, not to the (possibly cancelling) total."""
    A, B, C = (np.zeros(ine.shape[:2]) for _ in range(3))
    for i, term in body_terms(spec):
        kind, kw = spec[i]
        lin, ang = body_term_accels(kind, kw, term, pos, vel, ine)
        tau = _term_torque(kind, kw, term, pos)
        mask = kw.get("mask")
        if mask is not None:
            lin, ang, tau = (a * np.asarray(mask)[None, :] for a in (lin, ang, tau))
        A, B, C = A + lin, B + ang, C + tau
    return A, B, C


def assert_body_close(got, want, start, dt, n_ticks, scales, tol=1e-12, what="", check=True):
    """FAST body-kernel parity per body, on what the run changed.

    got / want: (WorldPos, WorldVel, WorldAccel, Force) after `n_ticks` ticks of (final) step `dt` from start =
    (pos, vel, ine); scales = body_scales(...) = (A, B, C).  For body i, with T = n_ticks and u = 8 ulps per tick:
      * dv = v_T - v_0 (linear):       T (tol dt A_i + u (|v_T| + dt A_i))
      * dx = x_T - x_0 - T dt v_0:     T (tol T dt^2 A_i + u (|x_T| + dt |v_T|))
      * dw = w_T - w_0 (angular):      T (tol dt B_i + u (|w_T| + dt B_i))
      * the attitude q:                T u + T^2 dt^2 tol B_i / 2
      * stage-4 WorldAccel:            tol A_i + u |a| (linear), tol B_i + u |alpha| (angular)
      * Force:                         m_i (tol A_i) + u |F| (linear), tol C_i + u |tau| (angular; C_i = sum of the
                                       terms' |tau|, i.e. B_i with each component multiplied by its own I_i)
    The linear and angular parts are separate checks.  Returns {quantity: worst error / bound} (every entry <= 1;
    check=False returns the ratios without asserting, for the self-tests that measure how far a fault lands)."""
    ine = start[2]  # the start state enters through the scales: the differences below are differences of changes
    A, B, C = scales
    T = n_ticks
    m = ine[..., 6]
    u = ULPS_PER_TICK * EPS
    inf = lambda a: np.max(np.abs(a), axis=-1)
    (gp, gv, ga, gf), (wp, wv, wa, wf) = got, want
    checks = {
        "dv": (inf(gv[..., 3:] - wv[..., 3:]), T * (tol * dt * A + u * (inf(wv[..., 3:]) + dt * A))),
        # x_T - x_0 - T dt v_0 is the same shift on both sides: the difference is gp - wp, and its size is weighed
        # against the displacement the forces drove (A_i) plus the ulps of |x_T|
        "dx": (inf(gp[..., 4:] - wp[..., 4:]), T * (tol * T * dt * dt * A + u * (inf(wp[..., 4:]) + dt * inf(wv[..., 3:])))),
        "dw": (inf(gv[..., :3] - wv[..., :3]), T * (tol * dt * B + u * (inf(wv[..., :3]) + dt * B))),
        "q": (inf(gp[..., :4] - wp[..., :4]), T * u + 0.5 * T * T * dt * dt * tol * B),
        "accel": (inf(ga[..., 3:] - wa[..., 3:]), tol * A + u * inf(wa[..., 3:])),
        "accel_ang": (inf(ga[..., :3] - wa[..., :3]), tol * B + u * inf(wa[..., :3])),
        "force": (inf(gf[..., 3:] - wf[..., 3:]), tol * m * A + u * inf(wf[..., 3:])),
        "force_ang": (inf(gf[..., :3] - wf[..., :3]), tol * C + u * inf(wf[..., :3])),
    }
    worst = {}
    for name, (err, bound) in checks.items():
        assert np.all(np.isfinite(err)), f"{what} {name}: non-finite result"
        ratio = np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0)
        i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        worst[name] = float(ratio[i])
        assert not check or ratio[i] <= 1.0, (f"{what} {name}: body (world {i[0]}, entity {i[1]}) error {err[i]:.3e} > bound "
                                              f"{bound[i]:.3e} ({ratio[i]:.3g}x); A_i = {A[i]:.3e}, B_i = {B[i]:.3e}")
    return worst


def near_world(seed, M, N):
    """A world for the effectors that act near the origin (g, thrust, drag, wrench, wheels, world wrench):
    random_world's state (|x| <= 1e3 m, |v| ~ 17 m/s), dt = 0.01, and effector columns whose every term moves a
    body's velocity far above its own ulps: thrust and wrench forces give 2..20 m/s^2, torques about 2 rad/s^2,
    and the wind differs from the body velocity by 2..10 m/s.  Returns (pos, vel, ine, columns, dt)."""
    pos, vel, ine = random_world(seed, M, N)
    rng = np.random.default_rng(seed + 1)
    m, i3 = ine[..., 6:7], ine[..., :3]
    d = rng.normal(size=(M, N, 3))
    wind = vel[..., 3:] + d / np.linalg.norm(d, axis=-1, keepdims=True) * rng.uniform(2.0, 10.0, (M, N, 1))
    cols = {
        "thrust": rng.uniform(2.0, 20.0, (M, N, 1)) * m,
        "thrust2": rng.uniform(2.0, 20.0, (M, N, 1)) * m,
        "wind": wind,
        "wind_pb": np.concatenate([wind, rng.uniform(0.3, 0.9, (M, N, 1)), rng.uniform(0.05, 0.5, (M, N, 1))], -1),
        "wrench": np.concatenate([rng.normal(0, 2, (M, N, 3)) * i3, rng.normal(0, 5, (M, N, 3)) * m], -1),
        "wrench_world": np.concatenate([rng.normal(0, 2, (M, N, 3)) * i3, rng.normal(0, 5, (M, N, 3)) * m], -1),
        "wheels": rng.normal(0, 1, (M, N, 9)) * np.tile(i3, 3),
    }
    return pos, vel, ine, cols, 0.01


def orbit_world(seed, M, N):
    """A world for frame gravity and J2: |x| = 6.9e6 m (+-2 %), orbital speeds (7.6 km/s across the radius, plus
    50 m/s at random) and dt = 1 s, so that the central, Coriolis, centrifugal and J2 terms each move a tick's dv
    and dx far above the ulps of |v| and |x|.  Attitude, angular velocity and inertia come from random_world.
    Returns (pos, vel, ine, columns, dt)."""
    pos, vel, ine = random_world(seed, M, N)
    rng = np.random.default_rng(seed + 1)
    m, i3 = ine[..., 6:7], ine[..., :3]
    x = rng.normal(size=(M, N, 3))
    x /= np.linalg.norm(x, axis=-1, keepdims=True)
    pos[..., 4:] = x * 6.9e6 * rng.uniform(0.98, 1.02, (M, N, 1))
    t = np.cross(x, rng.normal(size=(M, N, 3)))
    vel[..., 3:] = t / np.linalg.norm(t, axis=-1, keepdims=True) * 7.6e3 + rng.normal(0, 50, (M, N, 3))
    cols = {
        "wrench": np.concatenate([rng.normal(0, 0.05, (M, N, 3)) * i3, rng.normal(0, 1, (M, N, 3)) * m], -1),
        "wheels": rng.normal(0, 0.02, (M, N, 9)) * np.tile(i3, 3),
    }
    return pos, vel, ine, cols, 1.0


def mutate_term(O, spec, index, term, s):
    """Oracle effectors of `spec` with one term of effector `index` scaled by s (and nothing else changed)."""
    spec = [(k, dict(kw)) for k, kw in spec]
    kind, kw = spec[index]
    extra = []
    if term == "g":
        kw["g"] = tuple(s * c for c in kw.get("g", (0.0, 0.0, -9.81)))
    elif term == "thrust":
        kw["thrust"] = kw["thrust"] * s
    elif term == "drag":
        if kw["wind"].shape[-1] == 5:
            kw["wind"] = kw["wind"].copy()
            kw["wind"][..., 3] *= s
        else:
            kw["cd_rho"] = kw.get("cd_rho", 0.6125) * s
    elif term in ("wrench_force", "wrench_torque", "world_force", "world_torque"):
        if kind == "wrench":  # does the term sit in columns 0..2?
            first = (term == "wrench_torque") != kw.get("linear_first", False)
        else:
            first = term == "world_torque"
        kw["wrench"] = kw["wrench"].copy()
        kw["wrench"][..., :3] *= s if first else 1.0
        kw["wrench"][..., 3:] *= 1.0 if first else s
    elif term == "wheels":
        kw["torques"] = kw["torques"] * s
    elif term in ("central", "j2_central", "egm08"):
        kw["mu"] = kw.get("mu", MU_EARTH) * s
        if term == "j2_central":  # the J2 term is proportional to mu J2: keep it
            kw["j2"] = kw.get("j2", J2_EARTH) / s
    elif term == "j2":
        kw["j2"] = kw.get("j2", J2_EARTH) * s
    elif term in ("coriolis", "centrifugal"):
        # frame(mu, a om) + frame(0, b om) has Coriolis (a + b) and centrifugal (a^2 + b^2): pick (a, b) for a
        # Coriolis of s with centrifugal 1 + (s - 1)^2, or a centrifugal of s with Coriolis 1
        om = np.asarray(kw.get("omega", OMEGA_EARTH), dtype=np.float64)
        if term == "coriolis":
            a, b = 1.0, s - 1.0
        else:
            b = (1.0 - np.sqrt(1.0 + 2.0 * (s - 1.0))) / 2.0  # 2 b^2 - 2 b + (1 - s) = 0
            a = 1.0 - b
        kw["omega"] = tuple(a * om)
        extra = [("frame", {"mu": 0.0, "omega": tuple(b * om)})]
    elif term == "graph":
        if kind == "softened":
            kw["k2"] = kw.get("k2", 1e-3) * s
        else:
            kw["G"] = kw.get("G", 6.6743e-11) * s
    else:
        raise KeyError(term)
    spec[index] = (kind, kw)
    spec = spec[:index + 1] + extra + spec[index + 1:]
    return body_effectors(O, spec)[0]


# --------------------------------------------------------------------------- which kernels ran

_CAST = re.compile(r"\((?:bool|int|unsigned int|unsigned)\)")


def _canonical_kernel_name(name):
    """'void b200::k<(bool)1, (int)2, (unsigned int)32>(...)' and 'b200::k<true, 2, 32u>(...)' -> 'k<true, 2, 32>'."""
    n = name.replace("(bool)1", "true").replace("(bool)0", "false")
    n = _CAST.sub("", n)
    n = re.sub(r"\b(\d+)u\b", r"\1", n)
    n = n.removeprefix("void ").replace("b200::", "")
    depth = 0
    for k, ch in enumerate(n):  # drop the parameter list after the template arguments
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            return n[:k]
    return n


def launched_kernels(fn, settle=0.05):
    """Run fn() under torch.profiler (CUDA activity) and return (fn's result, canonical names of the kernels it
    launched, in launch order).  CUPTI records the launches of every runtime in the process, libb200_sixdof's
    statically linked one included.  The profiler can lose the records of a short window: callers compare the
    count with the library's kernel_launches."""
    import time

    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
        time.sleep(settle)  # a margin after the last launch: without it, short windows lost their records more often
    evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == DeviceType.CUDA]
    evs.sort(key=lambda e: e.start_ns())
    return out, [_canonical_kernel_name(e.name()) for e in evs]


def run_child(target, out, args, setting=None, timeout=900):
    """Run `target` ("module:function") as function(out, args) in a fresh child process, with every inherited B200_*
    route switch removed and `setting` ("B200_X=v") set, and load the .npz it wrote to `out`.  The switches are read
    once per process, and torch.profiler loses launch records of short windows more often once a process has run
    other CUDA work (seen with torch 2.11 / CUDA 12.8 on an H100), so kernel names are recorded in a fresh child."""
    import json
    import os
    import subprocess
    import sys

    env = {k: v for k, v in os.environ.items() if not k.startswith("B200_")}
    if setting:
        key, val = setting.split("=")
        env[key] = val
    module, func = target.split(":")
    code = f"import json, sys; from {module} import {func}; {func}(sys.argv[1], json.loads(sys.argv[2]))"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    argv = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, out, json.dumps(args)]
    p = subprocess.run(argv, cwd=root, env=env, capture_output=True, text=True, timeout=timeout)
    assert p.returncode == 0, f"{setting or 'default'} child failed ({p.returncode}):\n{p.stderr[-4000:]}"
    return np.load(out)


# the kernels that advance a tick; layout (AoS <-> SoA) kernels and copies are not part of a route
_TICK_FAMILIES = ("graph_dense_kernel<", "graph_dense_fast_kernel<", "graph_dense_world_kernel<", "graph_csr_kernel<",
                  "nbody_tick_fused_kernel<", "small_world_kernel<", "body_exact_kernel<", "body_fast_kernel<",
                  "body_fast_spec_kernel<", "egm08_force_kernel<")


def assert_route(names, expected, what=""):
    """Every prefix in `expected` names a kernel that ran, and every tick kernel that ran matches one of them."""
    ticks = [n for n in names if n.startswith(_TICK_FAMILIES)]
    for e in expected:
        assert any(n.startswith(e) for n in ticks), f"{what}: expected a launch of {e}, tick kernels launched: {sorted(set(ticks))}"
    for n in ticks:
        assert any(n.startswith(e) for e in expected), f"{what}: unexpected launch of {n} (expected {expected})"
    return ticks
