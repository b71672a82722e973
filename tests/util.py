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
    if kind == "drag":
        wind = kw["wind"]
        cd, area = kw.get("cd_rho", 0.6125), kw.get("area", 0.25)
        return (O.Effector(O.EFF_DRAG_QUADRATIC, p=(cd, area), column=wind), el.DragQuadratic(cd, area, "wind"),
                {"wind": wind})
    if kind == "thrust":
        thrust = kw["thrust"]
        axis = kw.get("axis", (-1.0, 0.0, 0.0))
        return (O.Effector(O.EFF_THRUST_BODY, p=axis, column=thrust), el.ThrustBody(axis, "thrust"),
                {"thrust": thrust})
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


def nbody_world(seed, M, N, dt, kick=1e-2, size=1.0, speed=1.0, soft=1e-2):
    """A softened all-pairs world where a tick's gravity is visible at FAST tolerance: positions in a cube of
    `size`, linear speeds ~ `speed`, and the gravity constant k scaled so that the median body gets a kick of
    `kick` * |v| per tick.  A tick moves a body by dt * speed, which must be at least 1e-5 of the cube, so that
    gravity evaluated at the wrong stage position differs visibly.  Attitude, angular velocity and inertia come
    from random_world.  Returns (pos, vel, ine, k, soft, S)."""
    assert dt * speed >= 1e-5 * size
    pos, vel, ine = random_world(seed, M, N)
    rng = np.random.default_rng(seed + 1)
    pos[..., 4:] = rng.uniform(-size, size, (M, N, 3))
    vel[..., 3:] = rng.normal(0, speed / np.sqrt(3), (M, N, 3))
    S1 = nbody_pair_scale(pos, ine, 1.0, soft)
    k = kick * np.median(np.linalg.norm(vel[..., 3:], axis=-1)) / (dt * np.median(S1))
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


def launched_kernels(fn):
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
        time.sleep(0.05)  # a margin after the last launch: without it, short windows lost their records more often
    evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == DeviceType.CUDA]
    evs.sort(key=lambda e: e.start_ns())
    return out, [_canonical_kernel_name(e.name()) for e in evs]


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
