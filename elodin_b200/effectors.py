"""Built-in effectors of the B200 six_dof() path.

In the reference an effector is an arbitrary JAX function traced by
`@el.map` / `@el.system` (python/elodin/__init__.py:160,360) and lowered through
XLA / Cranelift.  The B200 path has no tracing compiler: the effectors its
kernels know are the shapes SURVEY §8a-12 / §8a-8 list, each a faithful
restatement of the reference example it cites.  Anything else is rejected with
an error (no CPU fallback).

Effectors compose with `|` exactly like reference systems (`gravity | apply_drag`)
and are passed to `six_dof(sys=...)`.
"""

from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from . import _lib


class System:
    """Common base so effectors pipe with `|` (reference: System.pipe / __or__)."""

    def pipe(self, other: "System") -> "Pipe":
        return Pipe(_flatten(self) + _flatten(other))

    def __or__(self, other: "System") -> "Pipe":
        return self.pipe(other)


def _flatten(s) -> list:
    if s is None:
        return []
    if isinstance(s, Pipe):
        return list(s.systems)
    if isinstance(s, System):
        return [s]
    raise TypeError(
        f"{s!r} is not a built-in B200 effector: the B200 backend cannot trace arbitrary Python/JAX systems "
        "(see elodin_b200.effectors for the supported set; there is no CPU fallback)"
    )


@dataclass
class Pipe(System):
    systems: list = field(default_factory=list)


@dataclass
class Effector(System):
    def lower(self, world) -> "_lib.Effector":  # pragma: no cover - abstract
        raise NotImplementedError

    def column_name(self) -> Optional[str]:
        return getattr(self, "column", None)

    def with_mask(self, mask) -> "Effector":
        """Restrict the effector to the entity rows where `mask` is true — the query-join rule of
        the reference (query.rs:672-710): an @el.map effector only runs on entities that own every
        component it reads.  `World.build` sets this automatically from component membership."""
        self._mask = None if mask is None else np.ascontiguousarray(np.asarray(mask, dtype=np.uint8))
        return self

    def _attach_mask(self, e: "_lib.Effector") -> "_lib.Effector":
        m = getattr(self, "_mask", None)
        if m is not None:
            e.entity_mask = m.ctypes.data
        return e


def _base(kind, p=(), flags=0, column: Optional[str] = None, width=0) -> _lib.Effector:
    e = _lib.Effector()
    e.kind, e.flags = kind, flags
    for i, v in enumerate(p):
        e.p[i] = float(v)
    if column:
        e.column_id = _lib.component_id(column)
        e.column_width = width
    return e


@dataclass
class GravityConst(Effector):
    """`f + SpatialForce(linear=g * inertia.mass())` — examples/ball/sim.py:56-58,
    examples/rocket/main.py:292-294."""

    g: Sequence[float] = (0.0, 0.0, -9.81)

    def lower(self, world):
        return self._attach_mask(_base(_lib.EFF_GRAVITY_CONST, self.g))


@dataclass
class DragQuadratic(Effector):
    """apply_drag of examples/ball/sim.py:99-116: drag = 0.5*(Cd*rho*V**2*A) along the
    fluid-relative velocity `wind - v`, evaluated on the stage velocity.  Like the
    reference it returns SpatialForce(linear=...): accumulated torque is reset."""

    cd_rho: float = 0.5 * 1.225
    area: float = 2 * 3.1415 * 0.2 ** 2
    column: Optional[str] = "wind"
    per_body_params: bool = False  # column is [wind(3), Cd*rho, area] (per-world drag in Monte-Carlo batches)

    def lower(self, world):
        return self._attach_mask(_base(_lib.EFF_DRAG_QUADRATIC, (self.cd_rho, self.area), column=self.column,
                                       width=5 if self.per_body_params else 3))


@dataclass
class ThrustBody(Effector):
    """`f + SpatialForce(linear=p.angular() @ axis * thrust)` — examples/rocket/main.py:429-431."""

    axis: Sequence[float] = (-1.0, 0.0, 0.0)
    column: str = "thrust"

    def lower(self, world):
        return self._attach_mask(_base(_lib.EFF_THRUST_BODY, self.axis, column=self.column, width=1))


@dataclass
class WrenchBody(Effector):
    """Body-frame wrench rotated into the world frame.
    layout "torque_first": `f + p.angular() @ f_aero` (examples/rocket/main.py:407-413)
    layout "linear_first": falcon9 apply_body_wrenches (examples/falcon9/sim.py:659-672)."""

    column: str = "aero_force"
    layout: str = "torque_first"

    def lower(self, world):
        if self.layout not in ("torque_first", "linear_first"):
            raise ValueError(f"unknown wrench layout {self.layout!r}")
        flags = _lib.EFF_FLAG_WRENCH_LINEAR_FIRST if self.layout == "linear_first" else 0
        return self._attach_mask(_base(_lib.EFF_WRENCH_BODY, flags=flags, column=self.column, width=6))


@dataclass
class GravityFrame(Effector):
    """Point-mass gravity + Coriolis + centrifugal of a rotating frame —
    gravity_and_frame_forces, examples/falcon9/sim.py:350-361 + frames.py:91-109."""

    mu: float = 3.986004418e14
    omega: Sequence[float] = (0.0, 0.0, 7.292115e-5)

    def lower(self, world):
        return self._attach_mask(_base(_lib.EFF_GRAVITY_FRAME, (self.mu, *self.omega)))


@dataclass
class WrenchWorld(Effector):
    """`force + SpatialForce(..)` with a world-frame wrench column [tau(3), f(3)] computed outside six_dof (a host
    system, recorded telemetry) — the shape of examples/cube-sat/main.py:516-527 (gravity_effector adds a
    precomputed linear force) and examples/drone/sim.py:99-103 (f + SpatialForce(linear=drag))."""

    column: str = "external_force"

    def lower(self, world):
        return self._attach_mask(_base(_lib.EFF_WRENCH_WORLD, column=self.column, width=6))


@dataclass
class TorqueBodyFold(Effector):
    """Reaction-wheel edge fold, examples/cube-sat/main.py:492-505 (rw_effector): Force := fold over the body's
    wheels (out-edges, spawn order) of SpatialForce(torque = q @ tau_k).  The column holds the `n_wheels` body-frame
    wheel torques of each body, [tau_1 .. tau_K] (the torque halves of the wheels' rw_force rows).  Like every
    edge_fold it overwrites what earlier effectors put into Force."""

    column: str = "wheel_torques"
    n_wheels: int = 3

    def lower(self, world):
        if not 1 <= int(self.n_wheels) <= 8:
            raise ValueError("TorqueBodyFold supports 1..8 wheels per body")
        return self._attach_mask(_base(_lib.EFF_TORQUE_BODY_FOLD, column=self.column, width=3 * int(self.n_wheels)))


@dataclass
class GravityJ2(Effector):
    """Point-mass + J2 zonal gravity: `force + SpatialForce(linear=J2().compute_field(x, y, z, m))` —
    libs/nox-py/python/elodin/j2.py:5-29 (constants :7-9)."""

    mu: float = 3.986004418e14
    j2: float = 1.08262668e-3
    r_ref: float = 6.378e6

    def lower(self, world):
        return self._attach_mask(_base(_lib.EFF_GRAVITY_J2, (self.mu, self.j2, self.r_ref)))


@dataclass
class GravityEGM08(Effector):
    """Spherical-harmonic gravity: `force + SpatialForce(linear=EGM08(max_degree).compute_field(x, y, z, m))` —
    libs/nox-py/python/elodin/egm08.py, examples/cube-sat/main.py:47,516-527.  `c_bar` / `s_bar` are the fully normalised
    coefficient tables the reference loads from C_normal.npy / S_normal.npy (its constructor downloads them; pass the
    arrays you have), cut to `[: max_degree + 1, : max_degree + 1]` like egm08.py:51-56.  Evaluated by its own kernel once
    per tick at the three stage positions; parity: bit-identical to the oracle, equal to `GravityJ2` when only C20 is set."""

    c_bar: Optional[np.ndarray] = None
    s_bar: Optional[np.ndarray] = None
    max_degree: Optional[int] = None
    mu: float = 3.986004418e14
    r_ref: float = 6.378e6
    _keep: list = field(default_factory=list, repr=False, compare=False)

    def lower(self, world):
        if self.c_bar is None or self.s_bar is None:
            raise ValueError("GravityEGM08 needs the normalised C and S coefficient tables")
        L = int(self.max_degree) if self.max_degree is not None else int(np.asarray(self.c_bar).shape[0]) - 1
        if not 0 <= L <= 128:
            raise ValueError("GravityEGM08 supports max_degree 0..128")
        c = np.ascontiguousarray(np.asarray(self.c_bar, dtype=np.float64)[: L + 1, : L + 1])
        s = np.ascontiguousarray(np.asarray(self.s_bar, dtype=np.float64)[: L + 1, : L + 1])
        if c.shape != (L + 1, L + 1) or s.shape != (L + 1, L + 1):
            raise ValueError(f"coefficient tables must be at least {(L + 1, L + 1)}")
        self._keep[:] = [c, s]
        e = _base(_lib.EFF_GRAVITY_EGM08, (self.mu, self.r_ref, float(L)))
        e.table0, e.table1, e.table_len = c.ctypes.data, s.ctypes.data, c.size
        return self._attach_mask(e)


@dataclass
class GravityEdges(Effector):
    """GraphQuery.edge_fold gravity (python/elodin/__init__.py:454-557).

    kind "newton":   examples/three-body/main.py:63-70   (G)
    kind "softened": examples/n-body/sim.py:349-361      (k_squared, softening)
    `edges` are (from_entity_row, to_entity_row) pairs in spawn order; when None the
    world's spawned `GravityConstraint`-style edges are used."""

    kind: str = "newton"
    G: float = 6.6743e-11
    k_squared: float = 2.9591220828e-4 / (86400.0 * 86400.0)
    softening: float = 1.0e-10
    edges: Optional[np.ndarray] = None
    _keep: list = field(default_factory=list, repr=False, compare=False)

    def lower(self, world):
        edges = self.edges if self.edges is not None else (world.edge_rows() if world is not None else None)
        if edges is None:
            raise ValueError("GravityEdges needs an edge list")
        ed = np.asarray(edges, dtype=np.uint32).reshape(-1, 2)
        f = np.ascontiguousarray(ed[:, 0])
        t = np.ascontiguousarray(ed[:, 1])
        self._keep[:] = [f, t]
        if self.kind == "newton":
            e = _base(_lib.EFF_GRAVITY_EDGES_NEWTON, (self.G,))
        elif self.kind == "softened":
            e = _base(_lib.EFF_GRAVITY_EDGES_SOFTENED, (self.k_squared, self.softening))
        else:
            raise ValueError(f"unknown gravity kind {self.kind!r}")
        e.n_edges = len(f)
        e.edge_from = f.ctypes.data
        e.edge_to = t.ctypes.data
        return self._attach_mask(e)  # the library refuses a mask here: pass it on rather than drop it silently


def all_pairs_edges(n: int) -> np.ndarray:
    """Edges of examples/n-body/sim.py:334-338: for src, for dst != src."""
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    m = i != j
    return np.stack([i[m], j[m]], 1).astype(np.uint32)


# ---------------------------------------------------------------------------------------------------------------
# CompiledSystem.system_names -> built-in effectors (the host-side half of a `WorldExec::B200` arm, SURVEY §8f-3;
# same table and rules as include/b200_world.hpp:match_effectors)
_STRUCTURAL = {"<system>", "<compiled>", "<empty>", "clear_forces", "calc_accel", "six_dof", "rk4", "semi_implicit_euler",
               "increment_sim_tick", "advance_time"}


def default_effector_registry() -> dict:
    """Effector systems of the reference's own examples by function name (system.rs:213-222,908 carries the repr
    of the Python function, "<function NAME at 0x..>")."""
    return {
        "gravity": lambda: GravityConst((0.0, 0.0, -9.81)),                      # ball/sim.py:56-58, rocket/main.py:292-294
        "apply_drag": lambda: DragQuadratic(),                                    # ball/sim.py:99-116
        "apply_thrust": lambda: ThrustBody((-1.0, 0.0, 0.0), "thrust"),           # rocket/main.py:429-431
        "apply_aero_forces": lambda: WrenchBody("aero_force", "torque_first"),    # rocket/main.py:407-413
        "apply_body_wrenches": lambda: WrenchBody("body_wrench", "linear_first"), # falcon9/sim.py:659-672
        "gravity_and_frame_forces": lambda: GravityFrame(),                       # falcon9/sim.py:350-361
        "rw_effector": lambda: TorqueBodyFold("wheel_torques", 3),                # cube-sat/main.py:492-505
        "j2_gravity": lambda: GravityJ2(),                                        # python/elodin/j2.py:5-29
    }


def system_function_name(system_name: str) -> str:
    if not system_name.startswith("<function "):
        return system_name
    at = system_name.rfind(" at 0x")
    return system_name[len("<function "): at if at >= 0 else len(system_name) - 1]


def match_effectors(system_names: Sequence[str], registry: Optional[dict] = None) -> list:
    """Built-in effectors for a compiled pipeline's `system_names`, in order.  Structural six_dof() entries are
    skipped; any other system that is not in the registry raises B200Error(ERR_UNSUPPORTED) naming it — the B200
    backend has no tracing compiler and no CPU fallback."""
    registry = default_effector_registry() if registry is None else registry
    out = []
    for raw in system_names:
        name = system_function_name(raw)
        if name in _STRUCTURAL:
            continue
        make = registry.get(name)
        if make is None:
            why = f"system '{name}' is not a built-in B200 effector"
            if "<locals>" in name:
                why += (" (an @el.map wrapper: the wrapped function's name is not visible in system_names; register it under "
                        "the name you give it, or pass the effector list explicitly)")
            raise _lib.B200Error(_lib.ERR_UNSUPPORTED, why + "; the B200 backend cannot trace arbitrary systems and has no CPU fallback")
        out.append(make() if callable(make) else make)
    if len(out) > _lib.MAX_EFFECTORS:
        raise _lib.B200Error(_lib.ERR_UNSUPPORTED, f"too many effectors ({len(out)} > {_lib.MAX_EFFECTORS})")
    return out
