"""Host-side mirror of the nox-py ECS surface for the six_dof() path.

Reference (what each piece mirrors):
  * spatial value types          libs/nox-py/src/spatial.rs, libs/nox/src/spatial.rs
  * Component / Archetype / Body python/elodin/__init__.py:594-669, six_dof.rs:153-159
  * World (host columns)         libs/nox-py/src/world.rs:25-60,174-200
  * WorldBuilder.build / run     libs/nox-py/src/world_builder.rs:550-720,1737-1775
  * Exec.run / history           libs/nox-py/src/exec.rs:104-173
  * six_dof(), Integrator        libs/nox-py/src/lib.rs:106-127, six_dof.rs:161-203

Only data handling lives here (numpy host columns, entity/component indexing,
tick bookkeeping).  Every tick is integrated by libb200_sixdof.so on the GPU via
B200Exec; there is no Python/CPU integrator in this package.
"""

from __future__ import annotations

import dataclasses
import enum
import re
import copy
import os
import sys
import time
import typing
from statistics import NormalDist
from typing import Callable, Dict, List, Optional, Sequence, Union

import numpy as np

from . import _lib
from ._lib import component_id
from .effectors import Effector, System, _flatten
from .executor import B200Exec, partial_rank_correlation

# --------------------------------------------------------------------------- value types


def _vec(x, n) -> np.ndarray:
    a = np.zeros(n) if x is None else np.asarray(x, dtype=np.float64).reshape(n)
    return a


class Quaternion:
    """[i, j, k, w] storage, scalar last (libs/nox/src/quaternion.rs:100)."""

    def __init__(self, arr):
        self.arr = _vec(arr, 4)

    @staticmethod
    def identity() -> "Quaternion":
        return Quaternion([0.0, 0.0, 0.0, 1.0])

    @staticmethod
    def from_axis_angle(axis, angle) -> "Quaternion":
        axis = np.asarray(axis, dtype=np.float64)
        axis = axis / np.sqrt(axis @ axis)
        half = angle / 2.0
        return Quaternion(np.concatenate([axis * np.sin(half), [np.cos(half)]]))

    @staticmethod
    def from_euler(angles) -> "Quaternion":
        """roll, pitch, yaw — libs/nox/src/quaternion.rs:105-124."""
        r, p, y = [float(a) for a in angles]
        cr, sr, cp, sp, cy, sy = (np.cos(r / 2), np.sin(r / 2), np.cos(p / 2), np.sin(p / 2), np.cos(y / 2),
                                  np.sin(y / 2))
        return Quaternion([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy,
                           cr * cp * cy + sr * sp * sy])

    def vector(self) -> np.ndarray:
        return self.arr


class SpatialTransform:
    """7 f64: [q(4), x(3)] (libs/nox/src/spatial.rs:14)."""

    WIDTH = 7

    def __init__(self, arr=None, angular: Optional[Quaternion] = None, linear=None):
        if arr is not None:
            if angular is not None or linear is not None:
                raise ValueError("Cannot specify both array and linear/angular")
            self.arr = _vec(arr, 7)
        else:
            q = angular.arr if angular is not None else Quaternion.identity().arr
            self.arr = np.concatenate([q, _vec(linear, 3)])

    def linear(self):
        return self.arr[4:]

    def angular(self) -> Quaternion:
        return Quaternion(self.arr[:4])

    def asarray(self):
        return self.arr


class SpatialMotion:
    """6 f64: [angular(3), linear(3)] (libs/nox/src/spatial.rs:386,432-436)."""

    WIDTH = 6

    def __init__(self, angular=None, linear=None):
        self.arr = np.concatenate([_vec(angular, 3), _vec(linear, 3)])

    def linear(self):
        return self.arr[3:]

    def angular(self):
        return self.arr[:3]

    def asarray(self):
        return self.arr


class SpatialForce:
    """6 f64: [torque(3), force(3)] (libs/nox/src/spatial.rs:141,207-211)."""

    WIDTH = 6

    def __init__(self, arr=None, torque=None, linear=None):
        self.arr = _vec(arr, 6) if arr is not None else np.concatenate([_vec(torque, 3), _vec(linear, 3)])

    def force(self):
        return self.arr[3:]

    def torque(self):
        return self.arr[:3]

    def asarray(self):
        return self.arr


class SpatialInertia:
    """7 f64: [diag(3), momentum(3), mass]; `SpatialInertia(mass)` sets diag = mass
    (libs/nox-py/src/spatial.rs:385-397, libs/nox/src/spatial.rs:315-338)."""

    WIDTH = 7

    def __init__(self, mass, inertia=None):
        mass = float(mass)
        diag = np.ones(3) * mass if inertia is None else _vec(inertia, 3)
        self.arr = np.concatenate([diag, np.zeros(3), [mass]])

    def mass(self):
        return self.arr[6]

    def inertia_diag(self):
        return self.arr[:3]

    def asarray(self):
        return self.arr


# --------------------------------------------------------------------------- components


class PrimitiveType(enum.Enum):
    F64 = "f64"
    U64 = "u64"


class ComponentType:
    def __init__(self, ty: PrimitiveType = PrimitiveType.F64, shape: Sequence[int] = ()):
        self.ty, self.shape = ty, tuple(shape)

    @property
    def width(self) -> int:
        return int(np.prod(self.shape)) if self.shape else 1


ComponentType.F64 = ComponentType(PrimitiveType.F64, ())
ComponentType.U64 = ComponentType(PrimitiveType.U64, ())
ComponentType.SpatialPosF64 = ComponentType(PrimitiveType.F64, (7,))
ComponentType.SpatialMotionF64 = ComponentType(PrimitiveType.F64, (6,))
ComponentType.Edge = ComponentType(PrimitiveType.U64, (2,))


class Component:
    """`Component(name, ty, metadata=...)` — python/elodin/__init__.py Annotated metadata;
    id = FNV-1a (libs/impeller2/src/types.rs:40-45)."""

    def __init__(self, name: str, ty: Optional[ComponentType] = None, metadata: Optional[dict] = None):
        self.name, self.ty, self.metadata = name, ty, metadata or {}

    @property
    def id(self) -> int:
        return component_id(self.name)

    @staticmethod
    def of(annotated) -> "Component":
        for m in getattr(annotated, "__metadata__", ()):
            if isinstance(m, Component):
                return m
        raise TypeError(f"{annotated!r} carries no Component metadata")


Annotated = typing.Annotated

WorldPos = Annotated[SpatialTransform, Component("world_pos", ComponentType.SpatialPosF64,
                                                 {"element_names": "q0,q1,q2,q3,x,y,z", "priority": 5})]
WorldVel = Annotated[SpatialMotion, Component("world_vel", ComponentType.SpatialMotionF64,
                                              {"element_names": "ωx,ωy,ωz,x,y,z", "priority": 5})]
WorldAccel = Annotated[SpatialMotion, Component("world_accel", ComponentType.SpatialMotionF64,
                                                {"element_names": "αx,αy,αz,x,y,z", "priority": 5})]
Force = Annotated[SpatialForce, Component("force", ComponentType.SpatialMotionF64,
                                          {"element_names": "τx,τy,τz,x,y,z", "priority": 5})]
Inertia = Annotated[SpatialInertia, Component("inertia", ComponentType(PrimitiveType.F64, (7,)), {"priority": 5})]
Seed = Annotated[np.ndarray, Component("seed", ComponentType.U64, {"priority": 5})]
SimulationTick = Annotated[np.ndarray, Component("tick", ComponentType.F64, {"priority": 7})]
SimulationTimeStep = Annotated[np.ndarray, Component("simulation_time_step", ComponentType.F64, {"priority": 8})]


class Edge:
    """Directed edge between two entities (GraphQuery edges)."""

    def __init__(self, left: "EntityId", right: "EntityId"):
        self.left, self.right = EntityId(int(left)), EntityId(int(right))


class EntityId(int):
    pass


_snake = re.compile(r"(?<!^)(?=[A-Z])")


class Archetype:
    """Dataclass whose fields are Annotated[..., Component(...)] (reference Archetype)."""

    @classmethod
    def archetype_name(cls) -> str:
        return _snake.sub("_", cls.__name__).lower()

    def component_values(self) -> List[tuple]:
        hints = typing.get_type_hints(type(self), include_extras=True)
        out = []
        for f in dataclasses.fields(self):  # type: ignore[arg-type]
            comp = Component.of(hints[f.name])
            out.append((comp, getattr(self, f.name)))
        return out


def dataclass(cls):
    return dataclasses.dataclass(cls)


@dataclasses.dataclass
class Body(Archetype):
    """python/elodin/__init__.py:664-669."""

    world_pos: WorldPos = dataclasses.field(default_factory=SpatialTransform)
    world_vel: WorldVel = dataclasses.field(default_factory=SpatialMotion)
    inertia: Inertia = dataclasses.field(default_factory=lambda: SpatialInertia(mass=1.0))
    force: Force = dataclasses.field(default_factory=SpatialForce)
    world_accel: WorldAccel = dataclasses.field(default_factory=SpatialMotion)


def _flat(value) -> np.ndarray:
    if isinstance(value, Edge):
        return np.array([int(value.left), int(value.right)], dtype=np.uint64)
    if hasattr(value, "asarray"):
        return np.asarray(value.asarray(), dtype=np.float64).reshape(-1)
    return np.atleast_1d(np.asarray(value)).reshape(-1)


# --------------------------------------------------------------------------- systems


class Integrator(enum.Enum):
    Rk4 = "rk4"
    SemiImplicit = "semi_implicit"


@dataclasses.dataclass
class SixDof(System):
    time_step: Optional[float]
    effectors: list
    integrator: Integrator


def six_dof(time_step: Optional[float] = None, sys: Optional[System] = None,
            integrator: Integrator = Integrator.Rk4) -> SixDof:
    """`el.six_dof(time_step=None, sys=None, integrator=Integrator.Rk4)` (lib.rs:106-127):
    clear_forces | sys | calc_accel under the chosen integrator (six_dof.rs:161-203)."""
    return SixDof(time_step, _flatten(sys), integrator)


@dataclasses.dataclass
class HostSystem(System):
    """A per-tick host callback over the numpy columns (non-effector systems such as
    the rocket's thrust curve, examples/rocket/main.py:416-426).  It runs on the host
    between GPU ticks, like copy_db_to_world feeding external controls
    (impeller2_server.rs:607), and forces one tick per launch."""

    fn: Callable[["StepContext"], None]


def host_system(fn) -> HostSystem:
    return HostSystem(fn)


class StepContext:
    def __init__(self, exec_: "Exec"):
        self._exec = exec_

    @property
    def tick(self) -> int:
        return self._exec.tick

    def column(self, name: str) -> np.ndarray:
        """[n_worlds, n_entities_with_component, width] numpy view of a host column."""
        return self._exec.world.columns[component_id(name)].buffer

    def write_component(self, pair_name: str, value) -> None:
        ent, comp = pair_name.rsplit(".", 1)
        col = self._exec.world.columns[component_id(comp)]
        row = col.row_of(self._exec.world.entity_by_name(ent))
        col.buffer[:, row, :] = np.asarray(value, dtype=col.buffer.dtype).reshape(-1)
        self._exec.dirty.add(col.component.id)


# --------------------------------------------------------------------------- world


class Column:
    """`Column{buffer, entity_ids}` (world.rs:25-29) with a leading world axis."""

    def __init__(self, component: Component, width: int, dtype):
        self.component, self.width, self.dtype = component, width, dtype
        self.entity_ids: List[int] = []
        self.rows: List[np.ndarray] = []
        self.buffer: Optional[np.ndarray] = None

    def row_of(self, entity: int) -> int:
        return self.entity_ids.index(int(entity))


def quantised_time_step(simulation_rate: float) -> float:
    """`Duration::from_secs_f64(1/rate).as_secs_f64()` (world_builder.rs:221,
    world.rs:185-191): the step is rounded to whole nanoseconds; 120 Hz -> 0.008333333."""
    if simulation_rate <= 0:
        raise ValueError(f"simulation_rate must be > 0 Hz, got {simulation_rate}")
    ns = int(np.rint(1.0e9 / simulation_rate))
    secs, nanos = divmod(ns, 1_000_000_000)
    return float(secs) + float(nanos) / 1.0e9


def ticks_per_telemetry(simulation_rate: float, telemetry_rate: Optional[float]) -> int:
    """validate_rates, world_builder.rs:211-243."""
    if telemetry_rate is None:
        return 1
    if telemetry_rate <= 0:
        raise ValueError(f"telemetry_rate must be > 0 Hz, got {telemetry_rate}")
    ratio = simulation_rate / telemetry_rate
    rounded = round(ratio)
    if abs(ratio - rounded) > 1e-9 or rounded < 1:
        raise ValueError(
            f"telemetry_rate ({telemetry_rate} Hz) must evenly divide simulation_rate ({simulation_rate} Hz); got ratio {ratio}")
    return max(int(rounded), 1)


class World:
    """Host ECS world.  Entity 0 is `Globals` (tick, simulation_time_step), spawned on
    construction like World::add_globals (world.rs:174-183)."""

    def __init__(self):
        self.columns: Dict[int, Column] = {}
        self.entity_names: Dict[int, str] = {0: "Globals"}
        self.entity_len = 1
        self.edges: List[tuple] = []  # (component_name, from_entity, to_entity) in spawn order

    # -- spawning ---------------------------------------------------------------
    def spawn(self, archetypes, name: Optional[str] = None, id: Optional[str] = None) -> EntityId:
        ent = EntityId(self.entity_len)
        self.entity_len += 1
        if not isinstance(archetypes, (list, tuple)):
            archetypes = [archetypes]
        for arch in archetypes:
            for comp, value in arch.component_values():
                flat = _flat(value)
                if isinstance(value, Edge):
                    self.edges.append((comp.name, int(value.left), int(value.right)))
                col = self.columns.get(comp.id)
                if col is None:
                    col = Column(comp, len(flat), flat.dtype if flat.dtype == np.uint64 else np.float64)
                    self.columns[comp.id] = col
                if len(flat) != col.width:
                    raise _lib.B200ValueError(_lib.ERR_VALUE_SIZE_MISMATCH, "value size mismatch")
                col.entity_ids.append(int(ent))
                col.rows.append(flat.astype(col.dtype))
        if name is not None:
            self.entity_names[int(ent)] = name
        elif id is not None:
            self.entity_names[int(ent)] = id
        return ent

    def entity_by_name(self, name: str) -> int:
        for e, n in self.entity_names.items():
            if n == name or n.lower() == name:
                return e
        raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND, f"entity not found: {name}")

    # -- queries ---------------------------------------------------------------
    def body_entities(self) -> List[int]:
        col = self.columns.get(component_id("world_pos"))
        return list(col.entity_ids) if col else []

    def edge_rows(self) -> np.ndarray:
        """Spawned edges as (from_row, to_row) pairs over the Body rows, spawn order kept."""
        rows = {e: i for i, e in enumerate(self.body_entities())}
        out = [(rows[a], rows[b]) for (_, a, b) in self.edges if a in rows and b in rows]
        return np.asarray(out, dtype=np.uint32).reshape(-1, 2)

    def _clone_for_exec(self) -> "World":
        """Private copy for one Exec: same entities / names / edges, its own Column objects and buffers."""
        w = copy.copy(self)
        w.columns = {}
        for cid, col in self.columns.items():
            c = Column(col.component, col.width, col.dtype)
            c.entity_ids = list(col.entity_ids)
            c.rows = [r.copy() for r in col.rows]
            c.buffer = None if col.buffer is None else col.buffer.copy()
            w.columns[cid] = c
        w.entity_names = dict(self.entity_names)
        w.edges = list(self.edges)
        return w

    def finalize(self, n_worlds: int = 1) -> None:
        for col in self.columns.values():
            base = np.stack(col.rows).astype(col.dtype) if col.rows else np.zeros((0, col.width), col.dtype)
            col.buffer = np.broadcast_to(base, (n_worlds,) + base.shape).copy()

    # -- build / run -------------------------------------------------------------
    def build(self, system: System, simulation_rate: float = 120.0, generate_real_time: bool = False,
              telemetry_rate: Optional[float] = None, default_playback_speed: float = 1.0,
              max_ticks: Optional[int] = None, optimize: bool = False, db_path: Optional[str] = None,
              backend: str = "b200", math: str = "exact", n_worlds: int = 1, device: int = -1,
              world_params: Optional[Dict[str, np.ndarray]] = None, resident: Optional[bool] = None,
              ensemble: bool = False, ensemble_ring: Optional[int] = None, extrema: bool = False,
              thresholds: Optional[Sequence["Threshold"]] = None, quantiles: Optional[Sequence[float]] = None,
              covariance: Optional[Sequence] = None, histograms: Optional[Sequence["Histogram"]] = None,
              groups: Optional[Sequence[int]] = None, retain: Optional[Sequence[int]] = None,
              channels: Optional[Sequence["Channel"]] = None, moments: Optional[Sequence] = None,
              dwells: Optional[Sequence["Threshold"]] = None, outcomes: Optional[Sequence["Outcome"]] = None,
              process_group=None) -> "Exec":
        """`ensemble=True` records statistics over the world axis instead of per-world rows (see `Exec.ensemble`):
        the run stays on the device at any batch size.  `ensemble_ring` = telemetry samples the device ring holds
        between two reductions (default: as many as fit in 256 MiB, at least one).  With ensemble=True, `extrema=True`
        also keeps every world's extrema over its telemetry rows (`Exec.extrema`) and `thresholds` (up to 8
        `Threshold`s) every world's first threshold events (`Exec.threshold`), both on the device; `quantiles` (1 to 16
        levels in [0, 1]) also records numpy's linear quantiles over the worlds for every row (`Exec.quantiles`), and
        `covariance` the covariance over the worlds of a selection of components for every row and entity
        (`Exec.covariance`): items are a component name ("world_pos": all its planes) or (component, indices), e.g.
        covariance=[("world_pos", (4, 5, 6)), ("world_vel", (3, 4, 5))], at most 25 distinct planes; `histograms` (1 to
        8 `Histogram`s) the bin counts over the worlds of one or two components for every row (`Exec.histogram`).
        `groups` (1 to 1024 world counts summing to n_worlds) splits the worlds into consecutive groups, e.g. the sweep
        points of a plan ordered by `monte_carlo.plan_groups`, and also records the statistics of every group
        (`Exec.ensemble(pair, groups=True)`) and, where `histograms`, `quantiles` or `covariance` is given, the
        histograms, quantiles and covariance of every group (`Exec.histogram(i, groups=True)`,
        `Exec.quantiles(pair, groups=True)`, `Exec.covariance(entity, groups=True)`), beside the all-worlds tables.
        Group g's tables equal those of an Exec over exactly its worlds.  `retain` (distinct world indices, at least one,
        at most MAX_RETAINED_BODIES worlds x entities) also records the full rows of those worlds, gathered on the
        device, so that `history_worlds`, `history` (world 0, if retained), `attach_db`, `write_db`,
        `export.export_csv` and `monte_carlo.write_run_databases` work for them as in the default mode, with the same
        rows bit for bit; `Exec.retained` is the tuple in the order given.  `channels` (up to 8 `Norm` / `AxisAngle`
        objects with distinct names) adds derived values computed on the device from each body's row -- speeds,
        distances, altitudes, pointing angles -- as the component "<entity>.channels" (channel k at index k, in the
        order given; `Exec.channels` lists the names), which every ensemble table, the extrema and the thresholds
        cover like the sampled components.  `moments` (a selection in the syntax of `covariance`, channels as
        "channels") also keeps every world's run count, mean, spread and RMS of those components over its telemetry
        rows (`Exec.moments`), and `dwells` (up to 8 `Threshold`s) every world's count of rows beyond each bound with
        the first and last such tick (`Exec.dwell`), both folded on the device with the extrema.  `outcomes` (1 to 25
        `Outcome`s with distinct names) takes one value per world from those run summaries, a device column (a dispersed
        input or the final state) or host values, and reduces it over the worlds on the device when asked
        (`Exec.outcome_stats`, `outcome_quantiles`, `outcome_covariance`, `outcome_histogram`, each per group with
        `groups=True`): apogee percentiles per sweep point, an impact ellipse, an event probability, input-to-outcome
        correlations, without a per-world table reaching the host; `Exec.outcome_top_worlds` names the worst runs
        themselves (the k worlds with the largest or smallest value of each outcome), for `retain=` and per-run
        databases.  `process_group` (a torch.distributed group, with
        ensemble=True and quantiles or outcomes) makes this Exec one rank of a world-sharded campaign whose quantile
        tables are collective: every rank builds over its own worlds (`sharding.shard_worlds`, its groups cut by
        `sharding.shard_groups`) and `Exec.quantiles` (grouped or not, row 0 included) and `Exec.outcome_quantiles` are
        reduced over every rank's worlds (`sharding.gather_quantiles`), and `Exec.outcome_top_worlds` merged over them
        with campaign world indices (`sharding.gather_top_worlds`), exact, the same on every rank; every rank must
        then record and ask for them together.  The ring capacity becomes the ranks' least, so that every rank reduces at
        the same ticks.  The other tables stay per rank, merged with the other gather helpers of `sharding`."""
        if backend not in ("b200", "b200-exact", "b200-fast"):
            raise _lib.B200Error(
                _lib.ERR_UNSUPPORTED,
                f"unknown backend '{backend}': this package only provides 'b200' (no cranelift / jax fallback)")
        if backend == "b200-fast":
            math = "fast"
        return Exec(self, system, simulation_rate, telemetry_rate, max_ticks, math, n_worlds, device, world_params, resident,
                    ensemble, ensemble_ring, extrema, thresholds, quantiles, covariance, histograms, groups, retain,
                    channels, moments, dwells, outcomes, process_group)

    def run(self, system: System, simulation_rate: float = 120.0, generate_real_time: bool = False,
            telemetry_rate: Optional[float] = None, default_playback_speed: float = 1.0,
            max_ticks: Optional[int] = None, optimize: bool = False, is_canceled=None, pre_step=None,
            post_step=None, db_path: Optional[str] = None, interactive: bool = True, start_timestamp=None,
            log_level=None, backend: str = "b200", math: str = "exact", n_worlds: int = 1) -> "Exec":
        """Headless `World.run` (python/elodin/__init__.py:673-718): runs to max_ticks.  The
        DB server / editor layers of the reference are out of scope.  Like the reference's
        WorldBuilder::run it looks at sys.argv: `python sim.py bench --ticks N [--detail]`
        builds, runs N ticks and prints the reference's bench lines (world_builder.rs:868-909),
        which examples/n-body/benchmark_backends.py parses."""
        argv = sys.argv[1:]
        if argv[:1] == ["bench"]:
            ticks = int(argv[argv.index("--ticks") + 1]) if "--ticks" in argv else 1000
            t0 = time.perf_counter()
            ex = self.build(system, simulation_rate, generate_real_time, telemetry_rate, default_playback_speed,
                            max_ticks, optimize, db_path, backend, math, n_worlds)
            ex.build_ms = (time.perf_counter() - t0) * 1e3
            ex.run(ticks, show_progress=False)
            prof = ex.profile()
            tpt = int(prof["ticks_per_telemetry"])
            print(f"= tick time:          {prof['tick']:.3f} ms (batch of {tpt} ticks)")
            print(f"build time:           {prof['build']:.3f} ms")
            print(f"real_time_factor:     {prof['real_time_factor']:.3f}")
            if "--detail" in argv:
                print(f"copy_to_client time:  {prof['copy_to_client']:.3f} ms")
                print(f"execute_buffers time: {prof['execute_buffers']:.3f} ms")
                print(f"copy_to_host time:    {prof['copy_to_host']:.3f} ms")
                print(f"h2d_upload time:      {prof['h2d_upload']:.3f} ms")
                print(f"kernel_invoke time:   {prof['kernel_invoke']:.3f} ms ({tpt} invocations)")
                print(f"d2h_download time:    {prof['d2h_download']:.3f} ms")
                print(f"add_to_history time:  {prof['add_to_history']:.3f} ms")
            return ex
        if max_ticks is None:
            raise ValueError("elodin_b200.World.run is headless: pass max_ticks")
        ex = self.build(system, simulation_rate, generate_real_time, telemetry_rate, default_playback_speed,
                        max_ticks, optimize, db_path, backend, math, n_worlds)
        if db_path:
            # the reference's `World.run(db_path=...)` leaves an elodin-db directory behind (impeller2_server.rs:
            # 229-309, 390-438): init_db now, one commit per telemetry cycle while the run is in flight
            ts = None
            if start_timestamp is not None:
                ts = int(start_timestamp.timestamp() * 1e6) if hasattr(start_timestamp, "timestamp") else int(start_timestamp)
            ex.attach_db(db_path, ts)
        ex.run(max_ticks, show_progress=False, is_canceled=is_canceled, pre_step=pre_step, post_step=post_step)
        if db_path:
            ex.close_db()
        return ex


# the Body columns six_dof() writes, as planes of a B200_TRAJ_FULL sample (and of a state_stats table)
_SAMPLED = {"world_pos": (0, 7), "world_vel": (7, 13), "world_accel": (13, 19), "force": (19, 25)}
_ENSEMBLE_RING_BYTES = 256 << 20  # device memory of the ensemble mode's trajectory ring


# the derived channels of World.build(..., channels=[...]) in ensemble mode: planes 25 + k of an ensemble row, addressed
# as one more component, at most MAX_CHANNELS wide (build checks an index against the channels it has)
_CHANNELS = "channels"
_CHANNEL_SPAN = (_lib.ROW_PLANES, _lib.ROW_PLANES + _lib.MAX_CHANNELS)


def _sampled_span(pair: str, what: str):
    """`<entity>.<component>` -> (entity, (first, end) plane of the component in a 25-plane row, or of the channels)."""
    ent, _, comp = pair.rpartition(".")
    span = _CHANNEL_SPAN if comp == _CHANNELS else _SAMPLED.get(comp)
    if not ent or span is None:
        raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND,
                                  f"component not found: {pair} ({what} cover {', '.join(_SAMPLED)})")
    return ent, span


def _sampled_plane(span, index, where: str) -> int:
    """Plane `index` of the component at `span` (from _SAMPLED) in a 25-plane row; ValueError, prefixed by `where`, for an
    index that is not an integer in [0, width)."""
    width = span[1] - span[0]
    if isinstance(index, (bool, np.bool_)) or not isinstance(index, (int, np.integer)) or not 0 <= index < width:
        raise ValueError(f"{where}: index {index!r} is not an integer in [0, {width})")
    return span[0] + int(index)


def _channel_plane(plane: int, n_channels: int, where: str) -> int:
    """`plane` of an ensemble row (25 planes, then channel k at 25 + k); ValueError, prefixed by `where`, if it is a
    channel beyond the `n_channels` of the Exec."""
    if plane >= _lib.ROW_PLANES + n_channels:
        raise ValueError(f"{where}: channel {plane - _lib.ROW_PLANES}, this Exec has {n_channels}")
    return plane


# the tables of ensemble mode, by kind, and the World.build option, after ensemble=True, that records each.  stats,
# quantiles, covariance and histograms are reduced over the worlds per telemetry row (B200Exec.trajectory_<kind> /
# state_<kind>; with groups=[...] also group_<kind>, per group of worlds); the others are run summaries, folded per
# world (B200Exec.summary_begin) and downloaded by B200Exec.<kind>().
_OPTIONS = {"stats": (), "quantiles": ("quantiles=[...]",), "covariance": ("covariance=[...]",),
            "histograms": ("histograms=[...]",), "extrema": ("extrema=True",), "thresholds": ("thresholds=[...]",),
            "moments": ("moments=[...]",), "dwells": ("dwells=[...]",)}
_SUMMARIES = ("extrema", "thresholds", "moments", "dwells")


def _build_with(what: str, *options: str) -> "_lib.B200Error":
    """The refusal (ERR_INVALID_ARGUMENT) of `what` by an Exec built without World.build(..., ensemble=True, *options)."""
    return _lib.B200Error(_lib.ERR_INVALID_ARGUMENT,
                          f"{what}: build the Exec with World.build(..., {', '.join(('ensemble=True',) + options)})")


def _quantile_levels(levels) -> np.ndarray:
    """World.build(..., quantiles=...): 1 to MAX_QUANTILES real levels in [0, 1], order and duplicates kept."""
    if isinstance(levels, (str, bytes)) or not isinstance(levels, Sequence) and not isinstance(levels, np.ndarray):
        raise TypeError(f"quantiles take a sequence of levels in [0, 1], got {levels!r}")
    out = []
    for q in levels:
        if isinstance(q, (bool, np.bool_)) or not isinstance(q, (int, float, np.integer, np.floating)):
            raise TypeError(f"quantile level {q!r}: a real number in [0, 1]")
        if not 0.0 <= float(q) <= 1.0:  # NaN fails this too
            raise ValueError(f"quantile level {q!r}: not in [0, 1]")
        out.append(float(q))
    if not 1 <= len(out) <= _lib.MAX_QUANTILES:
        raise ValueError(f"{len(out)} quantile levels: 1 to {_lib.MAX_QUANTILES}")
    return np.array(out)


def _covariance_planes(spec, channel_names=(), option: str = "covariance", max_planes: int = _lib.MAX_COV_PLANES):
    """World.build(..., covariance=...) -> (planes of the 25-plane row layout, channel k at 25 + k, labels), selection
    order kept; a channel's label is its name.  `option` names the build option in the refusals (moments= takes the
    same selection, up to `max_planes` planes)."""
    if isinstance(spec, (str, bytes)) or not isinstance(spec, Sequence):
        raise TypeError(f"{option} takes a sequence of components or (component, indices) pairs, got {spec!r}")
    planes, labels = [], []
    for item in spec:
        if isinstance(item, str):
            comp, idx = item, None
        elif isinstance(item, (tuple, list)) and len(item) == 2:
            comp, idx = item
        else:
            comp, idx = None, None
        if not isinstance(comp, str):
            raise TypeError(f"{option} item {item!r}: a component name or a (component, indices) pair")
        span = _CHANNEL_SPAN if comp == _CHANNELS else _SAMPLED.get(comp)
        if span is None:
            raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND,
                                      f"component not found: {comp} (ensemble {option} covers {', '.join(_SAMPLED)})")
        width = len(channel_names) if comp == _CHANNELS else span[1] - span[0]
        for i in range(width) if idx is None else idx:
            where = f"{option} item {item!r}"
            plane = _channel_plane(_sampled_plane(span, i, where), len(channel_names), where)
            if plane in planes:
                raise ValueError(f"{option} selects {comp}[{int(i)}] twice")
            planes.append(plane)
            labels.append(channel_names[int(i)] if comp == _CHANNELS else f"{comp}[{int(i)}]")
    if not 1 <= len(planes) <= max_planes:
        raise ValueError(f"{option} selects {len(planes)} planes: 1 to {max_planes}")
    return planes, labels


def _world_groups(groups, n_worlds: int) -> List[int]:
    """World.build(..., groups=...): 1 to MAX_WORLD_GROUPS non-negative integer world counts summing to n_worlds."""
    if isinstance(groups, (str, bytes)) or not isinstance(groups, (Sequence, np.ndarray)):
        raise TypeError(f"groups take a sequence of world counts, got {groups!r}")
    sizes = list(np.asarray(groups).ravel()) if isinstance(groups, np.ndarray) else list(groups)
    for x in sizes:
        if isinstance(x, (bool, np.bool_)) or not isinstance(x, (int, np.integer)):
            raise TypeError(f"groups: world count {x!r} is not an integer")
        if x < 0:
            raise ValueError(f"groups: world count {x} is negative")
    if not 1 <= len(sizes) <= _lib.MAX_WORLD_GROUPS:
        raise ValueError(f"{len(sizes)} groups: 1 to {_lib.MAX_WORLD_GROUPS}")
    if sum(int(x) for x in sizes) != n_worlds:
        raise ValueError(f"groups: the world counts sum to {sum(int(x) for x in sizes)}, not to n_worlds = {n_worlds}")
    return [int(x) for x in sizes]


def _retained_worlds(retain, n_worlds: int, n_entities: int) -> tuple:
    """World.build(..., retain=...): 1 or more distinct integer world indices in [0, n_worlds), order kept, at most
    MAX_RETAINED_BODIES worlds x entities."""
    if isinstance(retain, (str, bytes)) or not isinstance(retain, (Sequence, np.ndarray)):
        raise TypeError(f"retain takes a sequence of world indices, got {retain!r}")
    worlds = list(np.asarray(retain).ravel()) if isinstance(retain, np.ndarray) else list(retain)
    for w in worlds:
        if isinstance(w, (bool, np.bool_)) or not isinstance(w, (int, np.integer)):
            raise TypeError(f"retain: world index {w!r} is not an integer")
        if not 0 <= w < n_worlds:
            raise ValueError(f"retain: world index {w} is not in [0, {n_worlds})")
    worlds = [int(w) for w in worlds]
    if not worlds:
        raise ValueError("retain: list at least one world")
    seen = set()
    for w in worlds:
        if w in seen:
            raise ValueError(f"retain: world {w} is listed twice")
        seen.add(w)
    if len(worlds) * n_entities > _lib.MAX_RETAINED_BODIES:
        raise ValueError(f"retain: {len(worlds)} worlds x {n_entities} entities = {len(worlds) * n_entities} bodies, "
                         f"at most {_lib.MAX_RETAINED_BODIES}")
    return tuple(worlds)


def _histogram_specs(histograms) -> List["Histogram"]:
    """World.build(..., histograms=...): 1 to MAX_HISTOGRAMS el.Histogram objects."""
    if isinstance(histograms, (str, bytes)) or not isinstance(histograms, Sequence):
        raise TypeError(f"histograms take a sequence of el.Histogram objects, got {histograms!r}")
    for h in histograms:
        if not isinstance(h, Histogram):
            raise TypeError(f"histograms take el.Histogram objects, got {h!r}")
    if not 1 <= len(histograms) <= _lib.MAX_HISTOGRAMS:
        raise ValueError(f"{len(histograms)} histograms: 1 to {_lib.MAX_HISTOGRAMS}")
    return list(histograms)


def _finite3(v, where: str) -> tuple:
    """A finite, non-zero 3-vector, as floats."""
    a = np.asarray(v, dtype=np.float64) if not isinstance(v, str) else np.zeros(0)
    if a.shape != (3,) or not np.all(np.isfinite(a)):
        raise ValueError(f"{where}: {v!r} is not a finite 3-vector")
    if not np.any(a != 0.0):
        raise ValueError(f"{where}: the vector is zero")
    return tuple(float(x) for x in a)


class Channel:
    """A derived channel of World.build(..., ensemble=True, channels=[...]): see `Norm` and `AxisAngle`."""

    name: str

    def _record(self) -> "_lib.Channel":
        raise NotImplementedError


class Norm(Channel):
    """`Norm(name, component, indices, center=None, minus=0.0)`: sqrt(sum_i (x_i - center_i)^2) - minus over 1 to 3
    distinct components `indices` of a sampled component (world_pos, world_vel, world_accel, force), per body and row,
    in correctly rounded f64 operations summed in index order (numpy's bits for the same expression).  Speed:
    Norm("speed", "world_vel", (3, 4, 5)); range from a pad: Norm("range", "world_pos", (4, 5), center=(x0, y0));
    altitude over a sphere: Norm("alt", "world_pos", (4, 5, 6), minus=R)."""

    def __init__(self, name: str, component: str, indices, center=None, minus: float = 0.0):
        where = f"Norm({name!r}, {component!r}, {indices!r})"
        if not isinstance(name, str) or not name:
            raise ValueError(f"{where}: the name must be a non-empty string")
        span = _SAMPLED.get(component)
        if span is None:
            raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND,
                                      f"component not found: {component} (channels cover {', '.join(_SAMPLED)})")
        idx = tuple(indices) if isinstance(indices, (tuple, list)) else (indices,)
        if not 1 <= len(idx) <= 3:
            raise ValueError(f"{where}: 1 to 3 indices")
        self.planes = tuple(_sampled_plane(span, i, where) for i in idx)
        if len(set(self.planes)) != len(self.planes):
            raise ValueError(f"{where}: an index listed twice")
        c = (0.0,) * len(idx) if center is None else tuple(np.asarray(center, dtype=np.float64).ravel())
        if len(c) != len(idx) or not all(np.isfinite(c)):
            raise ValueError(f"{where}: center {center!r} is not {len(idx)} finite numbers")
        if isinstance(minus, (bool, np.bool_)) or not np.isfinite(float(minus)):
            raise ValueError(f"{where}: minus {minus!r} is not a finite number")
        self.name, self.center, self.minus = name, tuple(float(x) for x in c), float(minus)

    def _record(self) -> "_lib.Channel":
        return _lib.channel(_lib.CHANNEL_NORM, len(self.planes), self.planes, self.center, (), self.minus)

    def __repr__(self) -> str:
        return f"Norm({self.name!r}, planes={self.planes}, center={self.center}, minus={self.minus})"


class AxisAngle(Channel):
    """`AxisAngle(name, axis, toward)`: the angle in radians, in [0, pi], between the body-frame `axis` rotated into the
    world frame by the body's world_pos quaternion and the world direction `toward` -- a fixed 3-vector, or
    (component, indices) of three consecutive components of a sampled component, e.g. ("world_vel", (3, 4, 5)) for the
    velocity (inertial angle of attack, flight-path angle).  atan2(|u x v|, u . v) with CUDA's double atan2 (2 ulp);
    neither the quaternion nor the direction needs to be unit.  A zero direction (a body at rest) gives 0.  Pitch from
    vertical of a body whose nose is -x: AxisAngle("pitch", (-1, 0, 0), (0, 0, 1))."""

    def __init__(self, name: str, axis, toward):
        where = f"AxisAngle({name!r}, {axis!r}, {toward!r})"
        if not isinstance(name, str) or not name:
            raise ValueError(f"{where}: the name must be a non-empty string")
        self.axis = _finite3(axis, f"{where}: axis")
        if isinstance(toward, (tuple, list)) and len(toward) == 2 and isinstance(toward[0], str):
            comp, idx = toward
            span = _SAMPLED.get(comp)
            if span is None:
                raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND,
                                          f"component not found: {comp} (channels cover {', '.join(_SAMPLED)})")
            idx = tuple(idx) if isinstance(idx, (tuple, list)) else (idx,)
            planes = tuple(_sampled_plane(span, i, where) for i in idx)
            if len(planes) != 3 or planes != (planes[0], planes[0] + 1, planes[0] + 2):
                raise ValueError(f"{where}: toward takes three consecutive indices of one component")
            self.plane, self.direction = planes[0], None
        else:
            self.plane, self.direction = None, _finite3(toward, f"{where}: toward")
        self.name = name

    def _record(self) -> "_lib.Channel":
        if self.plane is None:
            return _lib.channel(_lib.CHANNEL_AXIS_ANGLE, 0, (), self.axis, self.direction)
        return _lib.channel(_lib.CHANNEL_AXIS_ANGLE, 3, (self.plane,), self.axis)

    def __repr__(self) -> str:
        toward = self.direction if self.plane is None else f"planes {self.plane}..{self.plane + 2}"
        return f"AxisAngle({self.name!r}, axis={self.axis}, toward={toward})"


def _channel_list(channels) -> List[Channel]:
    """World.build(..., channels=...): 1 to MAX_CHANNELS Norm / AxisAngle objects with distinct names."""
    if isinstance(channels, (str, bytes)) or not isinstance(channels, Sequence):
        raise TypeError(f"channels take a sequence of el.Norm / el.AxisAngle objects, got {channels!r}")
    for c in channels:
        if not isinstance(c, Channel):
            raise TypeError(f"channels take el.Norm / el.AxisAngle objects, got {c!r}")
    if not 1 <= len(channels) <= _lib.MAX_CHANNELS:
        raise ValueError(f"{len(channels)} channels: 1 to {_lib.MAX_CHANNELS}")
    names = [c.name for c in channels]
    for n in names:
        if names.count(n) > 1:
            raise ValueError(f"channels: the name {n!r} is used twice")
    return list(channels)


class Threshold:
    """A per-world event for `World.build(..., ensemble=True, thresholds=[...])`: the first telemetry row at which
    component `index` of `pair` ("<entity>.<component>": world_pos, world_vel, world_accel or force) is strictly
    below `below`, or strictly above `above` (exactly one of the two).  It is a first-time condition, not a crossing:
    row 0 (the initial state) is checked too, so a world that starts beyond the bound fires at its initial tick.
    NaN never fires."""

    def __init__(self, pair: str, index: int, below: Optional[float] = None, above: Optional[float] = None):
        if (below is None) == (above is None):
            raise ValueError(f"Threshold({pair!r}, {index!r}): give exactly one of below= and above=")
        value = float(above if below is None else below)
        if np.isnan(value):
            raise ValueError(f"Threshold({pair!r}, {index!r}): the bound is NaN, it would never fire")
        self.entity, span = _sampled_span(pair, "thresholds")
        self.plane = _sampled_plane(span, index, f"Threshold({pair!r}, {index!r})")  # in the 25-plane row layout
        self.pair, self.index, self.above, self.value = pair, int(index), below is None, value

    def __repr__(self) -> str:
        return f"Threshold({self.pair!r}, {self.index}, {'above' if self.above else 'below'}={self.value!r})"


class Histogram:
    """A per-row histogram for `World.build(..., ensemble=True, histograms=[...])`: for every telemetry row, the bin
    counts over the worlds of component `index` of `pair` ("<entity>.<component>": world_pos, world_vel, world_accel or
    force), as np.histogram(x, bins=bins, range=range) counts them, or of the components of a pair of indices, as
    np.histogram2d(x, y, bins=bins, range=range) does -- over the finite values, with numpy's edges and rules, exactly.
    `range` is (lo, hi) for 1D and ((lo_x, hi_x), (lo_y, hi_y)) for 2D; `bins` an int (every axis) or one per axis, at
    most 4096 cells in all.  The edges (`edges`) must be finite and strictly increasing."""

    def __init__(self, pair: str, index, range, bins=10):
        where = f"Histogram({pair!r}, {index!r})"
        self.entity, span = _sampled_span(pair, "histograms")
        two = isinstance(index, (tuple, list))
        if two and len(index) != 2:
            raise ValueError(f"{where}: one index (1D) or a pair of indices (2D)")
        idx = tuple(index) if two else (index,)
        self._axes(where, tuple(_sampled_plane(span, i, where) for i in idx), range, bins)  # 25-plane row layout
        self.pair, self.index = pair, tuple(int(i) for i in idx) if two else int(index)

    def _axes(self, where: str, planes: tuple, range, bins) -> None:
        """The planes (one or two), bins, ranges, edges and record length, checked; refusals prefixed by `where`."""
        two, idx = len(planes) == 2, planes
        self.planes = planes
        if two and self.planes[0] == self.planes[1]:
            raise ValueError(f"{where}: the same component on both axes")
        bins_t = tuple(bins) if isinstance(bins, (tuple, list)) else (bins,) * len(idx)
        if len(bins_t) != len(idx) or any(isinstance(b, (bool, np.bool_)) or not isinstance(b, (int, np.integer)) or b < 1
                                          for b in bins_t):
            raise ValueError(f"{where}: bins {bins!r} is not a positive integer per axis")
        self.bins = tuple(int(b) for b in bins_t)
        cells = int(np.prod(self.bins))
        if cells > _lib.MAX_HISTOGRAM_CELLS:
            raise ValueError(f"{where}: {cells} cells, at most {_lib.MAX_HISTOGRAM_CELLS}")
        ranges = tuple(range) if two and isinstance(range, (tuple, list)) else (range,)
        if len(ranges) != len(idx) or not all(isinstance(r, (tuple, list)) and len(r) == 2 for r in ranges):
            raise ValueError(f"{where}: range {range!r} is not " + ("((lo, hi), (lo, hi))" if two else "(lo, hi)"))
        self.range, self._edges = [], []
        for (lo, hi), n in zip(ranges, self.bins):
            if not all(isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, (bool, np.bool_))
                       for v in (lo, hi)):
                raise ValueError(f"{where}: range ({lo!r}, {hi!r}) is not two real numbers")
            lo, hi = float(lo), float(hi)
            # the edges numpy uses, checked as b200_sixdof_*_histograms checks them
            ok = np.isfinite(lo) and np.isfinite(hi) and lo < hi and np.isfinite(hi - lo) and (hi - lo) / n != 0.0
            e = np.linspace(lo, hi, n + 1) if ok else None
            if not ok or not np.all(e[:-1] < e[1:]):
                raise ValueError(f"{where}: range ({lo!r}, {hi!r}) in {n} bins has no finite, strictly increasing edges")
            self.range.append((lo, hi))
            self._edges.append(e)
        self.range = tuple(self.range)
        self.record_len = (2 if two else 3) + cells  # f64 of its record in a row of the table

    @property
    def edges(self):
        """np.linspace(lo, hi, bins + 1) of the axis (1D), or of each axis (2D: a pair)."""
        e = [a.copy() for a in self._edges]
        return e[0] if len(e) == 1 else tuple(e)

    def _spec(self, row: int) -> tuple:
        """The B200Exec.trajectory_histograms spec of this histogram on the Body row `row`."""
        lo, hi = zip(*self.range)
        return (row, self.planes, self.bins, lo, hi)

    def __repr__(self) -> str:
        r = self.range[0] if len(self.range) == 1 else self.range
        b = self.bins[0] if len(self.bins) == 1 else self.bins
        return f"Histogram({self.pair!r}, {self.index!r}, range={r!r}, bins={b!r})"


def _histogram_record(h: Histogram, t: np.ndarray) -> Dict[str, object]:
    """The records of histogram `h` ([..., record_len] f64) -> Exec.histogram's dict of int64 counts and edges."""
    t = t.astype(np.int64)
    if len(h.bins) == 1:
        return {"counts": np.ascontiguousarray(t[..., 3:]), "nonfinite": t[..., 0].copy(), "below": t[..., 1].copy(),
                "above": t[..., 2].copy(), "edges": h.edges}
    return {"counts": np.ascontiguousarray(t[..., 2:]).reshape(*t.shape[:-1], *h.bins), "nonfinite": t[..., 0].copy(),
            "outside": t[..., 1].copy(), "edges": h.edges}


_EXTREMA_FIELDS = ("min", "max", "min_tick", "max_tick", "first_nonfinite_tick")
_MOMENT_FIELDS = ("count", "mean", "std", "rms")
_DWELL_FIELDS = ("rows", "first_tick", "last_tick")
# the Body columns on the device besides the effector inputs: what a column outcome may read
_BODY_COLUMNS = ("world_pos", "world_vel", "world_accel", "force", "inertia")


class Outcome:
    """One value per world for `World.build(..., ensemble=True, outcomes=[...])`, reduced over the worlds on the device
    by `Exec.outcome_stats`, `outcome_quantiles`, `outcome_covariance` and `outcome_histogram`:

    - `Outcome(name, "rocket.world_pos", 6, "max")`: a field of the extrema of component 6 (min, max, min_tick,
      max_tick, first_nonfinite_tick; needs extrema=True); `Outcome(name, "rocket.channels", 1, "rms")`: a field of the
      run moments of a component (count, mean, std, rms; needs moments= to select it).
    - `Outcome(name, "rocket.inertia", 6)`, with no field: the current device value of component 6 of a Body column --
      a dispersed input (inertia 6 = mass, an effector's input column) or, after a run, the final state.
    - `Outcome.threshold(name, i, "tick")` / `Outcome.threshold(name, i, "world_pos", 4)`: threshold i's record;
      `Outcome.dwell(name, i, "last_tick")`: dwell i's record.
    - `Outcome.values(name, array)`: [n_worlds] values from the host, e.g. a plan parameter no device column holds.
      In a world-sharded campaign each rank passes its own slice (`sharding.shard_worlds`).

    A tick that never happened (-1) is NaN, so the reductions leave those worlds out: the count of a threshold's tick
    is the number of worlds where it fired."""

    def __init__(self, name: str, pair: str, index, field: Optional[str] = None):
        where = f"Outcome({name!r}, {pair!r}, {index!r}{'' if field is None else f', {field!r}'})"
        self._name(name, where)
        self.name = name
        ent, _, comp = pair.rpartition(".") if isinstance(pair, str) else ("", "", "")
        if field is None:  # a device column: the width is known once the world is (World.build)
            if not ent or not comp:
                raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND, f"component not found: {pair!r}")
            if isinstance(index, (bool, np.bool_)) or not isinstance(index, (int, np.integer)) or index < 0:
                raise ValueError(f"{where}: index {index!r} is not a non-negative integer")
            self.kind, self.entity, self.component, self.index, self.field = _lib.OUTCOME_COLUMN, ent, comp, int(index), 0
            return
        self.entity, span = _sampled_span(pair, "outcomes")
        self.plane = _sampled_plane(span, index, where)  # of the ensemble row: 25 planes, then the channels
        if field in _EXTREMA_FIELDS:
            self.kind, self.field = _lib.OUTCOME_EXTREMA, _EXTREMA_FIELDS.index(field)
        elif field in _MOMENT_FIELDS:
            self.kind, self.field = _lib.OUTCOME_MOMENT, _MOMENT_FIELDS.index(field)
        else:
            raise ValueError(f"{where}: field {field!r} is none of {', '.join(_EXTREMA_FIELDS + _MOMENT_FIELDS)}")
        self.pair, self.index = pair, int(index)

    @staticmethod
    def _name(name, where: str) -> None:
        if not isinstance(name, str) or not name:
            raise ValueError(f"{where}: the name must be a non-empty string")

    @classmethod
    def _record_of(cls, kind: int, name: str, i, field: int, where: str) -> "Outcome":
        cls._name(name, where)
        if isinstance(i, (bool, np.bool_)) or not isinstance(i, (int, np.integer)) or i < 0:
            raise ValueError(f"{where}: index {i!r} is not a non-negative integer")
        o = cls.__new__(cls)
        o.name, o.kind, o.index, o.field = name, kind, int(i), field
        return o

    @classmethod
    def threshold(cls, name: str, i: int, component: str, index=None) -> "Outcome":
        """Threshold i's record of each world: "tick" (NaN where it never fired), or component `index` of the entity's
        state at that row (world_pos, world_vel, world_accel or force)."""
        where = f"Outcome.threshold({name!r}, {i!r}, {component!r}{'' if index is None else f', {index!r}'})"
        if component == "tick" and index is None:
            field = 0
        elif component in _SAMPLED and index is not None:
            field = 1 + _sampled_plane(_SAMPLED[component], index, where)
        else:
            raise ValueError(f"{where}: \"tick\", or one of {', '.join(_SAMPLED)} with an index")
        return cls._record_of(_lib.OUTCOME_THRESHOLD, name, i, field, where)

    @classmethod
    def dwell(cls, name: str, i: int, field: str) -> "Outcome":
        """Dwell i's record of each world: "rows", "first_tick" or "last_tick" (ticks NaN where no row counted)."""
        where = f"Outcome.dwell({name!r}, {i!r}, {field!r})"
        if field not in _DWELL_FIELDS:
            raise ValueError(f"{where}: field {field!r} is none of {', '.join(_DWELL_FIELDS)}")
        return cls._record_of(_lib.OUTCOME_DWELL, name, i, _DWELL_FIELDS.index(field), where)

    @classmethod
    def values(cls, name: str, values) -> "Outcome":
        """`values` [n_worlds] f64 from the host, copied to the device once when the Exec is built."""
        where = f"Outcome.values({name!r})"
        cls._name(name, where)
        v = np.asarray(values)
        if v.ndim != 1 or not (np.issubdtype(v.dtype, np.floating) or np.issubdtype(v.dtype, np.integer)):
            raise ValueError(f"{where}: values must be a 1-D array of numbers, got {v.dtype} {v.shape}")
        o = cls._record_of(_lib.OUTCOME_VALUES, name, 0, 0, where)
        o.array = np.ascontiguousarray(v, dtype=np.float64)
        return o

    def __repr__(self) -> str:
        kind = {_lib.OUTCOME_EXTREMA: "extrema", _lib.OUTCOME_MOMENT: "moment", _lib.OUTCOME_COLUMN: "column",
                _lib.OUTCOME_THRESHOLD: "threshold", _lib.OUTCOME_DWELL: "dwell", _lib.OUTCOME_VALUES: "values"}[self.kind]
        return f"Outcome({self.name!r}, {kind}, index={self.index}, field={self.field})"


def _outcome_list(outcomes) -> List[Outcome]:
    """World.build(..., outcomes=...): 1 to MAX_OUTCOMES el.Outcome objects with distinct names."""
    if isinstance(outcomes, (str, bytes)) or not isinstance(outcomes, Sequence):
        raise TypeError(f"outcomes take a sequence of el.Outcome objects, got {outcomes!r}")
    for o in outcomes:
        if not isinstance(o, Outcome):
            raise TypeError(f"outcomes take el.Outcome objects, got {o!r}")
    if not 1 <= len(outcomes) <= _lib.MAX_OUTCOMES:
        raise ValueError(f"{len(outcomes)} outcomes: 1 to {_lib.MAX_OUTCOMES}")
    names = [o.name for o in outcomes]
    for n in names:
        if names.count(n) > 1:
            raise ValueError(f"outcomes: the name {n!r} is used twice")
    return list(outcomes)


class _Row(np.ndarray):
    def to_numpy(self):
        return np.asarray(self)


class _Series(np.ndarray):
    """History rows; `[-1].to_numpy()` works like the reference's polars output."""

    def __getitem__(self, i):
        r = super().__getitem__(i)
        return r.view(_Row) if isinstance(r, np.ndarray) else r


class Exec:
    """`PyExec` (libs/nox-py/src/exec.rs:96-173): owns the world + a B200Exec."""

    _pg = None  # World.build(..., process_group=): the group the quantile tables are reduced over, None = this rank

    def __init__(self, world: World, system: System, simulation_rate: float, telemetry_rate: Optional[float],
                 max_ticks: Optional[int], math: str, n_worlds: int, device: int,
                 world_params: Optional[Dict[str, np.ndarray]], resident: Optional[bool] = None,
                 ensemble: bool = False, ensemble_ring: Optional[int] = None, extrema: bool = False,
                 thresholds: Optional[Sequence[Threshold]] = None, quantiles: Optional[Sequence[float]] = None,
                 covariance: Optional[Sequence] = None, histograms: Optional[Sequence[Histogram]] = None,
                 groups: Optional[Sequence[int]] = None, retain: Optional[Sequence[int]] = None,
                 channels: Optional[Sequence[Channel]] = None, moments: Optional[Sequence] = None,
                 dwells: Optional[Sequence[Threshold]] = None, outcomes: Optional[Sequence[Outcome]] = None,
                 process_group=None):
        systems = _flatten(system)
        six = [s for s in systems if isinstance(s, SixDof)]
        if len(six) != 1:
            raise _lib.B200Error(_lib.ERR_UNSUPPORTED, "the B200 backend runs exactly one six_dof() system per world")
        self.six = six[0]
        pre = systems[: systems.index(self.six)]
        post = systems[systems.index(self.six) + 1:]
        for s in pre + post:
            if not isinstance(s, HostSystem):
                raise _lib.B200Error(_lib.ERR_UNSUPPORTED,
                                     f"{s!r}: only host_system() callbacks may surround six_dof() (no tracing compiler)")
        self.pre_systems, self.post_systems = pre, post
        # The reference's build yields an independent exec: this one owns private copies of the world's columns
        # (a later World.build() re-finalises the World's own buffers) and of the effector objects (the query-join
        # masks below are per build — the caller's effectors are never mutated).
        world = world._clone_for_exec()
        self.world = world
        self._effectors = [copy.copy(e) for e in self.six.effectors]
        for e in self._effectors:
            if isinstance(e, Effector):
                e.with_mask(None)
        self.n_worlds = int(n_worlds)
        self.sim_time_step = quantised_time_step(simulation_rate)
        self.ticks_per_telemetry = ticks_per_telemetry(simulation_rate, telemetry_rate)
        self.max_ticks = max_ticks
        world.finalize(self.n_worlds)
        for name, arr in (world_params or {}).items():
            col = world.columns[component_id(name)]
            col.buffer[...] = np.asarray(arr, dtype=col.dtype).reshape(col.buffer.shape)
        bodies = world.body_entities()
        # join rule (query.rs:672-710): every Body column must list the same entities in the same order
        for cname in ("world_vel", "world_accel", "force", "inertia"):
            col = world.columns.get(component_id(cname))
            if col is None or col.entity_ids != bodies:
                raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND, f"component not found: {cname}")
        # ensemble-mode options: checked here, before any device call, the mode before any option's own values
        given = [name for name, value in (("extrema", extrema or None), ("thresholds", thresholds or None),
                                          ("quantiles", quantiles), ("covariance", covariance), ("histograms", histograms),
                                          ("groups", groups), ("retain", retain), ("channels", channels),
                                          ("moments", moments), ("dwells", dwells), ("outcomes", outcomes),
                                          ("process_group", process_group))
                 if value is not None]
        if given and not ensemble:
            msg = f"{', '.join(given)}: need World.build(..., ensemble=True)"
            raise ValueError(msg) if given == ["groups"] else _lib.B200Error(_lib.ERR_INVALID_ARGUMENT, msg)
        if process_group is not None and quantiles is None and outcomes is None:
            raise _lib.B200Error(_lib.ERR_INVALID_ARGUMENT, "process_group makes the quantile tables collective: build "
                                 "with World.build(..., ensemble=True, quantiles=[...]) or outcomes=[...]")
        self._pg = process_group
        self.groups = _world_groups(groups, self.n_worlds) if groups is not None else None
        self._retain = _retained_worlds(retain, self.n_worlds, len(bodies)) if retain is not None else None
        self._channels = _channel_list(channels) if channels is not None else []
        n_c = len(self._channels)  # channel k is plane 25 + k of an ensemble row
        self._extrema = bool(extrema)
        self._thresholds = list(thresholds or [])
        if len(self._thresholds) > _lib.MAX_THRESHOLDS:
            raise ValueError(f"{len(self._thresholds)} thresholds: at most {_lib.MAX_THRESHOLDS}")

        def condition_rows(conditions, option):  # (entity row, plane, above, bound) per Threshold
            out = []
            for t in conditions:
                if not isinstance(t, Threshold):
                    raise TypeError(f"{option} take el.Threshold objects, got {t!r}")
                out.append((self._body_row(t.entity, t.pair), _channel_plane(t.plane, n_c, repr(t)), t.above, t.value))
            return out

        self._threshold_rows = condition_rows(self._thresholds, "thresholds")
        self._moment_planes, self._moment_labels = ([], []) if moments is None else _covariance_planes(
            moments, self.channels, "moments", _lib.ROW_PLANES + n_c)
        if dwells is not None and (isinstance(dwells, (str, bytes)) or not isinstance(dwells, Sequence)):
            raise TypeError(f"dwells take a sequence of el.Threshold objects, got {dwells!r}")
        self._dwells = list(dwells or [])
        if len(self._dwells) > _lib.MAX_DWELLS:
            raise ValueError(f"{len(self._dwells)} dwells: at most {_lib.MAX_DWELLS}")
        self._dwell_rows = condition_rows(self._dwells, "dwells")
        self._outcomes = _outcome_list(outcomes) if outcomes is not None else []
        self._outcome_records = [self._outcome_record(o, n_c) for o in self._outcomes]
        # the run summaries this Exec folds (kinds of _OPTIONS)
        self._summaries = tuple(kind for kind, on in zip(_SUMMARIES, (self._extrema, self._thresholds,
                                                                      self._moment_planes, self._dwells)) if on)
        # the tables reduced per telemetry row: the arguments of B200Exec.trajectory_<kind> / state_<kind> per kind of
        # _OPTIONS, and per table this Exec records (the kind, or group_<kind> for its per-group table, in the order
        # they are reduced) the blocks of rows recorded so far ([k, ...] each)
        self._ens_args: Dict[str, tuple] = {"stats": ()} if ensemble else {}
        if quantiles is not None:
            self._ens_args["quantiles"] = (_quantile_levels(quantiles),)
        if covariance is not None:
            planes, self._cov_labels = _covariance_planes(covariance, self.channels)
            self._ens_args["covariance"] = (planes,)
        if histograms is not None:
            self._histograms = _histogram_specs(histograms)
            specs = []
            for h in self._histograms:
                specs.append(h._spec(self._body_row(h.entity, h.pair)))
                for p in h.planes:
                    _channel_plane(p, n_c, repr(h))
            self._ens_args["histograms"] = (specs,)
        grouped = [f"group_{kind}" for kind in ("stats", "histograms", "quantiles", "covariance")
                   if kind in self._ens_args and self.groups is not None]
        self._ens_rows: Dict[str, List[np.ndarray]] = {name: [] for name in [*self._ens_args, *grouped]}
        # Query join (query.rs:672-710): an effector only runs on the entities that own its input
        # component.  Full membership -> no mask; partial (order-preserving) membership -> entity mask +
        # a body-row-expanded copy of the column for the device; no members / foreign order -> error.
        self._partial: Dict[int, tuple] = {}
        for e in self._effectors:
            cname = e.column_name()
            if not cname:
                continue
            col = world.columns.get(component_id(cname))
            if col is None or not col.entity_ids:
                raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND, f"component not found: {cname}")
            if col.entity_ids == bodies:
                continue
            rows = [bodies.index(ent) for ent in col.entity_ids if ent in bodies]
            if len(rows) != len(col.entity_ids) or rows != sorted(rows):
                raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND, f"component not found: {cname} (owners are not Body entities)")
            mask = np.zeros(len(bodies), dtype=np.uint8)
            mask[rows] = 1
            e.with_mask(mask)
            self._partial[component_id(cname)] = (np.asarray(rows), np.zeros((self.n_worlds, len(bodies), col.width)))
        # Device-resident telemetry cycles (small interactive worlds): the state stays on the GPU for a whole
        # run() and every telemetry sample — all five Body columns — is recorded into the device trajectory
        # ring, read back in one transfer per `_ring_cap` cycles instead of one PCIe round trip per cycle.
        # Results are identical to the invoke_batch path (same kernels, same tick boundaries).
        n_bodies = len(bodies) * self.n_worlds
        self._ensemble = bool(ensemble)
        if resident is None:
            resident = os.environ.get("B200_RESIDENT", "1") != "0" and 0 < n_bodies <= 65536
        self._ring_cap = 0
        if self._ensemble:
            # Ensemble mode: the state never leaves the device between the initial upload and the end of run();
            # each ring-full of telemetry samples is reduced over the worlds in place, then the ring is reset.
            ld = (n_bodies + 127) // 128 * 128
            cap = ensemble_ring if ensemble_ring is not None else _ENSEMBLE_RING_BYTES // max((_lib.ROW_PLANES + n_c) * ld * 8, 1)
            self._ring_cap = int(max(1, min(4096, cap)))
            if self._pg is not None:  # every rank reduces at the same ticks: the ranks' least capacity
                from .sharding import all_reduce_min

                self._ring_cap = all_reduce_min(self._ring_cap, self._pg)
        elif resident and n_bodies:
            ld = (n_bodies + 127) // 128 * 128
            self._ring_cap = int(max(1, min(4096, (64 << 20) // (25 * ld * 8))))
        # ticks of one invoke_batch stay in registers up to 32 at a time (no effect on results)
        self.backend = B200Exec(len(bodies), self.n_worlds, self.sim_time_step, self.six.time_step, self._effectors,
                                self.six.integrator.value, math, device, max_fused_ticks=32, world=world,
                                trajectory_every=self.ticks_per_telemetry if self._ring_cap else 0,
                                trajectory_capacity=self._ring_cap, trajectory_full=bool(self._ring_cap))
        self.tick = 0
        self.build_ms = 0.0
        self._prof = {"execute_buffers": [], "add_to_history": [], "h2d_upload": [], "kernel_invoke": [], "d2h_download": []}
        self.dirty: set = set()
        self._db = None
        self._history: Dict[int, List[np.ndarray]] = {cid: [] for cid in self.world.columns}
        self._globals_hist: List[tuple] = []
        self._summary_tables: Dict[str, np.ndarray] = {}  # run summaries downloaded since the last fold
        if self._channels:  # before summary_begin, which fixes the row width
            self.backend.set_channels([c._record() for c in self._channels])
        if self._summaries:  # moments and dwells are optional keywords of B200Exec.summary_begin: passed when asked for
            self.backend.summary_begin(self._extrema, self._threshold_rows, **{
                k: v for k, v in (("moments", self._moment_planes), ("dwells", self._dwell_rows)) if v})
        if self._outcome_records:  # after summary_begin: outcomes name the summaries in force
            self.backend.set_outcomes(self._outcome_records)
        if self.groups is not None:
            self.backend.set_world_groups(self.groups)
        if self._ensemble:
            if self._retain is None:
                self._history = {}
            self._upload_inputs()
            self._add_ensemble_rows(ring=False)  # row 0: the initial state
        else:
            self._record()

    # -- data plumbing -------------------------------------------------------------
    def _record(self) -> None:
        for cid, col in self.world.columns.items():
            self._history[cid].append(col.buffer.copy())
        self._globals_hist.append((self.tick, self.sim_time_step))
        if getattr(self, "_db", None) is not None:
            self._db.flush()  # commit_world_head_unified: one row per (entity, component) per telemetry cycle

    def _bind_buffers(self) -> None:
        """Pointer tables for invoke_batch, built once: inputs are the world's own column buffers
        (updated in place, so the addresses are stable), outputs are executor-owned buffers that never
        alias an input (cranelift_exec.rs:101-107,138-154)."""
        be = self.backend
        self._tick_in = np.zeros(1, dtype=np.uint64)
        self._dt_in = np.array([self.sim_time_step])
        self._ins, self._outs = [], []
        for cid in be.input_ids:
            if cid == component_id("tick"):
                self._ins.append(self._tick_in)
            elif cid == component_id("simulation_time_step"):
                self._ins.append(self._dt_in)
            elif cid in self._partial:
                self._ins.append(self._partial[cid][1])  # body-row-expanded copy, refreshed before every invoke
            else:
                buf = self.world.columns[cid].buffer
                assert buf.flags.c_contiguous and buf.nbytes == be.column_bytes(cid)
                self._ins.append(buf)
        for cid in be.output_ids:
            if cid in (component_id("tick"), component_id("simulation_time_step")):
                self._outs.append(np.zeros(1, dtype=np.uint64 if cid == component_id("tick") else np.float64))
            elif cid in self._partial:
                self._outs.append(np.empty_like(self._partial[cid][1]))
            else:
                self._outs.append(np.empty_like(self.world.columns[cid].buffer))
        self._in_ptrs = [a.ctypes.data for a in self._ins]
        self._out_ptrs = [a.ctypes.data for a in self._outs]

    def _invoke(self, n: int) -> None:
        """WorldExec::run -> invoke_batch (cranelift_exec.rs:284-303,129-195)."""
        be = self.backend
        if not hasattr(self, "_in_ptrs"):
            self._bind_buffers()
        self._tick_in[0] = self.tick
        self._dt_in[0] = self.sim_time_step
        for cid, (rows, expanded) in self._partial.items():
            expanded[:, rows, :] = self.world.columns[cid].buffer
        be.invoke_batch_ptrs(self._in_ptrs, self._out_ptrs, n)
        for cid, buf in zip(be.output_ids, self._outs):
            if cid == component_id("tick"):
                self.tick = int(buf[0])  # world.advance_tick() x n
            elif cid != component_id("simulation_time_step") and cid not in self._partial:
                col = self.world.columns[cid]
                if col.buffer.nbytes != buf.nbytes:
                    raise _lib.B200ValueError(_lib.ERR_VALUE_SIZE_MISMATCH, "value size mismatch")
                np.copyto(col.buffer, buf)

    def _upload_inputs(self) -> None:
        """Every input column of the host world -> the device (the state the next ticks start from)."""
        be = self.backend
        tick_id, dt_id = component_id("tick"), component_id("simulation_time_step")
        for cid in be.input_ids:
            if cid == tick_id:
                be.upload(cid, np.array([self.tick], dtype=np.uint64))
            elif cid == dt_id:
                be.upload(cid, np.array([self.sim_time_step]))
            elif cid in self._partial:
                rows, expanded = self._partial[cid]
                expanded[:, rows, :] = self.world.columns[cid].buffer
                be.upload(cid, expanded)
            else:
                be.upload(cid, self.world.columns[cid].buffer)

    def _add_ensemble_rows(self, ring: bool, host_rows: bool = False) -> None:
        """Record one batch of ensemble rows, on the device: the ring's samples (ring=True; ticks_per_telemetry ticks
        apart, the last one at the current tick) or the current state as one row.  Reduces every table this Exec
        records, folds the run summaries, records the retained worlds' rows (from the host columns when `host_rows`)
        and appends the rows' globals."""
        be = self.backend
        for name, blocks in self._ens_rows.items():
            args = self._ens_args[name.removeprefix("group_")]
            if self._pg is not None and name.endswith("quantiles"):  # collective: over every rank's worlds
                from .sharding import gather_quantiles

                rows = gather_quantiles(be, *args, "ring" if ring else "state", name == "group_quantiles", self._pg)
                rows = rows if ring else rows[None]
            else:
                rows = getattr(be, f"trajectory_{name}")(*args) if ring else getattr(be, f"state_{name}")(*args)[None]
            blocks.append(rows)
        if self._summaries:
            (be.summary_add_trajectory if ring else be.summary_add_state)()
            self._summary_tables.clear()
        k, tpt = rows.shape[0], self.ticks_per_telemetry
        if self._retain is not None:
            self._add_retained_rows(ring, host_rows)
        self._globals_hist.extend((self.tick - (k - 1 - i) * tpt, self.sim_time_step) for i in range(k))
        if self._db is not None:
            self._db.flush()  # the k cycles of this batch, each with its own timestamp

    def _add_retained_rows(self, ring: bool, host_rows: bool) -> None:
        """The rows of the retained worlds for the batch _add_ensemble_rows records, as the default mode records them.
        With `host_rows` (the invoke_batch route: one row, the host columns current after the cycle's host systems and
        callbacks) every column comes from the host columns at those worlds, as in Exec._record, so that a host
        system's write to a sampled component is in the row.  Otherwise (the resident route, where no host code runs
        between the ticks) the sampled components are gathered on the device (the ring's samples, or the current
        state) and every other column comes from the host columns, as in Exec._run_resident."""
        be, idx = self.backend, list(self._retain)
        if host_rows:
            for cid, col in self.world.columns.items():
                self._history[cid].append(col.buffer[idx])
            return
        self._extend_history(be.trajectory_worlds(idx) if ring else be.state_worlds(idx)[None], idx)

    def _extend_history(self, rows: np.ndarray, worlds: Optional[List[int]] = None) -> None:
        """Append the k history rows of a [k, worlds, n_entities, 25] block of samples: the sampled components cut from
        its planes (one contiguous block per column, the rows are views), every column six_dof() does not write passed
        through from the host columns (at `worlds`, or every world)."""
        for name, (lo, hi) in _SAMPLED.items():
            self._history[component_id(name)].extend(np.ascontiguousarray(rows[..., lo:hi]))
        sampled = {component_id(name) for name in _SAMPLED}
        for cid, col in self.world.columns.items():
            if cid not in sampled:
                self._history[cid].extend([col.buffer.copy() if worlds is None else col.buffer[worlds]] * rows.shape[0])

    def _run_ensemble(self, ticks: int, is_canceled, pre_step, post_step) -> None:
        """Ensemble mode: one row of world-axis statistics per telemetry cycle, reduced on the device from the
        trajectory ring.  Runs without host callbacks stay on the device for the whole call (upload once, one
        reduction per ring-full); the others go one cycle at a time through invoke_batch, as the default mode does,
        and record their rows the same way.  The final state of every world is in the host columns on return."""
        be = self.backend
        tpt = self.ticks_per_telemetry
        remaining = int(ticks)
        host_cb = bool(self.pre_systems or self.post_systems or pre_step or post_step)
        if not host_cb and is_canceled is None:
            self._upload_inputs()
            whole = remaining // tpt
            while whole > 0:
                c = min(whole, self._ring_cap)
                t0 = time.perf_counter()
                be.trajectory_reset()
                be.step(c * tpt)
                self.tick += c * tpt
                self._add_ensemble_rows(ring=True)                    # c rows
                ms = (time.perf_counter() - t0) * 1e3
                self._prof["execute_buffers"] += [ms / c] * c
                for k_dst in ("add_to_history", "h2d_upload", "kernel_invoke", "d2h_download"):
                    self._prof[k_dst] += [0.0] * c                    # not separable on this path
                whole -= c
            remaining %= tpt
            if remaining:                                             # a last, partial cycle
                t0 = time.perf_counter()
                be.step(remaining)
                self.tick += remaining
                self._add_ensemble_rows(ring=False)
                self._prof["execute_buffers"].append((time.perf_counter() - t0) * 1e3)
                for k_dst in ("add_to_history", "h2d_upload", "kernel_invoke", "d2h_download"):
                    self._prof[k_dst].append(0.0)
            for name in _SAMPLED:                                     # the final state, once
                col = self.world.columns[component_id(name)]
                be.download(col.component.id, out=col.buffer)
            return
        while remaining > 0:
            n = min(tpt, remaining)
            per_call = 1 if host_cb else n
            done = 0
            be.trajectory_reset()
            while done < n:
                ctx = StepContext(self)
                if pre_step:
                    pre_step(self.tick, ctx)
                for s in self.pre_systems:
                    s.fn(ctx)
                t_inv = time.perf_counter()
                self._invoke(per_call)                                # host columns stay current
                self._prof["execute_buffers"].append((time.perf_counter() - t_inv) * 1e3 * (n / per_call))
                tm = be.timings()
                for k_src, k_dst in (("h2d_upload_ms", "h2d_upload"), ("kernel_invoke_ms", "kernel_invoke"), ("d2h_download_ms", "d2h_download")):
                    self._prof[k_dst].append(tm[k_src])
                for s in self.post_systems:
                    s.fn(ctx)
                if post_step:
                    post_step(self.tick, ctx)
                done += per_call
            t_hist = time.perf_counter()
            self._add_ensemble_rows(ring=n == tpt, host_rows=True)
            self._prof["add_to_history"].append((time.perf_counter() - t_hist) * 1e3)
            remaining -= n
            if is_canceled is not None and is_canceled():
                break

    def _no_rows(self, what: str):
        raise _lib.B200Error(_lib.ERR_UNSUPPORTED,
                             f"{what}: this Exec was built with ensemble=True and records statistics over the worlds, "
                             "not per-world rows; read them with Exec.ensemble('<entity>.<component>'), or keep the "
                             "rows of chosen worlds with World.build(..., ensemble=True, retain=[...])")

    @property
    def retained(self) -> Optional[tuple]:
        """The worlds of World.build(..., ensemble=True, retain=[...]) whose rows this Exec records, in that order;
        None without `retain`."""
        return self._retain

    def _history_slot(self, world: int, what: str) -> int:
        """The index of campaign world `world` on the world axis of the recorded history: the world itself in the
        default mode, its position in `retain` in ensemble mode.  `what` names the caller in the refusals: an ensemble
        Exec without `retain`, or a world it does not retain."""
        if not self._ensemble:
            return int(world)
        if self._retain is None:
            self._no_rows(what)
        if world not in self._retain:
            raise _lib.B200Error(_lib.ERR_INVALID_ARGUMENT,
                                 f"{what}: world {world!r} has no rows; this ensemble Exec records the rows of "
                                 f"retain={list(self._retain)}")
        return self._retain.index(world)

    def _run_resident(self, cycles: int) -> None:
        """`cycles` whole telemetry cycles without leaving the device: upload the host columns once, step,
        read the recorded samples back per ring-full, leave the final state in the host columns."""
        be = self.backend
        tpt = self.ticks_per_telemetry
        t0 = time.perf_counter()
        self._upload_inputs()
        upload_ms = (time.perf_counter() - t0) * 1e3
        while cycles > 0:
            c = min(cycles, self._ring_cap)
            t0 = time.perf_counter()
            be.trajectory_reset()
            be.step(c * tpt)
            traj = be.trajectory()                                   # [c, n_worlds, n_bodies, 25]
            run_ms = (time.perf_counter() - t0) * 1e3 + upload_ms
            upload_ms = 0.0
            t_hist = time.perf_counter()
            self._extend_history(traj)
            self._globals_hist.extend((self.tick + (k + 1) * tpt, self.sim_time_step) for k in range(c))
            self.tick += c * tpt
            for name, (lo, hi) in _SAMPLED.items():
                np.copyto(self.world.columns[component_id(name)].buffer, traj[-1, :, :, lo:hi])
            if getattr(self, "_db", None) is not None:
                self._db.flush()  # the c cycles of this ring read-back, each with its own timestamp
            hist_ms = (time.perf_counter() - t_hist) * 1e3
            self._prof["execute_buffers"] += [run_ms / c] * c
            self._prof["add_to_history"] += [hist_ms / c] * c
            for k_dst in ("h2d_upload", "kernel_invoke", "d2h_download"):
                self._prof[k_dst] += [0.0] * c                        # not separable on this path
            cycles -= c

    # -- public API ------------------------------------------------------------------
    def run(self, ticks: int = 1, show_progress: bool = True, is_canceled=None, pre_step=None, post_step=None):
        """exec.rs:111-173: `while remaining > 0 { exec.run(); commit_world_head }` — one
        invoke_batch of ticks_per_telemetry ticks per cycle, a history row per cycle.  Runs without host
        callbacks take the device-resident route for their whole cycles (same rows, one transfer)."""
        if self._ensemble:
            self._run_ensemble(ticks, is_canceled, pre_step, post_step)
            return self
        remaining = int(ticks)
        host_cb = bool(self.pre_systems or self.post_systems or pre_step or post_step)
        if self._ring_cap and not host_cb and is_canceled is None and remaining >= self.ticks_per_telemetry:
            whole = remaining // self.ticks_per_telemetry
            self._run_resident(whole)
            remaining -= whole * self.ticks_per_telemetry
        while remaining > 0:
            n = min(self.ticks_per_telemetry, remaining)
            per_call = 1 if host_cb else n
            done = 0
            while done < n:
                ctx = StepContext(self)
                if pre_step:
                    pre_step(self.tick, ctx)
                for s in self.pre_systems:
                    s.fn(ctx)
                t_inv = time.perf_counter()
                self._invoke(per_call)
                self._prof["execute_buffers"].append((time.perf_counter() - t_inv) * 1e3 * (n / per_call))
                tm = self.backend.timings()
                for k_src, k_dst in (("h2d_upload_ms", "h2d_upload"), ("kernel_invoke_ms", "kernel_invoke"), ("d2h_download_ms", "d2h_download")):
                    self._prof[k_dst].append(tm[k_src])
                for s in self.post_systems:
                    s.fn(ctx)
                if post_step:
                    post_step(self.tick, ctx)
                done += per_call
            t_hist = time.perf_counter()
            self._record()
            self._prof["add_to_history"].append((time.perf_counter() - t_hist) * 1e3)
            remaining -= n
            # like the reference (exec.rs:130-165): run the batch, commit it, then ask
            if is_canceled is not None and is_canceled():
                break
        return self

    def history(self, names: Union[str, Sequence[str]]):
        """`exec.history("e1.world_pos")` -> {name: rows[T, width]} (world 0; use
        `history_worlds` for the batch).  The reference returns a polars frame."""
        slot = self._history_slot(0, "history()")
        if isinstance(names, str):
            names = [names]
        out = {}
        for pair in names:
            ent, comp = pair.rsplit(".", 1)
            cid = component_id(comp)
            if ent.lower() == "globals":
                vals = [g[0] if comp == "tick" else g[1] for g in self._globals_hist]
                out[pair] = np.asarray(vals).view(_Series)
                continue
            col = self.world.columns.get(cid)
            if col is None:
                raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND, f"component not found: {pair}")
            row = col.row_of(self.world.entity_by_name(ent))
            out[pair] = np.stack([h[slot, row] for h in self._history[cid]]).view(_Series)
        return out

    def attach_db(self, path: str, start_timestamp_us: Optional[int] = None, world: int = 0):
        """Stream the telemetry of world `world` into an elodin-db directory while the run is in flight: `init_db` now
        (every pair registered, the rows recorded so far committed), then one commit per telemetry cycle
        (`commit_world_head_unified`, impeller2_server.rs:390-438) — per ring read-back on the device-resident route.
        `close_db()` finishes the directory.  `world` is the campaign's world index, a retained one in ensemble mode."""
        from . import db_sink

        if self._ensemble and self._retain is None:
            self._no_rows("attach_db()")
        if getattr(self, "_db", None) is not None:
            raise _lib.B200Error(_lib.ERR_INVALID_ARGUMENT, "a database is already attached")
        self._db = (db_sink.LiveDbWriter(self, path, world=world) if start_timestamp_us is None
                    else db_sink.LiveDbWriter(self, path, start_timestamp_us, world))
        return self._db

    def close_db(self):
        db, self._db = getattr(self, "_db", None), None
        return db.close() if db is not None else None

    def write_db(self, path: str, start_timestamp_us: Optional[int] = None, world: int = 0):
        """Write the recorded telemetry as an elodin-db directory (`elodin_b200.db_sink`): what the
        reference's `init_db` + `commit_world_head_unified` leave on disk for `elodin-db export` / the editor.
        `world` is the campaign's world index, a retained one in ensemble mode."""
        from . import db_sink

        if self._ensemble and self._retain is None:
            self._no_rows("write_db()")
        if start_timestamp_us is None:
            return db_sink.write_db(self, path, world=world)
        return db_sink.write_db(self, path, start_timestamp_us, world)

    def history_worlds(self, pair: str) -> np.ndarray:
        """`<entity>.<component>` -> [rows, n_worlds, width]: every recorded row of every world; in ensemble mode
        [rows, k, width] for the worlds of `retain`, in that order."""
        if self._ensemble and self._retain is None:
            self._no_rows("history_worlds()")
        ent, comp = pair.rsplit(".", 1)
        col = self.world.columns[component_id(comp)]
        row = col.row_of(self.world.entity_by_name(ent))
        return np.stack([h[:, row] for h in self._history[col.component.id]])

    def ensemble(self, pair: str, groups: bool = False) -> Dict[str, np.ndarray]:
        """`exec.ensemble("rocket.world_pos")` -> {"count", "mean", "std", "min", "max"}, each [rows, width]: one row
        per telemetry cycle (row 0 = the initial state), taken over the worlds whose value is finite; count = the
        number of such worlds (a diverged world is missing from it), std = sqrt(m2 / count) (numpy's ddof=0), NaN
        where no world is finite.  Needs World.build(..., ensemble=True); the sampled components are world_pos,
        world_vel, world_accel and force.  With groups=True (World.build(..., groups=[...])) each is [rows, G, width],
        taken over the worlds of each group."""
        t = self._table("ensemble", "stats", groups)
        row, (lo, hi) = self._sampled_row(pair, "ensemble statistics")
        t = t[..., row, lo:hi, :]  # [rows, (G,) width, 5]
        count = np.ascontiguousarray(t[..., 0])
        with np.errstate(invalid="ignore", divide="ignore"):
            std = np.sqrt(t[..., 2] / count)
        return {"count": count, "mean": np.ascontiguousarray(t[..., 1]), "std": std,
                "min": np.ascontiguousarray(t[..., 3]), "max": np.ascontiguousarray(t[..., 4])}

    def quantiles(self, pair: str, groups: bool = False) -> np.ndarray:
        """`exec.quantiles("rocket.world_pos")` -> [rows, n_q, width] f64: for every telemetry row (row 0 = the initial
        state) numpy's linear quantile over the worlds whose value is finite, at each level of World.build(...,
        quantiles=...) in the order given -- the layout of np.quantile(rows_k, q, axis=0) stacked over rows.  NaN where no
        world is finite.  The values are order statistics of the worlds (and one fixed lerp): exact, not estimates.
        With groups=True (World.build(..., groups=[...])) -> [rows, G, n_q, width], over the worlds of each group.
        Built with a `process_group`, the rows are over every rank's worlds (World.build)."""
        t = self._table("quantiles", "quantiles", groups)
        row, (lo, hi) = self._sampled_row(pair, "ensemble quantiles")
        return np.ascontiguousarray(np.swapaxes(t[..., row, lo:hi, :], -1, -2))  # from [rows, (G,) width, n_q]

    def covariance(self, entity: str, groups: bool = False) -> Dict[str, object]:
        """`exec.covariance("rocket")` -> {"count" [rows], "mean" [rows, p], "cov" [rows, p, p], "planes" [p] labels such
        as "world_pos[4]"}: for every telemetry row (row 0 = the initial state) the covariance over the worlds of the
        selection of World.build(..., covariance=...), in its order.  Only worlds whose p selected values are all
        finite count (listwise deletion, unlike Exec.ensemble, which counts per component); cov = co-moments / count
        (numpy's ddof=0, as Exec.ensemble's std), exactly symmetric, NaN where count = 0.  With groups=True
        (World.build(..., groups=[...])) a group axis follows the row axis: count [rows, G], mean [rows, G, p], cov
        [rows, G, p, p], over the worlds of each group."""
        t = self._table("covariance", "covariance", groups)[..., self._body_row(entity, entity), :]  # [rows, (G,) 1 + p + p*p]
        p = len(self._cov_labels)
        count = np.ascontiguousarray(t[..., 0])
        with np.errstate(invalid="ignore", divide="ignore"):
            cov = t[..., 1 + p:].reshape(*t.shape[:-1], p, p) / count[..., None, None]
        return {"count": count, "mean": np.ascontiguousarray(t[..., 1:1 + p]), "cov": cov, "planes": list(self._cov_labels)}

    def histogram(self, i: int, groups: bool = False) -> Dict[str, object]:
        """`exec.histogram(i)` -> for histogram i of World.build(..., histograms=[...]) and every telemetry row (row 0 =
        the initial state), int64 counts over the worlds: "counts" [rows, bins] (1D) or [rows, bins_x, bins_y] (2D,
        np.histogram2d's layout), "nonfinite" [rows] (worlds whose value, or either value, is NaN / inf), 1D "below" and
        "above" [rows] (finite values out of the range on each side), 2D "outside" [rows] (both finite, at least one out
        of range), and "edges" (np.linspace's; a pair for 2D).  Every world is counted once per row.  With groups=True
        (World.build(..., groups=[...])) a group axis follows the row axis: [rows, G, ...], over the worlds of each
        group."""
        t = self._table("histogram", "histograms", groups)
        if not 0 <= i < len(self._histograms):
            raise IndexError(f"histogram {i}: this Exec has {len(self._histograms)}")
        h = self._histograms[i]
        off = sum(x.record_len for x in self._histograms[:i])
        return _histogram_record(h, t[..., off:off + h.record_len])

    def _table(self, accessor: str, kind: str, groups: bool = False) -> np.ndarray:
        """Table `kind` of _OPTIONS (its per-group table with `groups`): the rows recorded so far, or the run summary,
        downloaded once per fold; refused by `accessor` if this Exec does not record it."""
        name = f"group_{kind}" if groups else kind
        if name in self._ens_rows:
            return np.concatenate(self._ens_rows[name])
        if name not in _SUMMARIES or name not in self._summaries:
            raise _build_with(f"{accessor}({'groups=True' if groups else ''})", *_OPTIONS[kind],
                              *(("groups=[...]",) if groups else ()))
        if name not in self._summary_tables:
            self._summary_tables[name] = getattr(self.backend, name)()
        return self._summary_tables[name]

    @property
    def channels(self) -> List[str]:
        """The names of the channels of World.build(..., channels=[...]), in order: index k of "<entity>.channels"."""
        return [c.name for c in self._channels]

    def _body_row(self, entity: str, pair: str) -> int:
        """The Body row of entity `entity`; ERR_COMPONENT_NOT_FOUND, naming `pair`, if it is not a Body entity."""
        bodies = self.world.body_entities()
        try:
            ent = self.world.entity_by_name(entity)
        except _lib.B200ValueError:
            ent = None
        if ent not in bodies:
            raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND, f"component not found: {pair}")
        return bodies.index(ent)

    def _sampled_row(self, pair: str, what: str):
        """`<entity>.<component>` -> (Body row of the entity, plane span of the component in an ensemble row: 25 planes,
        then the channels)."""
        ent, span = _sampled_span(pair, what)
        if span == _CHANNEL_SPAN:
            if not self._channels:
                raise _build_with(pair, "channels=[...]")
            span = (span[0], span[0] + len(self._channels))
        return self._body_row(ent, pair), span

    def extrema(self, pair: str) -> Dict[str, np.ndarray]:
        """`exec.extrema("rocket.world_pos")` -> {"min", "max", "min_tick", "max_tick", "first_nonfinite_tick"}, each
        [n_worlds, width], over every telemetry row of each world (row 0 = the initial state): min / max over the
        finite values (NaN if none), the tick of the row that holds them (the earliest on ties) and the tick of the first
        NaN / inf row; ticks are int64, -1 where they never applied.  Needs World.build(..., ensemble=True,
        extrema=True)."""
        t = self._table("extrema", "extrema")
        row, span = self._sampled_row(pair, "extrema")
        t = t[:, row, span[0]:span[1], :]  # [n_worlds, width, 5]
        out = {k: np.ascontiguousarray(t[..., f]) for f, k in enumerate(("min", "max"))}
        for f, k in enumerate(("min_tick", "max_tick", "first_nonfinite_tick"), start=2):
            out[k] = t[..., f].astype(np.int64)
        return out

    def threshold(self, i: int) -> Dict[str, np.ndarray]:
        """`exec.threshold(i)` -> {"tick": int64 [n_worlds], "world_pos": [n_worlds, 7], "world_vel", "world_accel",
        "force"}: for threshold i of World.build(..., thresholds=[...]), the tick of each world's first telemetry row
        that meets it (-1 = never) and the entity's state at that row (NaN where it never fired)."""
        t = self._table("threshold", "thresholds")
        if not 0 <= i < len(self._thresholds):
            raise IndexError(f"threshold {i}: this Exec has {len(self._thresholds)}")
        t = t[:, i, :]  # [n_worlds, 26]
        out = {"tick": t[:, 0].astype(np.int64)}
        for name, (lo, hi) in _SAMPLED.items():
            out[name] = np.ascontiguousarray(t[:, 1 + lo:1 + hi])
        return out

    def moments(self, pair: str) -> Dict[str, np.ndarray]:
        """`exec.moments("rocket.channels")` -> {"index": the selected indices of the component, ascending, "count"
        int64 [n_worlds, k], "mean", "std", "rms" [n_worlds, k]}: over each world's telemetry rows (row 0 = the initial
        state) whose value is finite, the number of rows, the mean, the spread (numpy's ddof=0) and the root mean square,
        for the components of World.build(..., moments=...).  NaN where count = 0; std and rms are +inf where the sum
        of squares overflowed."""
        t = self._table("moments", "moments")
        row, (lo, hi) = self._sampled_row(pair, "moments")
        cols = sorted((p, j) for j, p in enumerate(self._moment_planes) if lo <= p < hi)
        if not cols:
            raise _lib.B200Error(_lib.ERR_INVALID_ARGUMENT,
                                 f"moments({pair!r}): no index of it is selected by World.build(..., moments=[...])")
        t = t[:, row, [j for _, j in cols], :]  # [n_worlds, k, 3]
        n, mean, m2 = t[..., 0], t[..., 1], t[..., 2]
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            var = m2 / n
            out = {"index": np.array([p - lo for p, _ in cols], dtype=np.int64), "count": n.astype(np.int64),
                   "mean": np.ascontiguousarray(mean), "std": np.sqrt(var), "rms": np.sqrt(mean * mean + var)}
        return out

    def dwell(self, i: int) -> Dict[str, np.ndarray]:
        """`exec.dwell(i)` -> {"rows", "first_tick", "last_tick"}, each int64 [n_worlds]: for dwell i of World.build(...,
        dwells=[...]), the number of each world's telemetry rows (row 0 = the initial state) beyond its bound, and the
        ticks of the first and last of them (-1 where none).  `last_tick` of an error norm above a tolerance is the
        settling time.  Counts are rows, not seconds: a partial last cycle makes the rows unevenly spaced."""
        t = self._table("dwell", "dwells")
        if not 0 <= i < len(self._dwells):
            raise IndexError(f"dwell {i}: this Exec has {len(self._dwells)}")
        return {k: t[:, i, f].astype(np.int64) for f, k in enumerate(("rows", "first_tick", "last_tick"))}

    def _outcome_record(self, o: Outcome, n_c: int) -> tuple:
        """Outcome `o` -> its B200Exec.set_outcomes tuple (kind, field, index, entity row, column id, values), checked
        against this Exec's options and world before the handle exists."""
        where = repr(o)
        if o.kind in (_lib.OUTCOME_EXTREMA, _lib.OUTCOME_MOMENT):
            row = self._body_row(o.entity, o.pair)
            plane = _channel_plane(o.plane, n_c, where)
            if o.kind == _lib.OUTCOME_EXTREMA:
                if not self._extrema:
                    raise _build_with(where, "extrema=True")
                return (o.kind, o.field, plane, row)
            if plane not in self._moment_planes:
                raise _build_with(where, f"moments=[...] selecting {o.pair}[{o.index}]")
            return (o.kind, o.field, self._moment_planes.index(plane), row)
        if o.kind == _lib.OUTCOME_COLUMN:
            pair = f"{o.entity}.{o.component}"
            inputs = [e.column_name() for e in self._effectors if e.column_name()]
            if o.component not in _BODY_COLUMNS + tuple(inputs):
                raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND,
                                          f"component not found: {pair} (outcomes read the device columns: "
                                          f"{', '.join(_BODY_COLUMNS + tuple(inputs))})")
            row = self._body_row(o.entity, pair)
            width = self.world.columns[component_id(o.component)].width
            if o.index >= width:
                raise ValueError(f"{where}: index {o.index}, {pair} has {width} components")
            return (o.kind, o.index, 0, row, o.component)
        if o.kind == _lib.OUTCOME_VALUES:
            if o.array.shape != (self.n_worlds,):
                raise ValueError(f"{where}: {o.array.shape[0]} values, this Exec has {self.n_worlds} worlds")
            return (o.kind, 0, 0, 0, 0, o.array)
        have, option = ((len(self._thresholds), "thresholds") if o.kind == _lib.OUTCOME_THRESHOLD
                        else (len(self._dwells), "dwells"))
        if o.index >= have:
            raise ValueError(f"{where}: {option[:-1]} {o.index}, this Exec has {have}")
        return (o.kind, o.field, o.index)

    @property
    def outcomes(self) -> List[str]:
        """The names of World.build(..., outcomes=[...]), in order: the outcome axis of every outcome table."""
        return [o.name for o in self._outcomes]

    def _outcome_ready(self, accessor: str, groups: bool) -> None:
        if not self._outcomes or (groups and self.groups is None):
            raise _build_with(f"{accessor}({'groups=True' if groups else ''})", "outcomes=[...]",
                              *(("groups=[...]",) if groups else ()))

    def _outcome_plane(self, name: str) -> int:
        if name not in self.outcomes:
            raise _lib.B200ValueError(_lib.ERR_COMPONENT_NOT_FOUND,
                                      f"outcome not found: {name!r} (this Exec has {', '.join(self.outcomes)})")
        return self.outcomes.index(name)

    def outcome_values(self) -> Dict[str, np.ndarray]:
        """{name: [n_worlds]}: every outcome's value of every world, from the summaries as folded so far (ticks that
        never happened are NaN).  It downloads per-world values: meant for small campaigns and tests."""
        self._outcome_ready("outcome_values", False)
        t = self.backend.outcome_values()
        return {n: np.ascontiguousarray(t[:, k]) for k, n in enumerate(self.outcomes)}

    def outcome_stats(self, groups: bool = False) -> Dict[str, np.ndarray]:
        """{"count", "mean", "std", "min", "max"}, each [P] (or [G, P] with groups=True) in the order of `outcomes`:
        over the worlds whose value is finite, as Exec.ensemble.  Computed on the device now, from the summaries as
        folded so far.  The tables of world-sharded ranks merge with executor.merge_stats."""
        self._outcome_ready("outcome_stats", groups)
        t = self.backend.outcome_group_stats() if groups else self.backend.outcome_stats()
        count = np.ascontiguousarray(t[..., 0])
        with np.errstate(invalid="ignore", divide="ignore"):
            std = np.sqrt(t[..., 2] / count)
        return {"count": count, "mean": np.ascontiguousarray(t[..., 1]), "std": std,
                "min": np.ascontiguousarray(t[..., 3]), "max": np.ascontiguousarray(t[..., 4])}

    def outcome_quantiles(self, q, groups: bool = False) -> np.ndarray:
        """[n_q, P] (or [G, n_q, P] with groups=True): numpy's linear quantiles at the levels `q` of every outcome
        over the worlds whose value is finite, exact.  Built with a `process_group`, over every rank's worlds (a
        collective: every rank calls it with the same levels)."""
        self._outcome_ready("outcome_quantiles", groups)
        lv = _quantile_levels(list(np.atleast_1d(q)))
        if self._pg is not None:
            from .sharding import gather_quantiles

            t = gather_quantiles(self.backend, lv, "outcomes", groups, self._pg)
        else:
            t = self.backend.outcome_group_quantiles(lv) if groups else self.backend.outcome_quantiles(lv)
        return np.ascontiguousarray(np.swapaxes(t, -1, -2))

    def outcome_covariance(self, names: Optional[Sequence[str]] = None, groups: bool = False) -> Dict[str, object]:
        """{"count", "mean" [p], "cov" [p, p], "planes" (the names)} of the outcomes `names` (default: all), in
        Exec.covariance's layout (a group axis first with groups=True): over the worlds whose p values are all finite.
        The tables of world-sharded ranks merge with executor.merge_covariance."""
        self._outcome_ready("outcome_covariance", groups)
        names = list(self.outcomes if names is None else names)
        planes = [self._outcome_plane(n) for n in names]
        t = self.backend.outcome_group_covariance(planes) if groups else self.backend.outcome_covariance(planes)
        p = len(planes)
        count = np.array(t[..., 0])  # a scalar without groups
        with np.errstate(invalid="ignore", divide="ignore"):
            cov = t[..., 1 + p:].reshape(*t.shape[:-1], p, p) / count[..., None, None]
        return {"count": count, "mean": np.ascontiguousarray(t[..., 1:1 + p]), "cov": cov, "planes": names}

    def outcome_histogram(self, name, range, bins=10, groups: bool = False) -> Dict[str, object]:
        """The histogram of outcome `name` (1D) or of a pair of names (2D) over the worlds, in Exec.histogram's dict
        ("counts", "nonfinite", "below" / "above" or "outside", "edges"), with el.Histogram's range and bins rules (a
        group axis first with groups=True).  The tables of world-sharded ranks add up (executor.merge_histograms)."""
        self._outcome_ready("outcome_histogram", groups)
        two = isinstance(name, (tuple, list))
        where = f"outcome_histogram({name!r})"
        if two and len(name) != 2:
            raise ValueError(f"{where}: one name (1D) or a pair of names (2D)")
        h = Histogram.__new__(Histogram)
        h._axes(where, tuple(self._outcome_plane(n) for n in (name if two else (name,))), range, bins)
        spec = [h._spec(0)]
        t = self.backend.outcome_group_histograms(spec) if groups else self.backend.outcome_histograms(spec)
        return _histogram_record(h, t)

    def outcome_top_worlds(self, k: int, names: Optional[Sequence[str]] = None, largest: bool = True,
                           groups: bool = False) -> Dict[str, object]:
        """The worst runs: for each outcome of `names` (default: all), the k worlds with the largest (`largest`) or
        smallest finite value, found on the device.  {"count" [p] (the finite worlds), "value" [p, k], "world" [p, k]
        (int64 world indices, ready for World.build(..., retain=...) and monte_carlo.write_run_databases), "names"},
        with a group axis first with groups=True.  Ordered by value (IEEE totalOrder: -0 < +0), ties by ascending world
        index; slots past the count hold NaN and -1.  Built with a `process_group`, over every rank's worlds with
        campaign world indices (a collective: every rank calls it with the same arguments)."""
        if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= int(k) <= _lib.MAX_TOP_WORLDS:
            raise ValueError(f"outcome_top_worlds: k = {k!r}, an int in [1, {_lib.MAX_TOP_WORLDS}]")
        if not isinstance(largest, (bool, np.bool_)):
            raise TypeError(f"outcome_top_worlds: largest = {largest!r}, a bool")
        self._outcome_ready("outcome_top_worlds", groups)
        names = list(self.outcomes if names is None else ([names] if isinstance(names, str) else names))
        if not names or len(set(names)) != len(names):
            raise ValueError(f"outcome_top_worlds: names {names!r}, one or more distinct outcome names")
        planes = [self._outcome_plane(n) for n in names]
        k, largest = int(k), bool(largest)
        if self._pg is not None:
            from .sharding import gather_top_worlds

            t = gather_top_worlds(self.backend, planes, k, largest, groups, self._pg)
        else:
            t = (self.backend.outcome_group_top_worlds(planes, k, largest) if groups
                 else self.backend.outcome_top_worlds(planes, k, largest))
        return {"count": np.ascontiguousarray(t[..., 0]), "value": np.ascontiguousarray(t[..., 1:1 + k]),
                "world": t[..., 1 + k:].astype(np.int64), "names": names}

    def _rank_planes(self, accessor: str, names, groups: bool, least: int, sharded: bool = False) -> List[int]:
        """The planes of `names` for a rank method, every refusal made before any backend call.  The Exec methods rank
        one handle's worlds and refuse a world-sharded Exec; the collectives of `sharding` (sharded=True) need one."""
        self._outcome_ready(accessor, groups)
        if self._pg is not None and not sharded:
            raise _lib.B200Error(_lib.ERR_UNSUPPORTED,
                                 f"{accessor}: ranks over the worlds of a world-sharded campaign are not supported; "
                                 "build without process_group to rank one handle's worlds (or call "
                                 f"sharding.{accessor}(exec, ...) on every rank)")
        if self._pg is None and sharded:
            raise _lib.B200Error(_lib.ERR_INVALID_ARGUMENT,
                                 f"sharding.{accessor}: a collective over the ranks of a world-sharded campaign; build "
                                 "the Exec with World.build(..., process_group=...)")
        names = list(names)
        if len(names) < least or len(set(names)) != len(names):
            raise ValueError(f"{accessor}: names {names!r}, {least} or more distinct outcome names")
        return [self._outcome_plane(n) for n in names]

    def _rank_names(self, accessor: str, names, groups: bool, least: int, sharded: bool = False,
                    one: bool = False) -> tuple:
        """(names, planes) of a rank method: `names` (default: every outcome; with `one`, a single name too) resolved
        by _rank_planes."""
        names = list(self.outcomes if names is None else ([names] if one and isinstance(names, str) else names))
        return names, self._rank_planes(accessor, names, groups, least, sharded)

    def _sensitivity_names(self, inputs, outputs, groups: bool, sharded: bool = False) -> tuple:
        """(inputs, outputs, planes of inputs + outputs) of outcome_sensitivity, every refusal made before any backend
        call."""
        inputs = [inputs] if isinstance(inputs, str) else list(inputs)
        outputs = [outputs] if isinstance(outputs, str) else list(outputs)
        if not inputs or not outputs or set(inputs) & set(outputs):
            raise ValueError(f"outcome_sensitivity: inputs {inputs!r} and outputs {outputs!r}, non-empty and disjoint")
        if len(inputs) + len(outputs) > _lib.MAX_OUTCOMES:
            raise ValueError(f"outcome_sensitivity: {len(inputs) + len(outputs)} names, at most {_lib.MAX_OUTCOMES}")
        return inputs, outputs, self._rank_planes("outcome_sensitivity", inputs + outputs, groups, 2, sharded)

    def outcome_ranks(self, names: Optional[Sequence[str]] = None, groups: bool = False) -> Dict[str, np.ndarray]:
        """{name: [n_worlds]}: the midrank of every world in each outcome of `names` (default: all), computed on the
        device among the worlds whose selected values are all finite (scipy.stats.rankdata(method="average"); -0 and
        +0 are one value), within its group with groups=True; NaN for the other worlds.  It downloads per-world values:
        meant for small campaigns and tests.  A world-sharded Exec ranks over every rank's worlds with
        sharding.outcome_ranks."""
        names, planes = self._rank_names("outcome_ranks", names, groups, 1, one=True)
        return _ranks_dict(names, self.backend.outcome_group_ranks(planes) if groups else self.backend.outcome_ranks(planes))

    def outcome_rank_correlation(self, names: Optional[Sequence[str]] = None, groups: bool = False) -> Dict[str, object]:
        """Spearman rank correlation of the outcomes `names` (default: all; two or more), on the device: {"count",
        "rho" [p, p], "names"}, a group axis first with groups=True.  Over the worlds whose p values are all finite,
        ranked with midranks; NaN in the row and column of an outcome constant over them, and everywhere below 2
        worlds (as scipy.stats.spearmanr).  A world-sharded Exec uses sharding.outcome_rank_correlation."""
        names, planes = self._rank_names("outcome_rank_correlation", names, groups, 2)
        t = self.backend.outcome_group_rank_correlation(planes) if groups else self.backend.outcome_rank_correlation(planes)
        return _rank_correlation_dict(names, t)

    def outcome_sensitivity(self, inputs: Sequence[str], outputs: Sequence[str], groups: bool = False) -> Dict[str, object]:
        """How much each dispersed input drives each output: {"count", "rho" [n_out, n_in] (Spearman), "prcc"
        [n_out, n_in] (partial rank correlation: the correlation of the ranks of output y and input i once the ranks
        of the other inputs are regressed out), "inputs", "outputs"}, a group axis first with groups=True.  One device
        rank correlation over inputs + outputs; the PRCC of output y comes from the inverse of the rank correlation
        matrix of the inputs and y (executor.partial_rank_correlation), NaN where that matrix holds a NaN or is
        singular.  Every output shares one set of complete worlds, those whose inputs and outputs are all finite: to
        rank an output over only its own finite worlds, call it separately.  A world-sharded Exec uses
        sharding.outcome_sensitivity."""
        inputs, outputs, planes = self._sensitivity_names(inputs, outputs, groups)
        t = self.backend.outcome_group_rank_correlation(planes) if groups else self.backend.outcome_rank_correlation(planes)
        return _sensitivity_dict(inputs, outputs, t)

    def outcome_sobol(self, inputs: Sequence[str], outputs: Sequence[str], groups: bool = False, bootstrap: int = 100,
                      level: float = 0.95, seed: int = 0) -> Dict[str, object]:
        """Variance-based sensitivity of a Saltelli campaign (monte_carlo.saltelli, world k = plan row k), on the
        device: {"count" [n_out], "var" [n_out], "S1" [n_out, d], "ST" [n_out, d], "S1_conf", "ST_conf" [n_out, d],
        "inputs", "outputs"}, a group axis first with groups=True.  S1[y, i] is the share of output y's variance that
        input i explains alone, ST[y, i] that share with all of i's interactions (Saltelli 2010 and Jansen
        estimators); unlike rho and PRCC (outcome_sensitivity) they see non-monotone effects.  `inputs` is the
        design's `inputs`: its length d fixes the block of d + 2 worlds, the names only label the result.  Each output
        has its own count: the base samples whose d + 2 values of it are all finite.  The confidence half-widths are
        z * sd over `bootstrap` resamples (0: NaN) drawn from `seed`, z = NormalDist().inv_cdf(0.5 + level / 2), as
        SALib reports them.  A constant output, or fewer than 2 samples, gives NaN."""
        accessor = "outcome_sobol"
        inputs = [inputs] if isinstance(inputs, str) else list(inputs)
        outputs = [outputs] if isinstance(outputs, str) else list(outputs)
        if not 1 <= len(inputs) <= _lib.MAX_SOBOL_INPUTS or len(set(inputs)) != len(inputs):
            raise ValueError(f"{accessor}: inputs {inputs!r}, 1 to {_lib.MAX_SOBOL_INPUTS} distinct names (the design's inputs)")
        if not 1 <= len(outputs) <= _lib.MAX_OUTCOMES or len(set(outputs)) != len(outputs):
            raise ValueError(f"{accessor}: outputs {outputs!r}, 1 to {_lib.MAX_OUTCOMES} distinct outcome names")
        if isinstance(bootstrap, bool) or not isinstance(bootstrap, (int, np.integer)) or \
                not 0 <= int(bootstrap) <= _lib.MAX_SOBOL_RESAMPLES:
            raise ValueError(f"{accessor}: bootstrap = {bootstrap!r}, an int in [0, {_lib.MAX_SOBOL_RESAMPLES}]")
        if isinstance(level, bool) or not isinstance(level, (int, float, np.floating)) or not 0.0 < float(level) < 1.0:
            raise ValueError(f"{accessor}: level = {level!r}, a number in (0, 1)")
        if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)):
            raise TypeError(f"{accessor}: seed = {seed!r}, an int")
        self._outcome_ready(accessor, groups)
        if self._pg is not None:
            raise _lib.B200Error(_lib.ERR_UNSUPPORTED,
                                 f"{accessor}: Sobol indices over the worlds of a world-sharded campaign are not "
                                 "supported; build without process_group to analyse one handle's worlds")
        d = len(inputs)
        sizes = self.groups if groups else [self.n_worlds]
        bad = [n for n in sizes if n % (d + 2)]
        if bad:
            raise ValueError(f"{accessor}: {d} inputs make blocks of {d + 2} worlds, but "
                             f"{'a group has' if groups else 'the batch has'} {bad[0]} worlds (monte_carlo.saltelli "
                             "gives N (d + 2) worlds per sweep point)")
        planes = [self._outcome_plane(n) for n in outputs]
        be = self.backend
        t = (be.outcome_group_sobol(planes, d, int(bootstrap), int(seed)) if groups
             else be.outcome_sobol(planes, d, int(bootstrap), int(seed)))
        z = NormalDist().inv_cdf(0.5 + float(level) / 2)
        part = lambda k: np.ascontiguousarray(t[..., 3 + k * d:3 + (k + 1) * d])
        return {"count": np.ascontiguousarray(t[..., 0]), "var": np.ascontiguousarray(t[..., 1]), "S1": part(0),
                "ST": part(1), "S1_conf": z * part(2), "ST_conf": z * part(3), "inputs": inputs, "outputs": outputs}

    def column_array(self, cid) -> np.ndarray:
        cid = component_id(cid) if isinstance(cid, str) else int(cid)
        return self.world.columns[cid].buffer[0]

    def profile(self) -> dict:
        """Profiler::profile (libs/nox-py/src/profile.rs:28-56): mean ms per telemetry cycle and
        real_time_factor = time_step * ticks_per_telemetry / tick (history/DB commit included
        the way the reference includes add_to_history)."""
        mean = lambda k: float(np.mean(self._prof[k])) if self._prof[k] else 0.0
        tick = mean("execute_buffers") + mean("add_to_history")
        batch_ms = self.sim_time_step * 1e3 * max(self.ticks_per_telemetry, 1)
        out = {"build": self.build_ms, "copy_to_client": 0.0, "execute_buffers": mean("execute_buffers"), "copy_to_host": 0.0,
               "h2d_upload": mean("h2d_upload"), "kernel_invoke": mean("kernel_invoke"), "d2h_download": mean("d2h_download"),
               "add_to_history": mean("add_to_history"), "tick": tick, "time_step": self.sim_time_step * 1e3,
               "ticks_per_telemetry": float(self.ticks_per_telemetry),
               "real_time_factor": (batch_ms / tick) if tick > 0 else float("inf")}
        out.update({"backend": self.backend.timings()})
        return out


def _ranks_dict(names: List[str], t: np.ndarray) -> Dict[str, np.ndarray]:
    """Exec.outcome_ranks' dict of rank rows t [n_worlds, p]."""
    return {n: np.ascontiguousarray(t[:, k]) for k, n in enumerate(names)}


def _rank_correlation_dict(names: List[str], t: np.ndarray) -> Dict[str, object]:
    """Exec.outcome_rank_correlation's dict of rank correlation records t [..., 1 + p*p]."""
    p = len(names)
    return {"count": np.array(t[..., 0]), "rho": t[..., 1:].reshape(*t.shape[:-1], p, p), "names": names}


def _sensitivity_dict(inputs: List[str], outputs: List[str], t: np.ndarray) -> Dict[str, object]:
    """Exec.outcome_sensitivity's dict of rank correlation records t [..., 1 + p*p] over inputs + outputs: rho, and the
    PRCC of each output from the inputs' and its rows and columns."""
    p, n_in = len(inputs) + len(outputs), len(inputs)
    R = t[..., 1:].reshape(*t.shape[:-1], p, p)
    rho = np.ascontiguousarray(R[..., n_in:, :n_in])
    prcc = np.empty_like(rho)
    for y in range(len(outputs)):
        sub = list(range(n_in)) + [n_in + y]
        prcc[..., y, :] = partial_rank_correlation(R[..., sub, :][..., :, sub])
    return {"count": np.array(t[..., 0]), "rho": rho, "prcc": prcc, "inputs": inputs, "outputs": outputs}
