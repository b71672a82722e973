"""B200Exec — host-side mirror of the reference executor seam.

Reference: `CraneliftExec` / `WorldExec` (libs/nox-py/src/cranelift_exec.rs:13-195,
libs/nox-py/src/exec.rs:53-94).  Same contract: `invoke_batch(columns, n)` takes
the host column buffers (one per input ComponentId), integrates n ticks, and
returns every output column — but the state lives in GPU HBM between calls and
the ticks run in hand-written sm_90a kernels behind the C ABI
(include/b200_sixdof.h).  All numerics happen in libb200_sixdof.so.
"""

from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import component_id

WORLD_POS = component_id("world_pos")
WORLD_VEL = component_id("world_vel")
WORLD_ACCEL = component_id("world_accel")
FORCE = component_id("force")
INERTIA = component_id("inertia")
TICK = component_id("tick")
SIMULATION_TIME_STEP = component_id("simulation_time_step")

_WIDTHS = {WORLD_POS: 7, WORLD_VEL: 6, WORLD_ACCEL: 6, FORCE: 6, INERTIA: 7}


def _cid(c) -> int:
    return component_id(c) if isinstance(c, str) else int(c)


class B200Exec:
    """One executor = one world batch ([n_worlds, n_entities] bodies) on one GPU."""

    def __init__(
        self,
        n_entities: int,
        n_worlds: int = 1,
        sim_time_step: float = 1.0 / 120.0,
        time_step: Optional[float] = None,
        effectors: Optional[Sequence] = None,
        integrator: str = "rk4",
        math: str = "exact",
        device: int = -1,
        max_fused_ticks: int = 1,
        trajectory_every: int = 0,
        trajectory_capacity: int = 0,
        world=None,
        invoke_chunk_bodies: int = 0,
        trajectory_full: bool = False,
    ):
        from .effectors import _flatten

        L = _lib.lib()
        effs = []
        for e in (effectors if isinstance(effectors, (list, tuple)) else _flatten(effectors)):
            effs += _flatten(e)
        if len(effs) > _lib.MAX_EFFECTORS:
            raise _lib.B200Error(_lib.ERR_UNSUPPORTED, f"too many effectors ({len(effs)} > {_lib.MAX_EFFECTORS})")
        self._effector_objs = effs
        arr = (_lib.Effector * max(len(effs), 1))()
        self._column_widths: Dict[int, int] = dict(_WIDTHS)
        for i, e in enumerate(effs):
            arr[i] = e.lower(world)
            if arr[i].column_id:
                self._column_widths[int(arr[i].column_id)] = int(arr[i].column_width)
        d = _lib.Desc()
        d.abi_version = _lib.ABI_VERSION
        d.integrator = {"rk4": _lib.INTEGRATOR_RK4, "semi_implicit": _lib.INTEGRATOR_SEMI_IMPLICIT}[integrator]
        d.math_mode = {"exact": _lib.MATH_EXACT, "fast": _lib.MATH_FAST}[math]
        d.n_effectors = len(effs)
        d.n_entities, d.n_worlds = int(n_entities), int(n_worlds)
        d.sim_time_step = float(sim_time_step)
        d.time_step = math_nan() if time_step is None else float(time_step)
        d.effectors = arr
        d.device = int(device)
        d.max_fused_ticks = int(max_fused_ticks)
        d.trajectory_every = int(trajectory_every)
        d.trajectory_capacity = int(trajectory_capacity)
        d.invoke_chunk_bodies = int(invoke_chunk_bodies)
        d.trajectory_flags = _lib.TRAJ_FULL if trajectory_full else 0
        h = C.c_void_p()
        _lib.check(L.b200_sixdof_create(C.byref(d), C.byref(h)))
        self._L, self._h = L, h
        self.n_entities, self.n_worlds = int(n_entities), int(n_worlds)
        self.integrator, self.math = integrator, math
        ids = (C.c_uint64 * 32)()
        n = L.b200_sixdof_input_ids(h, ids, 32)
        self.input_ids = [int(ids[i]) for i in range(n)]
        n = L.b200_sixdof_output_ids(h, ids, 32)
        self.output_ids = [int(ids[i]) for i in range(n)]

    # ---- lifetime -------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None):
            self._L.b200_sixdof_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ---- metadata -------------------------------------------------------------
    def column_bytes(self, cid) -> int:
        return int(self._L.b200_sixdof_column_bytes(self._h, _cid(cid)))

    def column_shape(self, cid):
        cid = _cid(cid)
        if cid in (TICK, SIMULATION_TIME_STEP):
            return (1,)
        return (self.n_worlds, self.n_entities, self._column_widths[cid])

    @property
    def tick(self) -> int:
        return int(self._L.b200_sixdof_tick_count(self._h))

    # ---- data movement ----------------------------------------------------------
    def upload(self, cid, array) -> None:
        cid = _cid(cid)
        dtype = np.uint64 if cid == TICK else np.float64
        a = np.ascontiguousarray(array, dtype=dtype)
        _lib.check(self._L.b200_sixdof_upload(self._h, cid, a.ctypes.data, a.nbytes))
        # the copy out of `a` is asynchronous on the handle's stream
        _lib.check(self._L.b200_sixdof_sync(self._h))

    def upload_ptr(self, cid, ptr: int, nbytes: int) -> None:
        """Upload from a raw host or device pointer (e.g. a torch tensor's data_ptr())."""
        _lib.check(self._L.b200_sixdof_upload(self._h, _cid(cid), C.c_void_p(ptr), nbytes))

    def download(self, cid, out: Optional[np.ndarray] = None) -> np.ndarray:
        cid = _cid(cid)
        dtype = np.uint64 if cid == TICK else np.float64
        if out is None:
            out = np.empty(self.column_shape(cid), dtype=dtype)
        _lib.check(self._L.b200_sixdof_download(self._h, cid, out.ctypes.data, out.nbytes))
        return out

    def download_ptr(self, cid, ptr: int, nbytes: int) -> None:
        _lib.check(self._L.b200_sixdof_download(self._h, _cid(cid), C.c_void_p(ptr), nbytes))

    def set_state(self, pos=None, vel=None, inertia=None, accel=None, force=None, **columns) -> None:
        for cid, a in ((WORLD_POS, pos), (WORLD_VEL, vel), (INERTIA, inertia), (WORLD_ACCEL, accel), (FORCE, force)):
            if a is not None:
                self.upload(cid, a)
        for name, a in columns.items():
            self.upload(name, a)

    # ---- stepping ---------------------------------------------------------------
    def step(self, n_ticks: int = 1, sync: bool = False) -> None:
        _lib.check(self._L.b200_sixdof_step(self._h, int(n_ticks)))
        if sync:
            self.sync()

    def sync(self) -> None:
        _lib.check(self._L.b200_sixdof_sync(self._h))

    def invoke_batch(self, in_cols: Sequence[np.ndarray], n_ticks: int = 1,
                     out_cols: Optional[Sequence[np.ndarray]] = None):
        """CraneliftExec::invoke_batch (cranelift_exec.rs:129-195): `in_cols[i]` is the
        host buffer of `input_ids[i]`; returns the buffers of `output_ids`."""
        if len(in_cols) != len(self.input_ids):
            raise _lib.B200ValueError(_lib.ERR_VALUE_SIZE_MISMATCH, "wrong number of input columns")
        ins = []
        for cid, a in zip(self.input_ids, in_cols):
            if a is None:  # not dirty: the device-resident copy stands (world.rs:43,249-252)
                ins.append(None)
                continue
            a = np.ascontiguousarray(a, dtype=np.uint64 if cid == TICK else np.float64)
            if a.nbytes != self.column_bytes(cid):
                raise _lib.B200ValueError(_lib.ERR_VALUE_SIZE_MISMATCH, "value size mismatch")
            ins.append(a)
        if out_cols is None:
            out_cols = [np.empty(self.column_shape(cid), dtype=np.uint64 if cid == TICK else np.float64)
                        for cid in self.output_ids]
        elif len(out_cols) != len(self.output_ids):
            raise _lib.B200ValueError(_lib.ERR_VALUE_SIZE_MISMATCH, "wrong number of output columns")
        in_ptrs = (C.c_void_p * len(ins))(*[None if a is None else a.ctypes.data for a in ins])
        out_ptrs = (C.c_void_p * len(out_cols))(*[None if a is None else a.ctypes.data for a in out_cols])
        _lib.check(self._L.b200_sixdof_invoke_batch(self._h, in_ptrs, out_ptrs, int(n_ticks)))
        return list(out_cols)

    def invoke_batch_ptrs(self, in_ptrs: Sequence[Optional[int]], out_ptrs: Sequence[Optional[int]], n_ticks: int) -> None:
        """Raw-pointer form.  A None / 0 input = "not dirty" (the device-resident copy stands, world.rs:43,249-252);
        a None / 0 output = not read back after this batch."""
        ip = (C.c_void_p * len(in_ptrs))(*in_ptrs)
        op = (C.c_void_p * len(out_ptrs))(*out_ptrs)
        _lib.check(self._L.b200_sixdof_invoke_batch(self._h, ip, op, int(n_ticks)))

    def tick_fn(self, in_cols: Sequence[np.ndarray], out_cols: Sequence[np.ndarray]) -> None:
        """The TickFn-shaped entry (cranelift_exec.rs:11): one tick, void return."""
        _lib.check(self._L.b200_sixdof_bind_tick(self._h))
        ip = (C.c_void_p * len(in_cols))(*[a.ctypes.data for a in in_cols])
        op = (C.c_void_p * len(out_cols))(*[a.ctypes.data for a in out_cols])
        self._L.b200_sixdof_tick(ip, op)
        _lib.check(self._L.b200_sixdof_status(self._h))

    # ---- trajectory ---------------------------------------------------------------
    def trajectory_len(self) -> int:
        return int(self._L.b200_sixdof_trajectory_len(self._h))

    def trajectory_width(self) -> int:
        """13 = (world_pos[7], world_vel[6]); 25 with trajectory_full: + (world_accel[6], force[6])."""
        return int(self._L.b200_sixdof_trajectory_width(self._h))

    def _planes(self, ring: bool) -> tuple:
        """The planes a reduction reads, as table axes: [samples, n_entities, width] for the ring's samples,
        [n_entities, 25] for the current state."""
        if ring:
            return (self.trajectory_len(), self.n_entities, max(self.trajectory_width(), 13))
        return (self.n_entities, 25)

    def _rows(self, ring: bool) -> tuple:
        """The rows an ensemble reduction or run summary reads, as table axes: _planes() with the row widened by the
        channels (set_channels; channel k is plane 25 + k)."""
        p = self._planes(ring)
        return p[:-1] + (p[-1] + self.n_channels,)

    def trajectory(self) -> np.ndarray:
        """[samples, n_worlds, n_entities, width] — see trajectory_width()."""
        self.sync()
        n, _, width = self._planes(ring=True)
        out = np.empty((n, self.n_worlds, self.n_entities, width))
        _lib.check(self._L.b200_sixdof_trajectory_download(self._h, out.ctypes.data, out.nbytes))
        return out

    def trajectory_to_ptr(self, ptr: int, nbytes: int) -> None:
        _lib.check(self._L.b200_sixdof_trajectory_download(self._h, C.c_void_p(ptr), nbytes))

    def trajectory_reset(self) -> None:
        _lib.check(self._L.b200_sixdof_trajectory_reset(self._h))

    # ---- retained worlds (full rows of chosen worlds, gathered on the device) -----------------------------------
    def _download_worlds(self, ring: bool, worlds, shape, out_ptr: Optional[int], nbytes: Optional[int]):
        """b200_sixdof_{trajectory|state}_download_worlds(h, worlds, n, dst, bytes) into `out_ptr` (returning nothing)
        or into a new [shape] f64 array, returned."""
        ws = np.ascontiguousarray(np.asarray(worlds, dtype=np.uint64).ravel())
        fn = getattr(self._L, f"b200_sixdof_{'trajectory' if ring else 'state'}_download_worlds")
        out = None if out_ptr is not None else np.empty(shape)
        ptr = out_ptr if out is None else out.ctypes.data
        _lib.check(fn(self._h, ws.ctypes.data_as(C.POINTER(C.c_uint64)), ws.size, C.c_void_p(ptr),
                      int(np.prod(shape)) * 8 if nbytes is None else nbytes))
        return out

    def trajectory_worlds(self, worlds, out_ptr: Optional[int] = None, nbytes: Optional[int] = None):
        """The ring's samples of the worlds `worlds` (indices below n_worlds, in that order, repeats allowed):
        [samples, k, n_entities, width], equal to trajectory()[:, worlds] bit for bit, gathered on the device.  With
        `out_ptr` (a host or device pointer, e.g. a torch CUDA tensor's data_ptr()) and its `nbytes` the rows are
        written there and nothing is returned."""
        n, E, W = self._planes(ring=True)
        return self._download_worlds(True, worlds, (n, len(np.atleast_1d(worlds)), E, W), out_ptr, nbytes)

    def state_worlds(self, worlds, out_ptr: Optional[int] = None, nbytes: Optional[int] = None):
        """The current state of the worlds `worlds`: [k, n_entities, 25] -- world_pos[7], world_vel[6], world_accel[6],
        force[6] (the B200_TRAJ_FULL sample layout), equal to the downloaded columns at `worlds` bit for bit.
        `out_ptr` / `nbytes` as trajectory_worlds()."""
        return self._download_worlds(False, worlds, (len(np.atleast_1d(worlds)),) + self._planes(ring=False), out_ptr,
                                     nbytes)

    # ---- ensemble statistics (reductions over the world axis, on the device) ------------------------------------
    def _reduce(self, kind: str, ring, args: tuple, shape, out_ptr: Optional[int] = None,
                nbytes: Optional[int] = None) -> Optional[np.ndarray]:
        """b200_sixdof_{trajectory|state}_{kind}(h, *args, dst, bytes) (`ring` True | False; "outcome" for
        b200_sixdof_outcome_{kind}): into `out_ptr` (`nbytes`, by default those of `shape`), returning nothing, or into
        a new [shape] f64 array, returned."""
        source = ring if isinstance(ring, str) else "trajectory" if ring else "state"
        fn = getattr(self._L, f"b200_sixdof_{source}_{kind}")
        out = None if out_ptr is not None else np.empty(shape)
        ptr = out_ptr if out is None else out.ctypes.data
        _lib.check(fn(self._h, *args, C.c_void_p(ptr), int(np.prod(shape)) * 8 if nbytes is None else nbytes))
        return out

    def trajectory_stats(self, out: Optional[np.ndarray] = None) -> np.ndarray:
        """The ring's samples reduced over the worlds: [samples, n_entities, width, 5] with the fields (count, mean,
        m2 = sum (x - mean)^2, min, max) over the finite values (count = 0: NaN in the other four)."""
        shape = self._rows(ring=True) + (_lib.STATS_FIELDS,)
        if out is None:
            return self._reduce("stats", True, (), shape)
        if out.shape != shape or out.dtype != np.float64 or not out.flags.c_contiguous:
            raise _lib.B200ValueError(_lib.ERR_VALUE_SIZE_MISMATCH, f"trajectory statistics are {shape} f64, got {out.shape} {out.dtype}")
        self._reduce("stats", True, (), shape, out.ctypes.data)
        return out

    def trajectory_stats_to_ptr(self, ptr: int, nbytes: int) -> None:
        """trajectory_stats() into a raw host or device pointer (e.g. a torch CUDA tensor's data_ptr())."""
        self._reduce("stats", True, (), None, ptr, nbytes)

    def state_stats(self) -> np.ndarray:
        """The current state reduced over the worlds: [n_entities, 25, 5] — world_pos[7], world_vel[6],
        world_accel[6], force[6] (the B200_TRAJ_FULL sample layout), fields as trajectory_stats()."""
        return self._reduce("stats", False, (), self._rows(ring=False) + (_lib.STATS_FIELDS,))

    # ---- ensemble quantiles (order statistics over the world axis, on the device) -------------------------------
    @staticmethod
    def _levels(q) -> tuple:
        """q -> the (levels, n_q) arguments of the quantile entries."""
        lv = np.ascontiguousarray(np.atleast_1d(np.asarray(q, dtype=np.float64)).ravel())
        return lv.ctypes.data_as(C.POINTER(C.c_double)), lv.size  # the pointer keeps lv alive

    def trajectory_quantiles(self, q, out_ptr: Optional[int] = None) -> Optional[np.ndarray]:
        """The ring's samples: numpy's linear quantile over the finite values of the worlds at each level of `q`,
        [samples, n_entities, width, n_q] (NaN where no world is finite).  With `out_ptr` (a host or device pointer,
        e.g. a torch CUDA tensor's data_ptr()) the table is written there and nothing is returned."""
        lv = self._levels(q)
        return self._reduce("quantiles", True, lv, self._rows(ring=True) + (lv[1],), out_ptr)

    def state_quantiles(self, q) -> np.ndarray:
        """The current state: quantiles over the worlds, [n_entities, 25, n_q] in the B200_TRAJ_FULL plane layout."""
        lv = self._levels(q)
        return self._reduce("quantiles", False, lv, self._rows(ring=False) + (lv[1],))

    def quantile_reads(self) -> float:
        """Reads of the reduced planes the last quantile call made, averaged over its groups."""
        return float(self._L.b200_sixdof_quantile_reads(self._h))

    # ---- world-sharded quantiles: the quantile tables of the union of every rank's worlds, in rounds -------------
    @staticmethod
    def _words(buf) -> tuple:
        """A host (numpy) or device (torch) buffer, or None -> (pointer, bytes)."""
        if buf is None:
            return None, 0
        if isinstance(buf, np.ndarray):
            if not buf.flags.c_contiguous:
                raise ValueError("sharded quantile words: a C-contiguous buffer")
            return buf.ctypes.data, buf.nbytes
        return int(buf.data_ptr()), int(buf.numel()) * int(buf.element_size())

    def sharded_quantiles_shape(self, q, source: str = "ring", groups: bool = False) -> tuple:
        """The shape of the table b200_sixdof_sharded_quantiles_end writes: that of trajectory_ / state_ /
        outcome_[group_]quantiles(q) (`source` "ring", "state" or "outcomes")."""
        n_q = np.atleast_1d(np.asarray(q, dtype=np.float64)).size
        G = (self.world_groups,) if groups else ()
        if source == "ring":
            n, E, W = self._rows(ring=True)
            return (n,) + G + (E, W, n_q)
        if source == "state":
            return G + self._rows(ring=False) + (n_q,)
        if source == "outcomes":
            return G + (self.n_outcomes, n_q)
        raise ValueError(f"quantile source {source!r}: 'ring', 'state' or 'outcomes'")

    def sharded_quantiles_begin(self, q, source: str = "ring", groups: bool = False) -> int:
        """Begin this rank's part of a world-sharded quantile call (b200_sixdof_sharded_quantiles_begin): the source,
        grouping and levels are fixed here.  Returns the largest round in bytes (the partial buffer's least size)."""
        if source not in _lib.QUANTILE_SOURCES:
            raise ValueError(f"quantile source {source!r}: 'ring', 'state' or 'outcomes'")
        lv = self._levels(q)
        mx = C.c_uint64(0)
        _lib.check(self._L.b200_sixdof_sharded_quantiles_begin(self._h, _lib.QUANTILE_SOURCES[source], int(bool(groups)),
                                                                lv[0], lv[1], C.byref(mx)))
        self._sq_shape = self.sharded_quantiles_shape(q, source, groups)
        return int(mx.value)

    def sharded_quantiles_round(self, reduced, reduced_bytes: int, partial) -> int:
        """One round: `reduced` holds the ranks' u32 sum of this rank's last partial (None, 0 on the first round),
        `partial` (at least the begin's bytes; numpy or a torch CUDA tensor) receives this round's words.  Returns their
        size in bytes; 0: the table is ready (sharded_quantiles_end)."""
        rp, _ = self._words(reduced)
        pp, pcap = self._words(partial)
        out = C.c_uint64(0)
        _lib.check(self._L.b200_sixdof_sharded_quantiles_round(self._h, C.c_void_p(rp), int(reduced_bytes),
                                                                C.c_void_p(pp), pcap, C.byref(out)))
        return int(out.value)

    def sharded_quantiles_end(self) -> np.ndarray:
        """The table of the call, with the shape and bits of the unsharded entry on one handle holding every rank's
        worlds in rank order."""
        shape = getattr(self, "_sq_shape", ())
        out = np.empty(shape)
        _lib.check(self._L.b200_sixdof_sharded_quantiles_end(self._h, C.c_void_p(out.ctypes.data), out.nbytes))
        return out

    # ---- ensemble covariance (co-moments of a plane selection over the world axis, on the device) --------------
    @staticmethod
    def _selection(planes) -> tuple:
        """planes -> the (planes, n_p) arguments of the covariance entries."""
        sel = np.ascontiguousarray(np.atleast_1d(np.asarray(planes, dtype=np.uint32)).ravel())
        return sel.ctypes.data_as(C.POINTER(C.c_uint32)), sel.size  # the pointer keeps sel alive

    def trajectory_covariance(self, planes, out_ptr: Optional[int] = None) -> Optional[np.ndarray]:
        """The ring's samples: for the planes `planes` of the 25-plane sample layout, [samples, n_entities, 1 + p + p*p]
        records (n, mean[p], M[p][p] = co-moments) over the worlds whose p selected values are all finite (NaN after
        n where n = 0).  With `out_ptr` (a host or device pointer) the table is written there and nothing is returned."""
        sel = self._selection(planes)
        return self._reduce("covariance", True, sel, self._planes(ring=True)[:-1] + (1 + sel[1] + sel[1] ** 2,), out_ptr)

    def state_covariance(self, planes) -> np.ndarray:
        """The current state: [n_entities, 1 + p + p*p] records as trajectory_covariance()."""
        sel = self._selection(planes)
        return self._reduce("covariance", False, sel, self._planes(ring=False)[:-1] + (1 + sel[1] + sel[1] ** 2,))

    # ---- ensemble histograms (bin counts over the world axis, on the device) ---------------------------------------
    @staticmethod
    def _hist_specs(specs) -> tuple:
        """specs -> ((specs, n_specs) arguments of the histogram entries, f64 per row).  A spec is (entity row, planes,
        bins, lo, hi): one number each for 1D (plane of the 25-plane sample layout), a pair each for 2D."""
        specs = list(specs)
        arr = (_lib.Histogram * max(len(specs), 1))()
        row = 0
        for k, (entity, planes, bins, lo, hi) in enumerate(specs):
            planes, bins, lo, hi = (np.atleast_1d(np.asarray(v)).ravel() for v in (planes, bins, lo, hi))
            h = arr[k]
            h.entity, h.n_axes = int(entity), len(planes)
            for a in range(min(len(planes), 2)):
                h.plane[a], h.bins[a], h.lo[a], h.hi[a] = int(planes[a]), int(bins[a]), float(lo[a]), float(hi[a])
            cells = int(np.prod([int(b) for b in bins[:2]]))
            row += (2 if len(planes) == 2 else 3) + min(max(cells, 0), _lib.MAX_HISTOGRAM_CELLS)  # refused specs: C says why
        return (arr, len(specs)), row

    def trajectory_histograms(self, specs, out_ptr: Optional[int] = None) -> Optional[np.ndarray]:
        """The ring's samples: [samples, sum of the record lengths] f64, each row the specs' records in spec order -- 1D
        [nonfinite, below, above, counts[n]], 2D [nonfinite, outside, counts[na * nb]] (row-major), integer counts over
        the worlds with numpy's histogram / histogram2d rules.  With `out_ptr` (a host or device pointer) the table is
        written there and nothing is returned."""
        args, row = self._hist_specs(specs)
        return self._reduce("histograms", True, args, (self.trajectory_len(), row), out_ptr)

    def state_histograms(self, specs) -> np.ndarray:
        """The current state: [sum of the record lengths] f64, records as trajectory_histograms()."""
        args, row = self._hist_specs(specs)
        return self._reduce("histograms", False, args, (row,))

    # ---- grouped ensembles (the statistics and histograms above, one table per contiguous world range) ----------
    def set_world_groups(self, sizes) -> None:
        """Split the worlds into consecutive groups of `sizes` worlds (each >= 0, summing to n_worlds, at most
        MAX_WORLD_GROUPS); an empty `sizes` clears the setting.  The ungrouped tables are unchanged by it."""
        sz = np.ascontiguousarray(np.asarray(list(sizes), dtype=np.uint64).ravel())
        _lib.check(self._L.b200_sixdof_set_world_groups(self._h, sz.ctypes.data_as(C.POINTER(C.c_uint64)), sz.size))

    @property
    def world_groups(self) -> int:
        """The number of groups set, 0 = none."""
        return int(self._L.b200_sixdof_world_groups(self._h))

    def trajectory_group_stats(self) -> np.ndarray:
        """trajectory_stats() per group: [samples, G, n_entities, width, 5]; group g's record has the bits of
        trajectory_stats() on a batch of exactly its worlds."""
        n, E, W = self._rows(ring=True)
        return self._reduce("group_stats", True, (), (n, self.world_groups, E, W, _lib.STATS_FIELDS))

    def state_group_stats(self) -> np.ndarray:
        """state_stats() per group: [G, n_entities, 25, 5]."""
        return self._reduce("group_stats", False, (), (self.world_groups,) + self._rows(ring=False) + (_lib.STATS_FIELDS,))

    def trajectory_group_histograms(self, specs) -> np.ndarray:
        """trajectory_histograms(specs) per group: [samples, G, sum of the record lengths]."""
        args, row = self._hist_specs(specs)
        return self._reduce("group_histograms", True, args, (self.trajectory_len(), self.world_groups, row))

    def state_group_histograms(self, specs) -> np.ndarray:
        """state_histograms(specs) per group: [G, sum of the record lengths]."""
        args, row = self._hist_specs(specs)
        return self._reduce("group_histograms", False, args, (self.world_groups, row))

    def trajectory_group_quantiles(self, q) -> np.ndarray:
        """trajectory_quantiles(q) per group: [samples, G, n_entities, width, n_q]; group g's quantiles have the bits of
        trajectory_quantiles(q) on a batch of exactly its worlds (NaN for an empty group).  A world-sharded campaign
        reduces them over every rank's worlds with sharding.gather_quantiles(ex, q, "ring", groups=True)."""
        lv = self._levels(q)
        n, E, W = self._rows(ring=True)
        return self._reduce("group_quantiles", True, lv, (n, self.world_groups, E, W, lv[1]))

    def state_group_quantiles(self, q) -> np.ndarray:
        """state_quantiles(q) per group: [G, n_entities, 25, n_q]."""
        lv = self._levels(q)
        return self._reduce("group_quantiles", False, lv, (self.world_groups,) + self._rows(ring=False) + (lv[1],))

    def trajectory_group_covariance(self, planes) -> np.ndarray:
        """trajectory_covariance(planes) per group: [samples, G, n_entities, 1 + p + p*p]; group g's records have the
        bits of trajectory_covariance(planes) on a batch of exactly its worlds (n = 0 and NaN for an empty group).
        The tables of a world-sharded campaign, with groups cut by sharding.shard_groups, merge with
        merge_covariance."""
        sel = self._selection(planes)
        n, E, _ = self._planes(ring=True)
        return self._reduce("group_covariance", True, sel, (n, self.world_groups, E, 1 + sel[1] + sel[1] ** 2))

    def state_group_covariance(self, planes) -> np.ndarray:
        """state_covariance(planes) per group: [G, n_entities, 1 + p + p*p]."""
        sel = self._selection(planes)
        return self._reduce("group_covariance", False, sel, (self.world_groups, self.n_entities, 1 + sel[1] + sel[1] ** 2))

    # ---- derived channels (per-body values computed on the device, reduced as planes 25 + k) --------------------
    def set_channels(self, channels: Sequence) -> None:
        """Replace the channel set with `channels` (at most MAX_CHANNELS _lib.Channel records, or tuples (kind, n,
        planes, c, d, r0)); an empty set clears it.  Channel k is plane 25 + k of every ensemble table's rows.  Must come
        before summary_begin."""
        chans = list(channels)
        arr = (_lib.Channel * max(len(chans), 1))()
        for k, c in enumerate(chans):
            arr[k] = c if isinstance(c, _lib.Channel) else _lib.channel(*c)
        _lib.check(self._L.b200_sixdof_set_channels(self._h, arr, len(chans)))

    @property
    def n_channels(self) -> int:
        """The number of channels set, 0 = none."""
        return int(self._L.b200_sixdof_channels(self._h))

    def trajectory_channels(self, out_ptr: Optional[int] = None) -> Optional[np.ndarray]:
        """The channels of the ring's samples, recomputed on the device: [samples, n_worlds, n_entities, n_c].  With
        `out_ptr` (a host or device pointer) they are written there and nothing is returned."""
        return self._reduce("channels", True, (), (self.trajectory_len(), self.n_worlds, self.n_entities,
                                                   self.n_channels), out_ptr)

    def state_channels(self) -> np.ndarray:
        """The channels of the current state: [n_worlds, n_entities, n_c]."""
        return self._reduce("channels", False, (), (self.n_worlds, self.n_entities, self.n_channels))

    # ---- outcomes (one value per world, from the run summaries, a column or host values, reduced over the worlds)
    def set_outcomes(self, outcomes: Sequence) -> None:
        """Replace the outcome set with `outcomes` (at most MAX_OUTCOMES _lib.Outcome records, or tuples (kind, field,
        index, entity, column, values) with the trailing items optional: column a component name or id, values
        n_worlds f64 for OUTCOME_VALUES); an empty set clears it.  Outcomes name summaries of the summary in force:
        call it after summary_begin."""
        outs = list(outcomes)
        arr = (_lib.Outcome * max(len(outs), 1))()
        keep = []  # the values arrays, alive for the call (the library copies them)
        for k, o in enumerate(outs):
            if isinstance(o, _lib.Outcome):
                arr[k] = o
                continue
            kind, field, index, entity, column, values = tuple(o) + (0, 0, 0, None)[len(o) - 2:]
            r = arr[k]
            r.kind, r.field, r.index, r.entity = int(kind), int(field), int(index), int(entity)
            r.column = _cid(column) if column else 0
            if values is not None:
                keep.append(np.ascontiguousarray(np.asarray(values, dtype=np.float64).ravel()))
                r.values = keep[-1].ctypes.data_as(C.POINTER(C.c_double))
        _lib.check(self._L.b200_sixdof_set_outcomes(self._h, arr, len(outs)))

    @property
    def n_outcomes(self) -> int:
        """The number of outcomes set, 0 = none."""
        return int(self._L.b200_sixdof_outcomes(self._h))

    def outcome_values(self) -> np.ndarray:
        """[n_worlds, P]: every outcome's value of every world, written on the device now (-1 ticks as NaN)."""
        return self._reduce("values", "outcome", (), (self.n_worlds, self.n_outcomes))

    def outcome_stats(self) -> np.ndarray:
        """[P, 5]: state_stats()'s fields of every outcome over the worlds."""
        return self._reduce("stats", "outcome", (), (self.n_outcomes, _lib.STATS_FIELDS))

    def outcome_group_stats(self) -> np.ndarray:
        """[G, P, 5]: outcome_stats() per group of set_world_groups."""
        return self._reduce("group_stats", "outcome", (), (self.world_groups, self.n_outcomes, _lib.STATS_FIELDS))

    def outcome_quantiles(self, q) -> np.ndarray:
        """[P, n_q]: state_quantiles()'s levels of every outcome over the worlds whose value is finite."""
        lv = self._levels(q)
        return self._reduce("quantiles", "outcome", lv, (self.n_outcomes, lv[1]))

    def outcome_group_quantiles(self, q) -> np.ndarray:
        """[G, P, n_q]: outcome_quantiles(q) per group."""
        lv = self._levels(q)
        return self._reduce("group_quantiles", "outcome", lv, (self.world_groups, self.n_outcomes, lv[1]))

    def outcome_covariance(self, planes) -> np.ndarray:
        """[1 + p + p*p]: the covariance record of the outcomes `planes` (indices below P), as state_covariance()."""
        sel = self._selection(planes)
        return self._reduce("covariance", "outcome", sel, (1 + sel[1] + sel[1] ** 2,))

    def outcome_group_covariance(self, planes) -> np.ndarray:
        """[G, 1 + p + p*p]: outcome_covariance(planes) per group."""
        sel = self._selection(planes)
        return self._reduce("group_covariance", "outcome", sel, (self.world_groups, 1 + sel[1] + sel[1] ** 2))

    def outcome_histograms(self, specs) -> np.ndarray:
        """[sum of the record lengths]: state_histograms(specs) of the outcomes (entity row 0, planes below P)."""
        args, row = self._hist_specs(specs)
        return self._reduce("histograms", "outcome", args, (row,))

    def outcome_group_histograms(self, specs) -> np.ndarray:
        """[G, sum of the record lengths]: outcome_histograms(specs) per group."""
        args, row = self._hist_specs(specs)
        return self._reduce("group_histograms", "outcome", args, (self.world_groups, row))

    def outcome_top_worlds(self, planes, k: int, largest) -> np.ndarray:
        """[p, 1 + 2k]: per outcome of `planes` (distinct indices below P) the record [count, values[k], worlds[k]] of
        the first min(k, count) worlds whose value is finite, ordered by value (IEEE totalOrder, -0 < +0; descending
        when `largest`), ties by ascending world index; slots past count hold NaN and -1."""
        sel = self._selection(planes)
        return self._reduce("top_worlds", "outcome", sel + (int(k), int(largest)), (sel[1], 1 + 2 * int(k)))

    def outcome_group_top_worlds(self, planes, k: int, largest) -> np.ndarray:
        """[G, p, 1 + 2k]: outcome_top_worlds(planes, k, largest) per group; worlds are the handle's world indices."""
        sel = self._selection(planes)
        return self._reduce("group_top_worlds", "outcome", sel + (int(k), int(largest)),
                            (self.world_groups, sel[1], 1 + 2 * int(k)))

    def top_worlds_reads(self) -> float:
        """Reads of the outcome planes the last top-worlds call made, averaged over its (group, plane) tasks."""
        return float(self._L.b200_sixdof_top_worlds_reads(self._h))

    def outcome_ranks(self, planes) -> np.ndarray:
        """[n_worlds, p]: the midrank of every world in each outcome of `planes` (distinct indices below P) among the
        worlds whose p selected values are all finite (scipy.stats.rankdata(method="average"), -0 == +0); NaN for the
        other worlds."""
        sel = self._selection(planes)
        return self._reduce("ranks", "outcome", sel, (self.n_worlds, sel[1]))

    def outcome_group_ranks(self, planes) -> np.ndarray:
        """[n_worlds, p]: outcome_ranks(planes) within each group of set_world_groups."""
        sel = self._selection(planes)
        return self._reduce("group_ranks", "outcome", sel, (self.n_worlds, sel[1]))

    def outcome_rank_correlation(self, planes) -> np.ndarray:
        """[1 + p*p]: [n, rho[p][p]], the Spearman correlation of the outcomes `planes` (p >= 2) over the worlds whose p
        values are all finite: the covariance record of their ranks, rho = M[a][b] / sqrt(M[a][a] * M[b][b]), NaN in
        the row and column of a constant plane and everywhere when n < 2."""
        sel = self._selection(planes)
        return self._reduce("rank_correlation", "outcome", sel, (1 + sel[1] ** 2,))

    def outcome_group_rank_correlation(self, planes) -> np.ndarray:
        """[G, 1 + p*p]: outcome_rank_correlation(planes) per group."""
        sel = self._selection(planes)
        return self._reduce("group_rank_correlation", "outcome", sel, (self.world_groups, 1 + sel[1] ** 2))

    def rank_reads(self) -> float:
        """Reads of the outcome planes the last rank call made, averaged over its (group, plane) tasks."""
        return float(self._L.b200_sixdof_rank_reads(self._h))

    def outcome_sobol(self, planes, d: int, n_boot: int, seed: int) -> np.ndarray:
        """[p, 3 + 4d]: per outcome of `planes` (distinct indices below P) of a Saltelli campaign of d inputs
        (monte_carlo.saltelli: blocks of d + 2 worlds), the record [n, V, n_boot_ok, S1[d], ST[d], S1_sd[d], ST_sd[d]]:
        the first-order and total Sobol indices and the standard deviations of n_boot bootstrap resamples drawn from
        `seed` (include/b200_sixdof.h b200_sixdof_outcome_sobol)."""
        sel = self._selection(planes)
        args = sel + (int(d), int(n_boot), int(seed) % (1 << 64))
        return self._reduce("sobol", "outcome", args, (sel[1], 3 + 4 * int(d)))

    def outcome_group_sobol(self, planes, d: int, n_boot: int, seed: int) -> np.ndarray:
        """[G, p, 3 + 4d]: outcome_sobol(planes, d, n_boot, seed) per group of set_world_groups."""
        sel = self._selection(planes)
        args = sel + (int(d), int(n_boot), int(seed) % (1 << 64))
        return self._reduce("group_sobol", "outcome", args, (self.world_groups, sel[1], 3 + 4 * int(d)))

    # ---- world-sharded ranks: the midranks of the union of every rank's worlds, in rounds ----------------------------
    def sharded_ranks_begin(self, planes, groups: bool, rank: int, n_ranks: int) -> int:
        """Begin this rank's part of a world-sharded rank call (b200_sixdof_sharded_ranks_begin): the outcomes
        `planes`, the grouping, this rank's index and the rank count are fixed here.  Returns the largest round in bytes
        (the partial buffer's least size)."""
        sel = self._selection(planes)
        mx = C.c_uint64(0)
        _lib.check(self._L.b200_sixdof_sharded_ranks_begin(self._h, int(bool(groups)), sel[0], sel[1], int(rank),
                                                            int(n_ranks), C.byref(mx)))
        self._sr_shape = (sel[1], self.world_groups if groups else 1)
        return int(mx.value)

    def sharded_ranks_round(self, reduced, reduced_bytes: int, partial) -> int:
        """One round, as sharded_quantiles_round; 0: the ranks are ready (sharded_ranks_end)."""
        rp, _ = self._words(reduced)
        pp, pcap = self._words(partial)
        out = C.c_uint64(0)
        _lib.check(self._L.b200_sixdof_sharded_ranks_round(self._h, C.c_void_p(rp), int(reduced_bytes), C.c_void_p(pp),
                                                            pcap, C.byref(out)))
        return int(out.value)

    def sharded_ranks_end(self, ranks: bool = True, covariance: bool = True) -> tuple:
        """(ranks [n_worlds, p] or None, covariance [G or 1, 1 + p + p*p] or None): the campaign midranks of this
        rank's worlds, with the bits of outcome_[group_]ranks on one handle holding every rank's worlds in rank order,
        and the covariance records of this rank's rank planes (merge them over the ranks with merge_covariance)."""
        p, G = getattr(self, "_sr_shape", (0, 1))
        r = np.empty((self.n_worlds, p)) if ranks else None
        c = np.empty((G, 1 + p + p * p)) if covariance else None
        ptr = lambda a: C.c_void_p(a.ctypes.data if a is not None else None)
        _lib.check(self._L.b200_sixdof_sharded_ranks_end(self._h, ptr(r), r.nbytes if ranks else 0, ptr(c),
                                                          c.nbytes if covariance else 0))
        return r, c

    # ---- run summaries (reductions over the time axis, per world, on the device) --------------------------------
    @staticmethod
    def _conditions(rows: Sequence):
        """(entity row, plane, above, value) tuples -> a Threshold array (at least one element) and its length."""
        rows = list(rows)
        arr = (_lib.Threshold * max(len(rows), 1))()
        for i, (entity, plane, above, value) in enumerate(rows):
            arr[i] = _lib.Threshold(int(entity), int(plane), 1 if above else 0, float(value))
        return arr, len(rows)

    def summary_begin(self, extrema: bool, thresholds: Sequence = (), moments: Sequence = (), dwells: Sequence = ()) -> None:
        """Start (or start over) the run summaries: `extrema` keeps per-(world, entity, plane) extrema; `thresholds` =
        up to 8 (entity row, plane 0..24 or 25 + channel, above, value) tuples, each firing on value > bound (above) or < bound;
        `moments` = distinct planes (0..24 or 25 + channel) whose run count, mean and m2 are kept per (world, entity);
        `dwells` = up to 8 tuples as `thresholds`, each counting the rows beyond its bound.  Without moments and dwells
        this is b200_sixdof_summary_begin, else b200_sixdof_summary_start."""
        thr, n_thr = self._conditions(thresholds)
        mom = np.ascontiguousarray(np.asarray(list(moments), dtype=np.uint32).ravel())
        dwl, n_dwl = self._conditions(dwells)
        if mom.size == 0 and n_dwl == 0:
            _lib.check(self._L.b200_sixdof_summary_begin(self._h, 1 if extrema else 0, thr, n_thr))
        else:
            spec = _lib.SummarySpec(1 if extrema else 0, n_thr, thr, mom.size, n_dwl,
                                    mom.ctypes.data_as(C.POINTER(C.c_uint32)), dwl)
            _lib.check(self._L.b200_sixdof_summary_start(self._h, C.byref(spec)))
        self._n_thresholds, self._n_moments, self._n_dwells = n_thr, mom.size, n_dwl

    def summary_add_state(self) -> None:
        """Fold the current device state as one row at the current tick."""
        _lib.check(self._L.b200_sixdof_summary_add_state(self._h))

    def summary_add_trajectory(self) -> None:
        """Fold every sample now in the (trajectory_full) ring, each at the tick it was recorded."""
        _lib.check(self._L.b200_sixdof_summary_add_trajectory(self._h))

    def extrema(self) -> np.ndarray:
        """[n_worlds, n_entities, 25 + n_c, 5]: (min, max, min_tick, max_tick, first_nonfinite_tick) of every plane of
        the B200_TRAJ_FULL row layout, then of every channel, over the rows folded; min / max over the finite values (NaN if none), ticks -1 where
        they never applied."""
        out = np.empty((self.n_worlds,) + self._rows(ring=False) + (_lib.EXTREMA_FIELDS,))
        _lib.check(self._L.b200_sixdof_extrema_download(self._h, out.ctypes.data, out.nbytes))
        return out

    def thresholds(self) -> np.ndarray:
        """[n_worlds, n_thresholds, 26]: the tick of each threshold's first firing row (-1 = never), then the
        entity's 25 planes at that row (NaN if it never fired)."""
        out = np.empty((self.n_worlds, getattr(self, "_n_thresholds", 0), 26))
        _lib.check(self._L.b200_sixdof_thresholds_download(self._h, out.ctypes.data, out.nbytes))
        return out

    def moments(self) -> np.ndarray:
        """[n_worlds, n_entities, k, 3]: (n, mean, m2 = sum (x - mean)^2) over each world's finite rows of each of the k
        planes of `moments`, in the order given (n = 0: NaN mean and m2; m2 = +inf where the sum of squares overflowed)."""
        out = np.empty((self.n_worlds, self.n_entities, getattr(self, "_n_moments", 0), _lib.MOMENT_FIELDS))
        _lib.check(self._L.b200_sixdof_moments_download(self._h, out.ctypes.data, out.nbytes))
        return out

    def dwells(self) -> np.ndarray:
        """[n_worlds, n_dwells, 3]: (rows, first_tick, last_tick) of the rows beyond each dwell's bound (ticks -1 while
        no row has counted)."""
        out = np.empty((self.n_worlds, getattr(self, "_n_dwells", 0), _lib.DWELL_FIELDS))
        _lib.check(self._L.b200_sixdof_dwells_download(self._h, out.ctypes.data, out.nbytes))
        return out

    # ---- plumbing ---------------------------------------------------------------
    def set_stream(self, cuda_stream: Optional[int]) -> None:
        """Run on a caller-owned cudaStream_t (0 = the legacy default stream, which is what
        torch.cuda.current_stream().cuda_stream returns by default); None = private stream."""
        if cuda_stream is None:
            _lib.check(self._L.b200_sixdof_set_stream(self._h, C.c_void_p(0), 1))
        else:
            _lib.check(self._L.b200_sixdof_set_stream(self._h, C.c_void_p(int(cuda_stream)), 0))

    def timings(self) -> dict:
        t = _lib.Timings()
        _lib.check(self._L.b200_sixdof_timings(self._h, C.byref(t)))
        return {"h2d_upload_ms": t.h2d_upload_ms, "kernel_invoke_ms": t.kernel_invoke_ms,
                "d2h_download_ms": t.d2h_download_ms, "invoke_wall_ms": t.invoke_wall_ms,
                "kernel_launches": int(t.kernel_launches),
                "ticks": int(t.ticks)}

    def device_plane(self, cid, plane: int) -> int:
        return int(self._L.b200_sixdof_device_plane(self._h, _cid(cid), plane) or 0)

    @property
    def plane_stride(self) -> int:
        return int(self._L.b200_sixdof_plane_stride(self._h))


def _stack(tables: Sequence[np.ndarray], merge: str, layout: str, record_ok) -> np.ndarray:
    """The tables to `merge` as one contiguous f64 array [n_tables, ...]: at least one, all of one shape [..., layout]
    whose record width (the last axis) passes `record_ok`; B200ValueError otherwise."""
    parts = [np.asarray(t, dtype=np.float64) for t in tables]
    if not parts:
        raise _lib.B200ValueError(_lib.ERR_VALUE_SIZE_MISMATCH, f"{merge} needs at least one table")
    shape = parts[0].shape
    if not (shape and record_ok(shape[-1])) or any(p.shape != shape for p in parts):
        raise _lib.B200ValueError(_lib.ERR_VALUE_SIZE_MISMATCH,
                                  f"{merge}: the tables must share one shape [..., {layout}], got {[p.shape for p in parts]}")
    return np.ascontiguousarray(np.stack(parts))


def merge_stats(tables: Sequence[np.ndarray]) -> np.ndarray:
    """Merge statistics tables of the same shape [..., 5] (e.g. one per rank of a world-sharded campaign, or per
    handle) left to right, in list order, with b200_stats_merge: the table of the union of their worlds."""
    stacked = _stack(tables, "merge_stats", "5", lambda rec: rec == _lib.STATS_FIELDS)
    out = np.empty(stacked.shape[1:])
    dp = C.POINTER(C.c_double)
    _lib.check(_lib.lib().b200_stats_merge(stacked.ctypes.data_as(dp), len(stacked), out.size // _lib.STATS_FIELDS,
                                            out.ctypes.data_as(dp)))
    return out


def merge_covariance(tables: Sequence[np.ndarray]) -> np.ndarray:
    """Merge covariance tables of the same shape [..., 1 + p + p*p] (e.g. one per rank of a world-sharded campaign, or
    per handle) left to right, in list order, with b200_covariance_merge: the table of the union of their worlds."""
    p = lambda rec: math.isqrt(max(rec - 1, 0))  # p^2 <= p^2 + p < (p + 1)^2
    stacked = _stack(tables, "merge_covariance", "1 + p + p*p", lambda rec: rec >= 3 and p(rec) ** 2 + p(rec) + 1 == rec)
    out = np.empty(stacked.shape[1:])
    rec = out.shape[-1]
    dp = C.POINTER(C.c_double)
    _lib.check(_lib.lib().b200_covariance_merge(stacked.ctypes.data_as(dp), len(stacked), out.size // rec, p(rec),
                                                 out.ctypes.data_as(dp)))
    return out


def merge_histograms(tables: Sequence[np.ndarray]) -> np.ndarray:
    """Merge histogram tables of the same shape (e.g. one per rank of a world-sharded campaign, or per handle): their
    elementwise sum, which is exactly the table of the union of their worlds.  Every value must be a count (a
    non-negative integer) and every sum at most 2^53, where f64 counts stay exact."""
    stacked = _stack(tables, "merge_histograms", "records", lambda rec: rec >= 3)
    if not np.all((stacked >= 0) & (stacked == np.floor(stacked))):
        raise _lib.B200Error(_lib.ERR_INVALID_ARGUMENT, "merge_histograms: a value is not a count")
    out = stacked.sum(axis=0)
    if np.any(out > 2.0 ** 53):
        raise _lib.B200Error(_lib.ERR_INVALID_ARGUMENT, "merge_histograms: a count exceeds 2^53")
    return out


def top_world_keys(values, largest) -> np.ndarray:
    """The sort keys of the worst-worlds order: the IEEE totalOrder key of each f64 value (-0 < +0) as uint64,
    complemented when `largest`, so that ascending (key, world) is the order of b200_sixdof_outcome_top_worlds."""
    u = np.ascontiguousarray(values, dtype=np.float64).view(np.uint64)
    key = np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))
    return ~key if largest else key


def merge_top_worlds(tables: Sequence[np.ndarray], offsets: Sequence[int], largest) -> np.ndarray:
    """Merge worst-worlds tables of the same shape [..., 1 + 2k] (one per rank of a world-sharded campaign, in rank
    order, or per handle): table r's worlds are shifted by offsets[r] (its first world in the campaign), the candidates
    of every table re-ordered by (key, world) and the first k kept; the counts add up.  Exact: the ranks hold contiguous
    world ranges in rank order, so each rank's tie order by local index is the campaign's."""
    stacked = _stack(tables, "merge_top_worlds", "1 + 2k", lambda rec: rec >= 3 and rec % 2 == 1)
    if len(offsets) != len(stacked):
        raise ValueError(f"merge_top_worlds: {len(stacked)} tables and {len(offsets)} offsets")
    k = (stacked.shape[-1] - 1) // 2
    flat = stacked.reshape(len(stacked), -1, 1 + 2 * k)
    out = np.empty(flat.shape[1:])
    for t in range(flat.shape[1]):
        vals, worlds = [], []
        for r, rec in enumerate(flat[:, t]):
            n = min(int(rec[0]), k)
            vals.append(rec[1:1 + n])
            worlds.append(rec[1 + k:1 + k + n] + float(offsets[r]))
        v, w = np.concatenate(vals), np.concatenate(worlds)
        top = np.lexsort((w, top_world_keys(v, largest)))[:k]
        n = top.size
        out[t, 0] = flat[:, t, 0].sum()
        out[t, 1:1 + k] = np.nan
        out[t, 1 + k:] = -1.0
        out[t, 1:1 + n] = v[top]
        out[t, 1 + k:1 + k + n] = w[top]
    return out.reshape(stacked.shape[1:])


def rank_correlation(cov: np.ndarray, p: int) -> np.ndarray:
    """The rank correlation records [..., 1 + p*p] of covariance records [..., 1 + p + p*p] of rank planes, as the
    device computes them: rho[a][b] = M[a][b] / sqrt(M[a][a] * M[b][b]) (each operation correctly rounded, so the
    same bits), NaN where n < 2 or M[a][a] or M[b][b] is not > 0."""
    cov = np.asarray(cov, dtype=np.float64)
    n = cov[..., :1]
    M = cov[..., 1 + p:].reshape(*cov.shape[:-1], p, p)
    d = np.diagonal(M, axis1=-2, axis2=-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        rho = M / np.sqrt(d[..., :, None] * d[..., None, :])
    ok = (n[..., None] >= 2) & (d[..., :, None] > 0) & (d[..., None, :] > 0)
    rho = np.where(ok, rho, np.nan)
    return np.concatenate([n, rho.reshape(*cov.shape[:-1], p * p)], axis=-1)


def sobol_indices(cov: np.ndarray, d: int) -> tuple:
    """(n, V, S1 [..., d], ST [..., d]) of covariance records [..., 1 + q + q*q] (q = d + 2) of the derived planes
    (a, b, D_1 .. D_d) of a Saltelli campaign, as the device computes them (include/b200_sixdof.h
    b200_sixdof_outcome_sobol; each operation correctly rounded in the same order, so the same bits):
    V = (M_aa + M_bb) / (2n) + ((m_a - m_b) * (m_a - m_b)) * 0.25, S1_i = (M_bDi / n + m_b m_Di) / V,
    ST_i = (M_DiDi / n + m_Di m_Di) / (2V).  V is NaN where n < 2; S1 and ST are NaN where n < 2 or V is not > 0."""
    cov = np.asarray(cov, dtype=np.float64)
    q = d + 2
    n = cov[..., 0]
    m = cov[..., 1:1 + q]
    M = cov[..., 1 + q:].reshape(*cov.shape[:-1], q, q)
    with np.errstate(invalid="ignore", divide="ignore"):
        dab = m[..., 0] - m[..., 1]
        V = (M[..., 0, 0] + M[..., 1, 1]) / (2.0 * n) + (dab * dab) * 0.25
        Md = np.diagonal(M, axis1=-2, axis2=-1)[..., 2:]
        EbD = M[..., 1, 2:] / n[..., None] + m[..., 1:2] * m[..., 2:]
        EDD = Md / n[..., None] + m[..., 2:] * m[..., 2:]
        S1 = EbD / V[..., None]
        ST = EDD / (2.0 * V[..., None])
    ok = ((n >= 2) & (V > 0))[..., None]
    return n, np.where(n >= 2, V, np.nan), np.where(ok, S1, np.nan), np.where(ok, ST, np.nan)


def partial_rank_correlation(R: np.ndarray) -> np.ndarray:
    """PRCC from a rank correlation matrix R [..., n_in + 1, n_in + 1] whose last row and column are the output:
    [..., n_in], prcc_i = -P[i, y] / sqrt(P[i, i] * P[y, y]) with P = inv(R); NaN where R holds a NaN, R is singular
    or a diagonal of P is not > 0."""
    R = np.asarray(R, dtype=np.float64)
    k = R.shape[-1]
    flat = R.reshape(-1, k, k)
    out = np.full((flat.shape[0], k - 1), np.nan)
    for t, r in enumerate(flat):
        if not np.all(np.isfinite(r)):
            continue
        try:
            P = np.linalg.inv(r)
        except np.linalg.LinAlgError:
            continue
        if not np.all(np.isfinite(P)) or np.linalg.cond(r) > 1e12:
            continue
        d = np.diagonal(P)
        if not np.all(d > 0):
            continue
        out[t] = -P[:-1, -1] / np.sqrt(d[:-1] * d[-1])
    return out.reshape(*R.shape[:-2], k - 1)


def math_nan() -> float:
    return math.nan


def device_count() -> int:
    n = _lib.lib().b200_device_count()
    return max(int(n), 0)


def pinned_empty(shape, dtype=np.float64, device: Optional[int] = None) -> np.ndarray:
    """numpy array over page-locked host memory (b200_host_alloc); with `device`, on the NUMA node of that
    GPU's PCIe root (b200_host_alloc_local)."""
    L = _lib.lib()
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    p = L.b200_host_alloc(max(n, 1)) if device is None else L.b200_host_alloc_local(max(n, 1), int(device))
    if not p:
        raise _lib.B200Error(_lib.ERR_OUT_OF_MEMORY, L.b200_last_error().decode())
    buf = (C.c_char * max(n, 1)).from_address(p)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
    _PINNED[arr.ctypes.data] = p
    return arr


_PINNED: Dict[int, int] = {}


def pinned_free(arr: np.ndarray) -> None:
    p = _PINNED.pop(arr.ctypes.data, None)
    if p:
        _lib.lib().b200_host_free(C.c_void_p(p))
