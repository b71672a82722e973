"""Trajectory sink in the on-disk format of elodin-db (SURVEY §8f-1).

The reference's simulation server writes every (entity, component) pair of the ECS world into an
elodin-db directory: `init_db` (libs/nox-py/src/impeller2_server.rs:229-309) registers the pairs and
pushes the initial values, `commit_world_head_unified` (:390-438) appends one sample per telemetry
cycle.  `elodin-db export`, the editor and the CI regression gate all read that directory.  This
module writes a B200 run in the same layout, so those consumers open GPU runs unchanged:

    <db>/db_state                       postcard(DbConfig{recording, default_stream_time_step, metadata})
    <db>/<pair_id>/schema               postcard(Schema{prim_type, shape})               lib.rs:1424-1466
    <db>/<pair_id>/metadata             postcard(ComponentMetadata{component_id, name, metadata})
    <db>/<pair_id>/index                AppendLog<Timestamp>:  committed_len u64 | head_len u64 | start i64 | i64 µs ...
    <db>/<pair_id>/data                 AppendLog<u64>:        committed_len u64 | head_len u64 | element_size u64 | rows ...
    <db>/<entity_id>/metadata           entity-level metadata (no schema; skipped by the component scan)

`pair_id` is `ComponentId::new("<entity>.<component>")` printed in decimal (lib.rs:1570-1578).  Both
AppendLog files are sparse 8 GiB (+1 byte) files the reader mmaps (append_log.rs:48-95); `committed_len`
counts the 24-byte header.  postcard is the wire format of the `postcard` crate: LEB128 varints, zigzag
for signed integers, length-prefixed strings / sequences / maps, u32-varint enum discriminants.

`read_db` restates the reader side (`DB::open`, lib.rs:592-670, and `TimeSeries`) for the tests and for
`export_db_csv`, which produces the `elodin-db export --format csv --flatten` layout from a directory.
Nothing here touches the GPU: samples arrive as host arrays from `Exec.history` / the trajectory ring.
"""

from __future__ import annotations

import math
import os
import struct
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from ._lib import component_id

APPEND_LOG_FILE_SIZE = 8 * 1024 * 1024 * 1024  # append_log.rs:56
APPEND_LOG_HEADER = 24                          # committed_len + head_len + extra (8 bytes for both uses)
DB_VERSION = "0.19.0"                           # workspace version of the surveyed reference (Cargo.toml:68)
CREATION_INDEX_KEY = "_creation_index"          # lib.rs:54
_SKIP_DIRS = ("msgs", "assets", "simulation_source")  # lib.rs:606-611

# impeller2/src/types.rs:152-164 — discriminant order of PrimType
PRIM_TYPES = ("u8", "u16", "u32", "u64", "i8", "i16", "i32", "i64", "bool", "f32", "f64")
_PRIM_NUMPY = {"u8": "<u1", "u16": "<u2", "u32": "<u4", "u64": "<u8", "i8": "<i1", "i16": "<i2", "i32": "<i4",
               "i64": "<i8", "bool": "?", "f32": "<f4", "f64": "<f8"}


# ---------------------------------------------------------------------------------------------------
# postcard
# ---------------------------------------------------------------------------------------------------

def pc_varint(v: int) -> bytes:
    if v < 0:
        raise ValueError("varint of a negative value")
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def pc_zigzag(v: int, bits: int = 64) -> bytes:
    return pc_varint(((v << 1) ^ (v >> (bits - 1))) & ((1 << bits) - 1))


def pc_str(s: str) -> bytes:
    b = s.encode("utf-8")
    return pc_varint(len(b)) + b


def pc_map(m: Dict[str, str]) -> bytes:
    out = pc_varint(len(m))
    for k, v in m.items():
        out += pc_str(k) + pc_str(v)
    return out


class _Reader:
    def __init__(self, data: bytes):
        self.d, self.i = data, 0

    def varint(self) -> int:
        v = shift = 0
        while True:
            b = self.d[self.i]
            self.i += 1
            v |= (b & 0x7F) << shift
            if not b & 0x80:
                return v
            shift += 7
            if shift > 70:
                raise ValueError("varint too long")

    def string(self) -> str:
        n = self.varint()
        s = self.d[self.i:self.i + n].decode("utf-8")
        if len(self.d) < self.i + n:
            raise ValueError("truncated string")
        self.i += n
        return s

    def map(self) -> Dict[str, str]:
        return {self.string(): self.string() for _ in range(self.varint())}

    def done(self) -> None:
        if self.i != len(self.d):
            raise ValueError(f"{len(self.d) - self.i} trailing bytes")


@dataclass
class Schema:
    """`Schema{prim_type, shape}` (impeller2/src/schema.rs:11-16); ComponentSchema serialises as this."""

    prim_type: str = "f64"
    shape: Tuple[int, ...] = ()

    def encode(self) -> bytes:
        out = pc_varint(PRIM_TYPES.index(self.prim_type)) + pc_varint(len(self.shape))
        for d in self.shape:
            out += pc_varint(int(d))
        return out

    @staticmethod
    def decode(data: bytes) -> "Schema":
        r = _Reader(data)
        prim = PRIM_TYPES[r.varint()]
        shape = tuple(r.varint() for _ in range(r.varint()))
        r.done()
        return Schema(prim, shape)

    @property
    def size(self) -> int:  # ComponentSchema::size, lib.rs:1451-1453
        return int(np.prod(self.shape, dtype=np.int64)) * np.dtype(_PRIM_NUMPY[self.prim_type]).itemsize

    @property
    def dtype(self) -> np.dtype:
        return np.dtype(_PRIM_NUMPY[self.prim_type])


@dataclass
class ComponentMetadata:
    """impeller2/wkt/src/metadata.rs:8-13"""

    component_id: int
    name: str
    metadata: Dict[str, str] = field(default_factory=dict)

    def encode(self) -> bytes:
        return pc_varint(self.component_id) + pc_str(self.name) + pc_map(self.metadata)

    @staticmethod
    def decode(data: bytes) -> "ComponentMetadata":
        r = _Reader(data)
        m = ComponentMetadata(r.varint(), r.string(), r.map())
        r.done()
        return m


@dataclass
class DbConfig:
    """impeller2/wkt/src/msgs.rs:291-295; Duration serialises as (secs: u64, nanos: u32)."""

    recording: bool = False
    default_stream_time_step_ns: int = 16_666_667
    metadata: Dict[str, str] = field(default_factory=dict)

    def encode(self) -> bytes:
        secs, nanos = divmod(self.default_stream_time_step_ns, 1_000_000_000)
        return bytes([1 if self.recording else 0]) + pc_varint(secs) + pc_varint(nanos) + pc_map(self.metadata)

    @staticmethod
    def decode(data: bytes) -> "DbConfig":
        r = _Reader(data)
        rec = r.d[r.i] != 0
        r.i += 1
        secs, nanos = r.varint(), r.varint()
        c = DbConfig(rec, secs * 1_000_000_000 + nanos, r.map())
        r.done()
        return c


def duration_ns(seconds: float) -> int:
    """`Duration::from_secs_f64(s).as_nanos()`: nearest nanosecond (same rule as world.quantised_time_step)."""
    if not (seconds >= 0.0) or math.isinf(seconds):
        raise ValueError(f"duration must be finite and non-negative, got {seconds}")
    return int(np.rint(seconds * 1.0e9))


def pair_id(entity: str, component: str) -> int:
    """ComponentId::from_pair (impeller2/src/types.rs:54-59) == ComponentId::new("entity.component")."""
    return component_id(f"{entity}.{component}")


def _metadata_strings(md: dict) -> Dict[str, str]:
    """PyComponent::new (libs/nox-py/src/component.rs:81-95): str as is, numbers through f64 Display."""
    out = {}
    for k, v in md.items():
        if isinstance(v, str):
            out[k] = v
        elif isinstance(v, bool):
            out[k] = "1" if v else "0"
        elif isinstance(v, (int, float, np.integer, np.floating)):
            f = float(v)
            out[k] = str(int(f)) if f.is_integer() and abs(f) < 1e16 else repr(f)
        else:
            out[k] = ""
    return out


# ---------------------------------------------------------------------------------------------------
# AppendLog / TimeSeries
# ---------------------------------------------------------------------------------------------------

class AppendLog:
    """Writer side of append_log.rs: header, committed region, sparse tail."""

    def __init__(self, path: str, extra: bytes):
        if len(extra) != 8:
            raise ValueError("AppendLog extra must be 8 bytes (Timestamp / u64)")
        self.path = path
        self._f = open(path, "x+b", buffering=0)                               # create_new(true)
        self._f.seek(APPEND_LOG_FILE_SIZE)
        self._f.write(b"\0")                                      # append_log.rs:62-63: sparse 8 GiB + 1
        self._f.seek(0)
        self._f.write(struct.pack("<QQ", APPEND_LOG_HEADER, 0) + extra)
        self._end = APPEND_LOG_HEADER

    def write(self, buf: bytes) -> int:
        """AppendLog::write (:168-186): data first, then the committed length."""
        if self._end + len(buf) > APPEND_LOG_FILE_SIZE + 1:
            raise OverflowError("AppendLog map overflow")
        self._f.seek(self._end)
        self._f.write(buf)
        off = self._end - APPEND_LOG_HEADER
        self._end += len(buf)
        self._f.seek(0)
        self._f.write(struct.pack("<Q", self._end))
        return off

    def __len__(self) -> int:
        return self._end - APPEND_LOG_HEADER

    def close(self) -> None:
        if self._f:
            self._f.flush()
            os.fsync(self._f.fileno())
            self._f.close()
            self._f = None


class TimeTravel(ValueError):
    """Error::TimeTravel — a sample older than the last committed one (time_series.rs:205-222)."""


class TimeSeries:
    """time_series.rs:10-40: an index log of i64 µs timestamps and a data log of fixed-size rows."""

    def __init__(self, path: str, start_timestamp: int, element_size: int):
        os.makedirs(path, exist_ok=True)
        self.index = AppendLog(os.path.join(path, "index"), struct.pack("<q", start_timestamp))
        self.data = AppendLog(os.path.join(path, "data"), struct.pack("<Q", element_size))
        self.element_size = element_size
        self._last: Optional[int] = None

    def push_buf(self, timestamp: int, buf: bytes) -> None:
        if len(buf) != self.element_size:
            raise ValueError(f"sample of {len(buf)} bytes in a series of {self.element_size}-byte rows")
        if self._last is not None and self._last > timestamp:
            raise TimeTravel(f"time travel: {timestamp} after {self._last}")
        self.data.write(buf)                                      # data first, index last (consistent reads)
        self.index.write(struct.pack("<q", timestamp))
        self._last = timestamp

    def push_many(self, timestamps: np.ndarray, rows: np.ndarray) -> None:
        ts = np.ascontiguousarray(timestamps, dtype="<i8")
        rows = np.ascontiguousarray(rows)
        if len(ts) == 0:
            return
        if rows.nbytes != len(ts) * self.element_size:
            raise ValueError("rows do not match the element size")
        if (self._last is not None and self._last > int(ts[0])) or np.any(np.diff(ts) < 0):
            raise TimeTravel("time travel inside a batch of samples")
        self.data.write(rows.tobytes())
        self.index.write(ts.tobytes())
        self._last = int(ts[-1])

    def close(self) -> None:
        self.data.close()
        self.index.close()


# ---------------------------------------------------------------------------------------------------
# the sink
# ---------------------------------------------------------------------------------------------------

class DbSink:
    """Writes one elodin-db directory.  Use `insert_component` for each (entity, component) pair, then
    `commit` per telemetry sample — or `write_db(exec, path)` for a whole recorded run."""

    def __init__(self, path: str, start_timestamp_us: int, default_playback_speed: float = 1.0):
        if os.path.exists(os.path.join(path, "db_state")):
            raise FileExistsError(f"{path} already holds a database")
        os.makedirs(path, exist_ok=True)
        self.path = path
        self.start_timestamp = int(start_timestamp_us)
        self.config = DbConfig(False, duration_ns(default_playback_speed / 60.0),     # impeller2_server.rs:298-307
                               {"version.created": DB_VERSION, "version.last_opened": DB_VERSION,
                                "time.start_timestamp": str(self.start_timestamp)})
        self.series: Dict[int, TimeSeries] = {}
        self.meta: Dict[int, ComponentMetadata] = {}
        self._next_creation_index = 0
        self._save_state()

    def _save_state(self) -> None:
        with open(os.path.join(self.path, "db_state"), "wb") as f:
            f.write(self.config.encode())

    def _write_metadata(self, md: ComponentMetadata) -> None:
        d = os.path.join(self.path, str(md.component_id))
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "metadata"), "wb") as f:
            f.write(md.encode())
        self.meta[md.component_id] = md

    def set_entity_metadata(self, name: str, metadata: Optional[dict] = None) -> None:
        """impeller2_server.rs:285-294: one metadata-only directory per entity."""
        self._write_metadata(ComponentMetadata(component_id(name), name, _metadata_strings(metadata or {})))

    def insert_component(self, entity: str, component: str, schema: Schema, metadata: Optional[dict] = None) -> int:
        """init_db + State::insert_component (lib.rs:1216-1330): metadata, schema, empty time series."""
        name = f"{entity}.{component}"
        pid = component_id(name)
        if pid in self.series:
            raise ValueError(f"{name} registered twice")
        md = _metadata_strings(metadata or {})
        md[CREATION_INDEX_KEY] = str(self._next_creation_index)   # ensure_component_creation_index
        self._next_creation_index += 1
        self._write_metadata(ComponentMetadata(pid, name, md))
        d = os.path.join(self.path, str(pid))
        with open(os.path.join(d, "schema"), "wb") as f:
            f.write(schema.encode())
        # Component::create passes Timestamp(i64::MAX) as the index header's start (lib.rs:1322-1323)
        self.series[pid] = TimeSeries(d, (1 << 63) - 1, schema.size)
        return pid

    def commit(self, pid: int, timestamp_us: int, row: np.ndarray) -> None:
        self.series[pid].push_buf(int(timestamp_us), np.ascontiguousarray(row).tobytes())

    def commit_many(self, pid: int, timestamps_us: np.ndarray, rows: np.ndarray) -> None:
        self.series[pid].push_many(timestamps_us, rows)

    def close(self) -> None:
        for s in self.series.values():
            s.close()
        self._save_state()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def sample_timestamps(start_us: int, sim_time_step: float, sample_ticks) -> np.ndarray:
    """Timestamps of the recorded samples, as the reference stamps them (exec.rs:134-152, impeller2_server.rs:560-580,
    631-636): sample 0 is the initial state at `start`; a batch that ends after `tick` ticks in total is committed at
    `start + floor(dt_ns * (tick - 1) / 1000)` µs — whatever its length, so short tail batches (`this_batch` override,
    exec.rs:131-139) and repeated run() calls are stamped by the ticks they really covered.  `sample_ticks[k]` is the
    tick counter of recorded row k (Exec._globals_hist)."""
    dt_ns = duration_ns(sim_time_step)
    ticks = [int(t) for t in sample_ticks]
    out = np.empty(len(ticks), dtype=np.int64)
    for k, tick in enumerate(ticks):
        out[k] = start_us + (dt_ns * max(tick - 1, 0)) // 1000 if k else start_us
    return out


def history_slot(exec_, world: int, what: str) -> int:
    """The index of campaign world `world` on the world axis of `exec_._history` (rows are indexed h[slot, row]): the
    Exec's own mapping (world.Exec._history_slot: the world itself, or its slot among an ensemble Exec's retained
    worlds, refusing any other), else the world itself for an object that only carries `_history`."""
    slot = getattr(exec_, "_history_slot", None)
    return int(world) if slot is None else slot(world, what)


class LiveDbWriter:
    """The telemetry sink while a run is in flight: `init_db` once (every (entity, component) pair registered, row 0 =
    the initial state), then `flush()` appends the history rows recorded since the last flush — one
    `commit_world_head_unified` (impeller2_server.rs:390-438) per telemetry cycle.  `Exec.attach_db` calls flush after
    every recorded cycle on the invoke_batch route and after every ring read-back (<= ring capacity cycles, still one
    AppendLog row per cycle with that cycle's timestamp) on the device-resident route."""

    def __init__(self, exec_, path: str, start_timestamp_us: int = 1_767_225_600_000_000, world: int = 0):
        from .export import _entity_key

        self.exec_, self.world, self.start = exec_, int(world), int(start_timestamp_us)
        self._slot = history_slot(exec_, world, "attach_db() / write_db()")
        self.sink = DbSink(path, start_timestamp_us)
        self.rows_written = 0
        w = exec_.world
        self._globals = []
        for comp, md, prim in (("tick", {"priority": 7}, "u64"), ("simulation_time_step", {"priority": 8}, "f64")):
            self._globals.append((self.sink.insert_component("globals", comp, Schema(prim, ()), md), prim))
        self._pairs = []  # (pair id, column id, row, dtype)
        names = set()
        for cid, col in w.columns.items():
            comp = col.component
            prim = "u64" if np.dtype(col.dtype) == np.uint64 else "f64"
            if comp.ty is not None and comp.ty.width == col.width:
                shape = tuple(comp.ty.shape)                           # the declared ComponentType
            else:
                shape = () if col.width == 1 else (col.width,)
            for row, ent in enumerate(col.entity_ids):
                ename = w.entity_names.get(ent)
                if ename is None:
                    continue
                key = _entity_key(ename)
                names.add(key)
                pid = self.sink.insert_component(key, comp.name, Schema(prim, shape), comp.metadata)
                self._pairs.append((pid, cid, row, Schema(prim).dtype))
        self.sink.set_entity_metadata("globals")
        for key in sorted(names):
            self.sink.set_entity_metadata(key)
        self.flush()

    def flush(self) -> int:
        """Append every history row recorded since the last flush; returns how many."""
        ex = self.exec_
        g = ex._globals_hist
        i0, i1 = self.rows_written, len(g)
        if i1 <= i0:
            return 0
        # a row's timestamp depends on its own tick only (exec.rs:134-152), so a later flush stamps exactly what a
        # whole-run write would have
        ts = sample_timestamps(self.start, ex.sim_time_step, [x[0] for x in g[:i1]])[i0:]
        for (pid, prim), k in zip(self._globals, (0, 1)):
            self.sink.commit_many(pid, ts, np.asarray([x[k] for x in g[i0:i1]], dtype=Schema(prim).dtype))
        for pid, cid, row, dtype in self._pairs:
            rows = np.stack([h[self._slot, row] for h in ex._history[cid][i0:i1]]).astype(dtype, copy=False)
            self.sink.commit_many(pid, ts, rows)
        self.rows_written = i1
        return i1 - i0

    def close(self) -> DbSink:
        self.flush()
        self.sink.close()
        return self.sink


def write_db(exec_, path: str, start_timestamp_us: int = 1_767_225_600_000_000, world: int = 0) -> DbSink:
    """Write the recorded history of `exec_` (elodin_b200.world.Exec) for world `world` as an elodin-db
    directory: what `init_db` + one `commit_world_head_unified` per telemetry cycle leave on disk."""
    return LiveDbWriter(exec_, path, start_timestamp_us, world).close()


# ---------------------------------------------------------------------------------------------------
# reader (DB::open + TimeSeries), used by the tests and by export_db_csv
# ---------------------------------------------------------------------------------------------------

@dataclass
class StoredSeries:
    component_id: int
    name: str
    schema: Schema
    metadata: Dict[str, str]
    start_timestamp: int
    timestamps: np.ndarray
    values: np.ndarray


def _read_log(path: str) -> Tuple[bytes, bytes]:
    with open(path, "rb") as f:
        head = f.read(APPEND_LOG_HEADER)
        if len(head) != APPEND_LOG_HEADER:
            raise ValueError(f"{path}: short AppendLog header")
        committed, _head_len = struct.unpack_from("<QQ", head)
        if committed < APPEND_LOG_HEADER:
            raise ValueError(f"{path}: committed_len {committed} below the header size")
        body = f.read(committed - APPEND_LOG_HEADER)
        if len(body) != committed - APPEND_LOG_HEADER:
            raise ValueError(f"{path}: committed_len past the end of the file")
    return head[16:24], body


def read_db(path: str) -> Tuple[DbConfig, Dict[str, StoredSeries], Dict[int, ComponentMetadata]]:
    """Component scan of DB::open (lib.rs:592-670): numeric directories with a `schema` are components,
    `metadata` names them; returns (db_state, series by name, all metadata by id)."""
    state_path = os.path.join(path, "db_state")
    if not os.path.exists(state_path):
        raise FileNotFoundError(f"missing db_state: {state_path}")
    with open(state_path, "rb") as f:
        config = DbConfig.decode(f.read())
    series: Dict[str, StoredSeries] = {}
    metas: Dict[int, ComponentMetadata] = {}
    for entry in sorted(os.listdir(path)):
        d = os.path.join(path, entry)
        if not os.path.isdir(d) or entry in _SKIP_DIRS:
            continue
        try:
            cid = int(entry)
        except ValueError:
            raise ValueError(f"invalid component id directory {entry!r}")
        md = None
        if os.path.exists(os.path.join(d, "metadata")):
            with open(os.path.join(d, "metadata"), "rb") as f:
                md = ComponentMetadata.decode(f.read())
            metas[cid] = md
        if not os.path.exists(os.path.join(d, "schema")):
            continue
        with open(os.path.join(d, "schema"), "rb") as f:
            schema = Schema.decode(f.read())
        extra_i, index = _read_log(os.path.join(d, "index"))
        extra_d, data = _read_log(os.path.join(d, "data"))
        elem = struct.unpack("<Q", extra_d)[0]
        if elem != schema.size:
            raise ValueError(f"{entry}: element size {elem} does not match schema size {schema.size}")
        ts = np.frombuffer(index, dtype="<i8")
        if len(data) != len(ts) * elem:
            raise ValueError(f"{entry}: {len(ts)} timestamps for {len(data)} data bytes")
        vals = np.frombuffer(data, dtype=schema.dtype).reshape((len(ts),) + tuple(schema.shape))
        name = md.name if md else str(cid)
        start = struct.unpack("<q", extra_i)[0]
        if len(ts):
            start = min(start, int(ts[0]))                          # TimeSeries::start_timestamp
        series[name] = StoredSeries(cid, name, schema, md.metadata if md else {}, start, ts, vals)
    return config, series, metas


def _safe_name(name: str) -> str:
    from .export import _safe_file

    return _safe_file(name)


def export_db_csv(db_path: str, out_dir: str) -> List[str]:
    """`elodin-db export --format csv --flatten` over a directory written by `write_db`: one
    `<entity>.<component>.csv` per series, `time` + flattened element columns (export.py documents the
    naming; private components would be skipped — none are written here)."""
    import datetime as dt

    from .export import _fmt, _safe_file

    _, series, _ = read_db(db_path)
    os.makedirs(out_dir, exist_ok=True)
    written = []
    epoch = dt.datetime(1970, 1, 1)
    for name, s in sorted(series.items()):
        names = s.metadata.get("element_names")
        width = int(np.prod(s.schema.shape, dtype=np.int64)) if s.schema.shape else 1
        elems = names.split(",") if names else [str(i) for i in range(width)]
        header = [name] if (not s.schema.shape and not names) else [f"{name}_{e}" for e in elems]
        flat = s.values.reshape(len(s.timestamps), -1)
        p = os.path.join(out_dir, _safe_file(name) + ".csv")
        with open(p, "w", newline="") as f:
            f.write(",".join(["time"] + header) + "\n")
            for t, r in zip(s.timestamps, flat):
                f.write(",".join([(epoch + dt.timedelta(microseconds=int(t))).isoformat()] + [_fmt(x) for x in r]) + "\n")
        written.append(p)
    return written
