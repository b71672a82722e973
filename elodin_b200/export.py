"""CSV telemetry export in the layout of `elodin-db export --format csv --flatten`.

The reference's CI regression gate (scripts/ci/regress.sh) exports every (entity, component)
time series to `<entity>.<component>.csv` and diffs the directory against
scripts/ci/baseline/<example>-csv with scripts/ci/compare_baseline_csv.py (same file set, same
headers ignoring `time`, same row count, values within tolerances.json).  `export_csv` writes a
B200 run in that layout so the same gate — and anything else that consumes those exports —
works on GPU runs unchanged.

Naming (observed in scripts/ci/baseline/three-body-csv): entity names are lower-cased with
spaces -> "_" ("A -> B" -> "a_>_b"); columns are `<entity>.<component>` for scalars and
`<entity>.<component>_<element>` otherwise, with the component's `element_names` metadata
(python/elodin/__init__.py:594-625) or 0..n-1; file names are made Windows-safe exactly like
scripts/ci/windows_paths.py:21-22 ("_>_" -> "_to_", ">" -> "to").
"""

from __future__ import annotations

import datetime as _dt
import os
import re
from typing import List, Optional

import numpy as np



_WORD_SPLIT = re.compile(r"[ \-_]+")
_CASE_SPLIT = re.compile(r"(?<=[a-z])(?=[A-Z])|(?<=[A-Z])(?=[A-Z][a-z])")


def _entity_key(name: str) -> str:
    """Entity name -> id, as WorldBuilder derives it (libs/nox-py/src/world_builder.rs:281-285):
    `name.without_boundaries(digits).to_case(Case::Snake)` of the convert_case crate — words split
    at spaces / hyphens / underscores and lower->Upper or ACRONYMWord boundaries (not at digits),
    lower-cased and joined with "_".  "A -> B" -> "a_>_b", "fooBar" -> "foo_bar", "e1" -> "e1"."""
    words = []
    for tok in _WORD_SPLIT.split(name):
        words += [w for w in _CASE_SPLIT.split(tok) if w]
    return "_".join(w.lower() for w in words)


def _safe_file(name: str) -> str:
    return name.replace("_>_", "_to_").replace(">", "to")


def _fmt(v) -> str:
    if isinstance(v, (np.integer, int)):
        return str(int(v))
    return repr(float(v))


def export_csv(exec_, out_dir: str, start_timestamp: Optional[_dt.datetime] = None, world: int = 0) -> List[str]:
    """Write one CSV per (entity, component) of `exec_`'s recorded history (world `world`: the campaign's world index,
    a retained one for an ensemble Exec)."""
    from .db_sink import history_slot, sample_timestamps

    slot = history_slot(exec_, world, "export_csv()")
    os.makedirs(out_dir, exist_ok=True)
    w = exec_.world
    t0 = start_timestamp or _dt.datetime(2026, 1, 1)
    # the same time base as the elodin-db sink: row k is stamped by the ticks it really covers (exec.rs:134-152)
    us = sample_timestamps(0, exec_.sim_time_step, [g[0] for g in exec_._globals_hist])
    times = [(t0 + _dt.timedelta(microseconds=int(u))).isoformat() for u in us]
    written = []

    def write(stem: str, header: List[str], rows) -> None:
        path = os.path.join(out_dir, _safe_file(stem) + ".csv")
        with open(path, "w", newline="") as f:
            f.write(",".join(["time"] + header) + "\n")
            for t, r in zip(times, rows):
                f.write(",".join([t] + [_fmt(x) for x in np.atleast_1d(r)]) + "\n")
        written.append(path)

    write("globals.tick", ["globals.tick"], [g[0] for g in exec_._globals_hist])
    write("globals.simulation_time_step", ["globals.simulation_time_step"], [g[1] for g in exec_._globals_hist])
    for cid, col in w.columns.items():
        comp = col.component
        names = comp.metadata.get("element_names")
        elems = names.split(",") if names else [str(i) for i in range(col.width)]
        for row, ent in enumerate(col.entity_ids):
            ename = w.entity_names.get(ent)
            if ename is None:
                continue
            key = _entity_key(ename)
            base = f"{key}.{comp.name}"
            header = [base] if (col.width == 1 and not names) else [f"{base}_{e}" for e in elems]
            series = [h[slot, row] for h in exec_._history[cid]]
            write(base, header, series)
    return written
