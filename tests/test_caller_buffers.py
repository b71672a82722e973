"""invoke_batch, upload and download with device-resident caller buffers, and every entry on a caller-owned stream.

A caller that keeps its columns on the GPU (torch tensors, `data_ptr()`) hands b200_sixdof_invoke_batch device
pointers; plan_batch sees them with is_device_pointer and sends the call down the pipelined world ranges, with
device-to-device copies per range and pass-through outputs (Inertia, effector columns) copied on the copy-out stream.
A caller that runs the handle on its own stream (b200_sixdof_set_stream, as bench.py and RowShardedWorld do) expects
every entry to be ordered after the work it already queued there.  The contract these tests hold the library to:

  C1  Results do not depend on where the buffers live: the same batch with numpy host buffers, with every buffer on
      the device, with device inputs and host outputs, host inputs and device outputs, host and device alternating
      column by column, later calls whose pass-through inputs are device, host or NULL (not dirty), and the two
      globals (tick, simulation_time_step) as device tensors, gives the same bits.  EXACT equals the oracle bit for
      bit; FAST stays within the per-body bounds of tests.util.
  C2  On a caller stream, an entry reads its inputs after the caller's queued writes and writes its outputs after the
      caller's queued reads.  Each stream case delays the stream with torch.cuda._sleep and proves the delay was still
      running when the entry was called.
  C3  Entries that return data return with it complete: upload returns once a host source has been read.

The transport restatement (`transport`, `worlds_per_range`, `ranges`, `call_launches`) restates
b200_sixdof_invoke_batch's choice between the packed and the pipelined path, its world ranges and its layout
launches; tick launches come from tests.test_trajectory_routes.plan.  Every GPU call asserts the kernel_launches
delta the restatement predicts, so a device buffer cannot quietly take another path.
"""

import functools
import os

import numpy as np
import pytest

import elodin_b200 as el
from elodin_b200.executor import FORCE, INERTIA, WORLD_ACCEL, WORLD_POS, WORLD_VEL
from tests import test_nbody_routes as NR
from tests.test_egm08_field import tables as egm_tables
from tests.test_trajectory_routes import plan
from tests.util import assert_body_close, assert_nbody_close, body_effectors, body_scales, near_world, orbit_world

TICK, DT_ID = el.component_id("tick"), el.component_id("simulation_time_step")
STATE = (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)
GLOBALS = (TICK, DT_ID)
PAIR_MIN_BODIES = 2 * 128 * 3 * 132  # kPairMinBodies (body_kernels.cu): one full wave of body pairs on 132 SMs
PACKED_MAX_BODIES = (256 << 10) // (32 * 8)  # invoke_batch packs at most 1024 bodies
DEFAULT_CHUNK = 131072  # bodies per pipelined range without invoke_chunk_bodies (B200_CHUNK_BODIES unset)

# --------------------------------------------------------------------------- the transport, restated


def transport(n_bodies, n_inputs, chunk, device_buffers):
    """b200_sixdof_invoke_batch's `small` predicate: "packed" (one pinned block each way) or "pipelined"."""
    small = n_bodies > 0 and n_bodies * 32 * 8 <= (256 << 10) and n_inputs <= 16 and not chunk and not device_buffers
    return "packed" if small else "pipelined"


def worlds_per_range(M, N, chunk):
    """wpc: worlds per pipelined range (N = 1 rounds down to a multiple of 128 once it reaches 128)."""
    n = max(N, 1)
    w = max(1, (chunk or DEFAULT_CHUNK) // n)
    if n == 1 and w >= 128:
        w = w // 128 * 128
    if M * N == 0:
        w = max(M, 1)
    return w


def ranges(M, wpc):
    """[(first world, worlds)] of the pipelined ranges."""
    return [(w0, min(wpc, M - w0)) for w0 in range(0, M, wpc)]


def tick_launches(route, T, fused):
    """launch_ticks' kernel_launches for T ticks over one world range: "body" (one body launch per max_fused_ticks
    ticks), "small" (small_world_kernel, the same), "egm" (field + body per tick), "graph" (gravity + body per tick),
    "fused" (one n-body launch per tick)."""
    multi = route in ("body", "small")
    per_launch = 2 if route in ("egm", "graph") else 1
    return plan(dict(every=1, cap=0, fused=fused, steps=(T,)), multi, per_launch)[0][0]["delta"]


def call_launches(M, N, chunk, route, fused, T, uploads, downloads, null_pass, device_buffers, n_inputs):
    """kernel_launches of one invoke_batch call: per range one aos_to_soa per UPLOAD column, the ticks and one
    soa_to_aos per DOWNLOAD column (packed: one multi-column launch each way around the ticks of the whole batch),
    then one download per pass-through output whose input was NULL."""
    if transport(M * N, n_inputs, chunk, device_buffers) == "packed":
        return (uploads > 0) + tick_launches(route, T, fused) + (downloads > 0) + null_pass
    rs = ranges(M, worlds_per_range(M, N, chunk))
    return sum(uploads + tick_launches(route, T, fused) + downloads for _, nw in rs if nw * N) + null_pass


def input_is_live(cid, math, integ):
    """input_is_live: Force never crosses; WorldAccel only in EXACT RK4."""
    if cid == FORCE:
        return False
    if cid == WORLD_ACCEL:
        return math == "exact" and integ == "rk4"
    return True


def pass_through(cid):
    return cid not in STATE and cid not in GLOBALS


# --------------------------------------------------------------------------- the cases

BODY_SPEC = ("gravity", "thrust", "drag")


def _body(M, N, chunk=0, maths=("exact", "fast"), ticks=(2, 3), fused=2, every=0):
    return dict(fam="body", M=M, N=N, chunk=chunk, maths=maths, ticks=ticks, fused=fused, every=every, integ="rk4")


def _nbody(M, N, chunk, maths, ticks=(1, 2, 3), fused=1, integ="rk4"):
    return dict(fam="nbody", M=M, N=N, chunk=chunk, maths=maths, ticks=ticks, fused=fused, every=0, integ=integ)


CASES = {
    # packed with host buffers; device buffers force the pipeline (one range)
    "1x1": _body(1, 1),
    "1024x1": _body(1024, 1),
    "341x3": _body(341, 3),
    # pipelined with either
    "1025x1": _body(1025, 1),
    # N = 1: 200-body ranges round down to 128 worlds, ragged last range (300 = 128 + 128 + 44)
    "n1-rounding": _body(300, 1, chunk=200),
    # 77-world ranges of 3 bodies: ranges start at the odd bodies 231 and 462
    "odd-starts": _body(200, 3, chunk=77 * 3),
    # a range of 101 379 bodies (body pairs, a pair straddling two worlds) and a ragged tail of 3 003
    "pair": _body(33793 + 1001, 3, chunk=33793 * 3, maths=("fast",)),
    # the one-launch n-body tick (ping-pong planes) in >= 2 ranges, 1 + 2 + 3 ticks: nbody_tick_fused_kernel (N = 40,
    # a handle batch of 100 < 3 x 132 CTAs) and graph_dense_world_kernel with FUSE (N = 64, 130)
    "fused-40": _nbody(20, 40, 10 * 40, ("fast",)),
    "fused-64": _nbody(6, 64, 4 * 64, ("fast",)),
    "fused-130": _nbody(5, 130, 2 * 130, ("fast",)),
    # EXACT dense gravity + body kernel, two launches per tick
    "exact-dense-130": _nbody(3, 130, 2 * 130, ("exact",), ticks=(2, 1)),
    # small_world_kernel: 4 ticks per launch, 10-world ranges (41 = 4 x 10 + 1)
    "small-7": _nbody(41, 7, 10 * 7, ("exact", "fast"), ticks=(5, 3), fused=4),
    # every effector column kind as a device input and a pass-through output, EGM08 masked to some entities
    "effectors": dict(fam="effectors", M=40, N=5, chunk=0, maths=("exact", "fast"), ticks=(2, 1), fused=1, every=0,
                      integ="rk4"),
    # the trajectory ring over several calls: samples at ticks 3, 6, 9 of 2 + 4 + 3 ticks in 77-world ranges
    "ring": _body(170, 3, chunk=77 * 3, ticks=(2, 4, 3), every=3),
}
DT_SCALE = (1.0, 0.75, 1.0)  # simulation_time_step of call k, relative to the case's dt (changed between calls)


def route_of(case, math):
    if case["fam"] == "nbody":
        N = case["N"]
        if N <= 32:
            return "small"
        if math == "fast" and case["integ"] == "rk4":
            return "fused"
        return "graph"
    return "egm" if case["fam"] == "effectors" else "body"


CASE_KEYS = [(n, m) for n, c in CASES.items() for m in c["maths"]]  # (case, math mode)
CASE_IDS = [f"{n}-{m}" for n, m in CASE_KEYS]


@functools.lru_cache(maxsize=4)
def world(name):
    """(start = (pos, vel, ine), oracle-side spec or None, library effectors, {column name: array}, dt, S or None)."""
    c = CASES[name]
    M, N = c["M"], c["N"]
    if c["fam"] == "nbody":
        (pos, vel, ine, S), _, ge, cols = NR._setup(None, M, N, False)
        return (pos, vel, ine), None, ge, cols, NR.DT, S
    if c["fam"] == "body":
        pos, vel, ine, cc, dt = near_world(11 * M + N, M, N)
        spec = [("gravity", {}), ("thrust", {"thrust": cc["thrust"]}), ("drag", {"wind": cc["wind"]})]
    else:
        pos, vel, ine, cc, dt = orbit_world(17, M, N)
        rng = np.random.default_rng(18)
        m = ine[..., 6:7]
        cb, sb = egm_tables(8, "kaula")
        mask = np.array([1, 0, 1, 1, 0], dtype=np.uint8)
        # the wheel fold overwrites what the effectors before it accumulated: first, so that every column acts
        spec = [("wheels", {"torques": cc["wheels"]}), ("thrust", {"thrust": rng.uniform(2.0, 20.0, (M, N, 1)) * m}),
                ("wrench", {"wrench": cc["wrench"]}), ("egm08", {"c_bar": cb, "s_bar": sb, "L": 8, "mask": mask})]
    _, ge, cols = body_effectors(None, spec)
    return (pos, vel, ine), spec, ge, cols, dt, None


def _oracle_effs(O, name, spec):
    if spec is None:
        return NR._setup(O, CASES[name]["M"], CASES[name]["N"], False)[1]
    return body_effectors(O, spec)[0]


@functools.lru_cache(maxsize=2)
def oracle_run(name):
    """The oracle's (pos, vel, accel, force) after every tick of the case's calls (index 0: the start)."""
    from oracle import oracle as O

    O.build()
    O.set_dot_mode(0)
    c = CASES[name]
    start, spec, _, _, dt, _ = world(name)
    w = O.World(*start)
    oe = _oracle_effs(O, name, spec)
    z = np.zeros(start[0].shape[:2] + (6,))
    out = [(start[0], start[1], z, z)]
    threads = max(1, min(O.max_threads(), os.cpu_count() or 1))
    for k, T in enumerate(c["ticks"]):
        for _ in range(T):
            (w.rk4 if c["integ"] == "rk4" else w.semi_implicit)(dt * DT_SCALE[k], 1, oe, threads=threads)
            out.append(tuple(a.copy() for a in (w.pos, w.vel, w.accel, w.force)))
    return out


# --------------------------------------------------------------------------- buffer placements

PLACEMENTS = ("device", "device_in", "device_out", "alternating", "later_mixed", "globals_device")


def kinds(placement, ids, is_input, k):
    """Where each buffer of call k lives: "h" (numpy), "d" (torch CUDA tensor) or None (NULL).  Call 0 hands over
    every input; later calls hand over simulation_time_step (changed) and, in "later_mixed", the pass-through
    inputs as device, host and NULL in turn; the other inputs are not dirty.  Every output is read."""
    out = []
    n_pass = 0
    for j, cid in enumerate(ids):
        present = not is_input or k == 0 or cid == DT_ID
        kind = "h"
        if placement in ("device", "globals_device", "later_mixed"):
            kind = "d"
        elif placement == "device_in":
            kind = "d" if is_input else "h"
        elif placement == "device_out":
            kind = "h" if is_input else "d"
        elif placement == "alternating":
            kind = "d" if (j + (0 if is_input else 1)) % 2 == 0 else "h"
        if is_input and k > 0 and placement == "later_mixed" and pass_through(cid):
            present, kind = True, ("d", "h", None)[n_pass % 3]
            n_pass += 1
        if cid in GLOBALS and placement != "globals_device":
            kind = "h"
        out.append(kind if present and kind else None)
    return out


def _table(name, dt, tick):
    start, _, _, cols, _, _ = world(name)
    pos, vel, ine = start
    M, N = pos.shape[:2]
    t = {TICK: np.array([tick], dtype=np.uint64), DT_ID: np.array([dt]), WORLD_POS: pos, WORLD_VEL: vel,
         INERTIA: ine, WORLD_ACCEL: np.zeros((M, N, 6)), FORCE: np.zeros((M, N, 6))}
    t.update({el.component_id(n): a for n, a in cols.items()})
    return t


def _open(name, math):
    c = CASES[name]
    start, _, ge, _, dt, _ = world(name)
    kw = dict(max_fused_ticks=c["fused"], invoke_chunk_bodies=c["chunk"])
    if c["every"]:
        kw.update(trajectory_every=c["every"], trajectory_capacity=8)
    return el.B200Exec(c["N"], c["M"], dt, None, ge, c["integ"], math, **kw)


def _device(a):
    import torch

    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else a).to("cuda")


def _host_of(buf, shape, dtype):
    if isinstance(buf, np.ndarray):
        return buf.copy()
    a = buf.cpu().numpy()
    return (a.view(np.uint64) if dtype == np.uint64 else a).reshape(shape)


def run_case(name, math, placement):
    """One handle, the case's calls with `placement` ("host" = numpy everywhere).  Returns per call {cid: output},
    the kernel_launches deltas and the deltas the restatement predicts, and the ring after the last call."""
    import torch

    c = CASES[name]
    dt = world(name)[4]
    res = {"outs": [], "delta": [], "want": [], "paths": []}
    with _open(name, math) as ex:
        tick = 0
        for k, T in enumerate(c["ticks"]):
            table = _table(name, dt * DT_SCALE[k], tick)
            ik = ["h"] * len(ex.input_ids) if placement == "host" else kinds(placement, ex.input_ids, True, k)
            ok = ["h"] * len(ex.output_ids) if placement == "host" else kinds(placement, ex.output_ids, False, k)
            if placement == "host" and k > 0:
                ik = [("h" if cid == DT_ID else None) for cid in ex.input_ids]
            ins, outs = [], []
            for cid, kd in zip(ex.input_ids, ik):
                ins.append(None if kd is None else np.ascontiguousarray(table[cid]) if kd == "h" else _device(table[cid]))
            for cid, kd in zip(ex.output_ids, ok):
                dtype = np.uint64 if cid == TICK else np.float64
                shape = ex.column_shape(cid)
                if kd == "h":
                    outs.append(np.full(shape, np.nan) if dtype == np.float64 else np.zeros(shape, dtype))
                else:
                    outs.append(torch.full(shape, float("nan"), dtype=torch.float64, device="cuda") if dtype == np.float64
                                else torch.zeros(shape, dtype=torch.int64, device="cuda"))
            torch.cuda.synchronize()  # the device inputs are written (their copies ran on torch's stream)
            ptr = lambda b: None if b is None else b.ctypes.data if isinstance(b, np.ndarray) else b.data_ptr()
            n0 = ex.timings()["kernel_launches"]
            ex.invoke_batch_ptrs([ptr(b) for b in ins], [ptr(b) for b in outs], T)
            res["delta"].append(ex.timings()["kernel_launches"] - n0)
            dev = any(kd == "d" for cid, kd in zip(ex.input_ids, ik) if cid not in GLOBALS) or \
                any(kd == "d" for cid, kd in zip(ex.output_ids, ok) if cid not in GLOBALS)
            ups = sum(1 for cid, kd in zip(ex.input_ids, ik) if kd and cid not in GLOBALS and input_is_live(cid, math, c["integ"]))
            downs = sum(1 for cid, kd in zip(ex.output_ids, ok) if kd and cid in STATE)
            given = {cid for cid, kd in zip(ex.input_ids, ik) if kd}
            null_pass = sum(1 for cid, kd in zip(ex.output_ids, ok) if kd and pass_through(cid) and cid not in given)
            res["want"].append(call_launches(c["M"], c["N"], c["chunk"], route_of(c, math), c["fused"], T, ups, downs,
                                             null_pass, dev, len(ex.input_ids)))
            res["paths"].append(transport(c["M"] * c["N"], len(ex.input_ids), c["chunk"], dev))
            res["outs"].append({cid: _host_of(b, ex.column_shape(cid), np.uint64 if cid == TICK else np.float64)
                                for cid, b in zip(ex.output_ids, outs)})
            tick += T
        res["ring"] = ex.trajectory() if c["every"] else None
        res["pass_ids"] = [cid for cid in ex.output_ids if pass_through(cid)]
    return res


# --------------------------------------------------------------------------- CPU: the restatement


def test_restatement_on_hand_worked_cases():
    """The transport, range and launch restatement on cases worked by hand from b200_sixdof_invoke_batch."""
    # the packed path: at most 1024 bodies, 16 inputs, no invoke_chunk_bodies, no device buffer
    assert transport(1, 7, 0, False) == "packed" and transport(1, 7, 0, True) == "pipelined"
    assert transport(1024, 7, 0, False) == "packed" and transport(1025, 7, 0, False) == "pipelined"
    assert transport(1023, 16, 0, False) == "packed" and transport(1023, 17, 0, False) == "pipelined"
    assert transport(4, 7, 4, False) == "pipelined" and transport(0, 7, 0, False) == "pipelined"
    # wpc: N = 1 rounds to a multiple of 128 once it reaches 128; other N do not round
    assert worlds_per_range(300, 1, 200) == 128 and worlds_per_range(300, 1, 127) == 127
    assert worlds_per_range(300, 1, 0) == 131072 and worlds_per_range(300, 1, 255) == 128
    assert worlds_per_range(200, 3, 231) == 77 and worlds_per_range(200, 3, 2) == 1
    assert worlds_per_range(7, 0, 5) == 7  # no bodies: one range of every world
    assert ranges(300, 128) == [(0, 128), (128, 128), (256, 44)]
    assert ranges(200, 77) == [(0, 77), (77, 77), (154, 46)]
    assert ranges(5, 2) == [(0, 2), (2, 2), (4, 1)]
    # tick launches: body / small-world launches fuse max_fused_ticks ticks, the others run one tick per launch
    assert [tick_launches("body", T, 2) for T in (1, 2, 3, 5)] == [1, 1, 2, 3]
    assert [tick_launches("small", T, 4) for T in (3, 5)] == [1, 2]
    assert [tick_launches(r, 3, 4) for r in ("egm", "graph", "fused")] == [6, 6, 3]
    # FAST free bodies, 1025 x 1, 2 ticks: uploads pos, vel, inertia (WorldAccel and Force are dead), downloads
    # the 4 state columns, Inertia passed through from its input
    assert call_launches(1025, 1, 0, "body", 1, 2, 3, 4, 0, False, 7) == 3 + 2 + 4
    # the same with 200-body ranges (3 ranges) and Inertia not dirty (one download after the ranges)
    assert call_launches(300, 1, 200, "body", 1, 2, 3, 4, 1, False, 7) == 3 * 9 + 1
    # packed: one layout launch each way around the ticks of the whole batch
    assert call_launches(341, 3, 0, "body", 2, 3, 4, 4, 0, False, 9) == 1 + 2 + 1
    assert call_launches(341, 3, 0, "body", 2, 3, 4, 4, 0, True, 9) == 4 + 2 + 4
    # a later call with every input NULL: no upload launch
    assert call_launches(341, 3, 0, "body", 2, 3, 0, 4, 2, False, 9) == 0 + 2 + 1 + 2
    # the one-launch n-body tick over 2 + 2 + 1 worlds, 3 ticks
    assert call_launches(5, 130, 260, "fused", 1, 3, 3, 4, 0, True, 7) == 3 * (3 + 3 + 4)
    # the restated input_is_live
    assert [input_is_live(c, "exact", "rk4") for c in (FORCE, WORLD_ACCEL, WORLD_POS)] == [False, True, True]
    assert [input_is_live(WORLD_ACCEL, m, i) for m, i in (("fast", "rk4"), ("exact", "semi_implicit"))] == [False, False]


def test_placements_cover_every_buffer_mix():
    """Each placement gives the buffer mix it is named for, and later calls hand over what the protocol says."""
    ins = [TICK, DT_ID, WORLD_POS, WORLD_VEL, INERTIA, WORLD_ACCEL, FORCE, 77, 78, 79]
    outs = [TICK, DT_ID, WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE, INERTIA, 77, 78, 79]
    non_global = lambda ids, ks: [k for c, k in zip(ids, ks) if c not in GLOBALS]
    assert set(non_global(ins, kinds("device", ins, True, 0))) == {"d"}
    assert set(non_global(outs, kinds("device_in", outs, False, 0))) == {"h"}
    assert set(non_global(ins, kinds("device_out", ins, True, 0))) == {"h"}
    alt = non_global(ins, kinds("alternating", ins, True, 0)) + non_global(outs, kinds("alternating", outs, False, 0))
    assert {"d", "h"} <= set(alt) and all(a != b for a, b in zip(alt[:8], alt[1:8]))
    later = dict(zip(ins, kinds("later_mixed", ins, True, 1)))
    assert [later[c] for c in (INERTIA, 77, 78, 79)] == ["d", "h", None, "d"]
    assert [later[c] for c in (TICK, WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE)] == [None] * 5 and later[DT_ID] == "h"
    assert kinds("globals_device", ins, True, 0)[:2] == ["d", "d"] and kinds("device", ins, True, 0)[:2] == ["h", "h"]
    assert kinds("globals_device", ins, True, 1)[:2] == [None, "d"]


def test_gpu_cases_reach_every_boundary():
    """The GPU case list reaches every transport boundary the device buffers change."""
    geo = {n: (c["M"], c["N"], c["chunk"]) for n, c in CASES.items()}

    def path(n, dev):
        M, N, chunk = geo[n]
        return transport(M * N, 9, chunk, dev)

    # would be packed with host buffers; device buffers force the pipeline, one range
    for n in ("1x1", "1024x1", "341x3"):
        M, N, chunk = geo[n]
        assert path(n, False) == "packed" and path(n, True) == "pipelined", n
        assert len(ranges(M, worlds_per_range(M, N, chunk))) == 1, n
    assert geo["1024x1"][0] * geo["1024x1"][1] == PACKED_MAX_BODIES and geo["341x3"][0] * 3 == PACKED_MAX_BODIES - 1
    assert path("1025x1", False) == "pipelined" and geo["1025x1"][0] == PACKED_MAX_BODIES + 1
    # N = 1 rounding to 128-world ranges, ragged last
    M, N, chunk = geo["n1-rounding"]
    rs = ranges(M, worlds_per_range(M, N, chunk))
    assert N == 1 and chunk // N != 128 and all(nw == 128 for _, nw in rs[:-1]) and 0 < rs[-1][1] < 128 and len(rs) >= 3
    # ranges that start at odd bodies
    M, N, chunk = geo["odd-starts"]
    assert any((w0 * N) % 2 == 1 for w0, _ in ranges(M, worlds_per_range(M, N, chunk)))
    # a range past kPairMinBodies and a ragged tail below it
    M, N, chunk = geo["pair"]
    rs = ranges(M, worlds_per_range(M, N, chunk))
    assert rs[0][1] * N >= PAIR_MIN_BODIES and 0 < rs[-1][1] < rs[0][1] and len(rs) == 2
    assert "fast" in CASES["pair"]["maths"]
    # the fused n-body routes: nbody_tick_fused_kernel below 64 bodies on a batch below 3 x 132 CTAs, the world
    # kernel with FUSE at 64 and 130 bodies, each in >= 2 ranges, with odd and even tick counts
    for n, lo, hi in (("fused-40", 33, 63), ("fused-64", 64, 1024), ("fused-130", 64, 1024)):
        M, N, chunk = geo[n]
        assert lo <= N <= hi and route_of(CASES[n], "fast") == "fused", n
        assert len(ranges(M, worlds_per_range(M, N, chunk))) >= 2, n
        assert sorted(CASES[n]["ticks"]) == [1, 2, 3], n
    M, N, _ = geo["fused-40"]
    assert -(-N // 8) * M < 3 * 132
    assert {N for N in (geo["fused-64"][1], geo["fused-130"][1])} == {64, 130}
    # other graph routes: EXACT dense 130 bodies (two launches per tick), small world 7 bodies, both in >= 2 ranges
    assert CASES["exact-dense-130"]["maths"] == ("exact",) and route_of(CASES["exact-dense-130"], "exact") == "graph"
    assert geo["exact-dense-130"][1] == 130 and route_of(CASES["small-7"], "fast") == "small" and geo["small-7"][1] == 7
    for n in ("exact-dense-130", "small-7"):
        M, N, chunk = geo[n]
        assert len(ranges(M, worlds_per_range(M, N, chunk))) >= 2, n
    # effector columns: thrust and wind (every body case), wrench, 3 wheels and EGM08 with an entity mask
    assert BODY_SPEC == tuple(k for k, _ in world("1x1")[1])
    spec = world("effectors")[1]
    assert [k for k, _ in spec] == ["wheels", "thrust", "wrench", "egm08"]
    assert spec[0][1]["torques"].shape[-1] == 9 and 0 < int(np.sum(spec[3][1]["mask"])) < CASES["effectors"]["N"]
    # the ring over several calls, sampling inside and at the end of calls
    c = CASES["ring"]
    ends = np.cumsum(c["ticks"])
    samples = range(c["every"], int(ends[-1]) + 1, c["every"])
    assert c["every"] == 3 and len(c["ticks"]) >= 3
    assert any(s not in ends for s in samples) and any(s in ends for s in samples)
    # simulation_time_step changes between calls, and every case makes a later call
    assert len(set(DT_SCALE)) > 1 and all(len(c["ticks"]) >= 2 for c in CASES.values())


# --------------------------------------------------------------------------- GPU: device buffers on every transport


@functools.lru_cache(maxsize=2)
def host_run(name, math):
    return run_case(name, math, "host")


def _state_of(outs):
    return tuple(outs[c] for c in STATE)


@pytest.mark.gpu
@pytest.mark.parametrize("key", CASE_KEYS, ids=CASE_IDS)
def test_host_buffers_match_the_oracle(oracle, key):
    """The reference run (numpy host buffers) after every call: EXACT equals the oracle bit for bit, FAST is within
    the per-body bounds; the tick column counts the ticks; pass-through outputs equal their inputs."""
    name, math = key
    c = CASES[name]
    res = host_run(name, math)
    want = oracle_run(name)
    start, spec, _, _, dt, S = world(name)
    assert res["delta"] == res["want"], f"{name} {math}: kernel_launches {res['delta']}, restated {res['want']}"
    table = _table(name, dt, 0)
    t = 0
    for k, T in enumerate(c["ticks"]):
        t += T
        got, ref = _state_of(res["outs"][k]), want[t]
        what = f"{name} {math} call {k} (tick {t})"
        assert int(res["outs"][k][TICK][0]) == t, what
        assert res["outs"][k][DT_ID][0] == dt * DT_SCALE[k], what
        for cid in res["pass_ids"]:
            assert np.array_equal(res["outs"][k][cid], table[cid]), f"{what}: pass-through {cid:#x}"
        if math == "exact":
            for q, a, b in zip(("pos", "vel", "accel", "force"), got, ref):
                assert np.array_equal(a, b), f"{what} {q}: max abs diff {np.max(np.abs(a - b))}"
        elif S is not None:
            assert_nbody_close(got, ref, start, dt, t, S, what=what)
        else:
            assert_body_close(got, ref, start, dt, t, body_scales(spec, *start), what=what)
    if c["every"]:
        ring = res["ring"]
        ticks = list(range(c["every"], t + 1, c["every"]))
        assert ring.shape[0] == len(ticks), name
        for s, tt in enumerate(ticks):
            ref = np.concatenate([want[tt][0], want[tt][1]], -1)
            if math == "exact":
                assert np.array_equal(ring[s, ..., :13], ref), f"{name} exact ring sample {s} (tick {tt})"
        last = np.concatenate(_state_of(res["outs"][-1])[:2], -1)
        assert np.array_equal(ring[-1, ..., :13], last), f"{name} {math}: last sample != the state the call returned"


@pytest.mark.gpu
@pytest.mark.parametrize("placement", PLACEMENTS)
@pytest.mark.parametrize("key", CASE_KEYS, ids=CASE_IDS)
def test_device_buffers_give_the_host_bits(key, placement):
    """The same calls with the buffers on the device (or mixed): every output of every call, and the ring, equal the
    host-buffer run bit for bit, on the path and with the launches the restatement predicts."""
    name, math = key
    ref = host_run(name, math)
    got = run_case(name, math, placement)
    what = f"{name} {math} {placement}"
    assert got["paths"][0] == "pipelined", what
    assert got["delta"] == got["want"], f"{what}: kernel_launches {got['delta']}, restated {got['want']}"
    for k, (a, b) in enumerate(zip(got["outs"], ref["outs"])):
        for cid in b:
            assert a[cid].dtype == b[cid].dtype and np.array_equal(a[cid], b[cid], equal_nan=True), \
                f"{what} call {k}: column {cid:#x} differs from the host-buffer run"
    if ref["ring"] is not None:
        assert np.array_equal(got["ring"], ref["ring"]), f"{what}: ring differs from the host-buffer run"


# --------------------------------------------------------------------------- GPU: caller-owned streams

DELAY_S = 0.2  # how long each case holds its stream back (bounded: at most about 0.3 s)
STREAMS = ("side", "legacy")
SM, SN = 3000, 1  # the stream cases' batch: pipelined either way (3000 bodies)


@pytest.fixture(scope="module")
def sleep_cycles():
    """torch.cuda._sleep cycles for DELAY_S, from a timed 20M-cycle sleep on this device."""
    import torch

    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    torch.cuda._sleep(20_000_000)
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b)
    assert ms > 0.0
    cycles = int(20_000_000 * DELAY_S * 1e3 / ms)
    return min(cycles, int(20_000_000 * 0.3e3 / ms))


def _stream(kind):
    import torch

    return torch.cuda.Stream() if kind == "side" else torch.cuda.default_stream()


def _delayed(S, cycles, work):
    """On S: sleep, then `work()` (the caller's queued write or read); returns an event recorded after them, which
    must still be pending when the entry is called."""
    import torch

    with torch.cuda.stream(S):
        torch.cuda._sleep(cycles)
        out = work()
        ev = torch.cuda.Event()
        ev.record(S)
    return ev, out


def _pending(ev, what):
    assert not ev.query(), f"{what}: the delayed stream work had finished before the entry was called: the case proves nothing"


def _stream_world(seed=5):
    pos, vel, ine, cc, dt = near_world(seed, SM, SN)
    spec = [("gravity", {}), ("thrust", {"thrust": cc["thrust"]}), ("drag", {"wind": cc["wind"]})]
    _, ge, cols = body_effectors(None, spec)
    return (pos, vel, ine), ge, cols, dt


def _stream_exec(traj=False):
    start, ge, cols, dt = _stream_world()
    kw = dict(trajectory_every=1, trajectory_capacity=4, trajectory_full=True) if traj else {}
    return el.B200Exec(SN, SM, dt, None, ge, "rk4", "fast", max_fused_ticks=2, **kw), start, cols, dt


def _full_table(ex, start, cols, dt, tick=0):
    pos, vel, ine = start
    t = {TICK: np.array([tick], dtype=np.uint64), DT_ID: np.array([dt]), WORLD_POS: pos, WORLD_VEL: vel,
         INERTIA: ine, WORLD_ACCEL: np.zeros((SM, SN, 6)), FORCE: np.zeros((SM, SN, 6))}
    t.update({el.component_id(n): a for n, a in cols.items()})
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAMS)
def test_upload_from_a_device_source_after_a_queued_write(kind, sleep_cycles):
    """upload reads a device source after the caller's write queued on its stream."""
    import torch

    S = _stream(kind)
    ex, start, cols, dt = _stream_exec()
    with ex:
        ex.set_stream(S.cuda_stream)
        ex.set_state(*start, **cols)
        new = start[0] + 1.0
        src = _device(start[0])
        newd = _device(new)
        torch.cuda.synchronize()
        ev, _ = _delayed(S, sleep_cycles, lambda: src.copy_(newd))
        _pending(ev, f"upload device source ({kind})")
        ex.upload_ptr(WORLD_POS, src.data_ptr(), src.numel() * 8)
        got = ex.download(WORLD_POS)
        torch.cuda.synchronize()
    assert np.array_equal(got, new), f"{kind}: upload read the device source before the caller's queued write"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAMS)
def test_upload_from_pinned_memory_returns_after_reading_it(kind, sleep_cycles):
    """upload from pinned host memory returns only once the source has been read: a caller may overwrite it
    right after the call, while the handle's stream is still busy."""
    import torch

    S = _stream(kind)
    ex, start, cols, dt = _stream_exec()
    src = el.pinned_empty(start[0].shape)
    try:
        with ex:
            ex.set_stream(S.cuda_stream)
            ex.set_state(*start, **cols)
            src[...] = start[0] + 1.0
            ev, _ = _delayed(S, sleep_cycles, lambda: None)
            _pending(ev, f"upload pinned source ({kind})")
            ex.upload_ptr(WORLD_POS, src.ctypes.data, src.nbytes)
            src[...] = -7.0  # the caller reuses its buffer
            torch.cuda.synchronize()
            got = ex.download(WORLD_POS)
    finally:
        el.pinned_free(src)
    assert np.array_equal(got, start[0] + 1.0), f"{kind}: upload returned before it had read the pinned source"


def _invoke_reference(table, n_ticks):
    """The undelayed run: a fresh handle, numpy host buffers, one call."""
    ex, _, _, _ = _stream_exec()
    with ex:
        out = ex.invoke_batch([table[c] for c in ex.input_ids], n_ticks)
        return dict(zip(ex.output_ids, out))


def _stream_buffers(ex, table, fill):
    """invoke_batch buffers of the stream cases: every column a torch CUDA tensor (outputs filled with `fill`),
    except the two globals, numpy scalars (their device form is a placement of test_device_buffers_give_the_host_bits).
    Returns (inputs, outputs, pointer of a buffer)."""
    import torch

    ins = [np.ascontiguousarray(table[c]) if c in GLOBALS else _device(table[c]) for c in ex.input_ids]
    outs = [np.zeros(1, np.uint64) if c == TICK else np.zeros(1) if c == DT_ID else
            torch.full(ex.column_shape(c), fill, dtype=torch.float64, device="cuda") for c in ex.output_ids]
    return ins, outs, lambda b: b.ctypes.data if isinstance(b, np.ndarray) else b.data_ptr()


def _host(b):
    return b.copy() if isinstance(b, np.ndarray) else b.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAMS)
def test_invoke_batch_reads_inputs_after_queued_writes(kind, sleep_cycles):
    """invoke_batch with device inputs and device outputs on a caller stream: every input, including those whose
    output is a pass-through copy (Inertia, thrust, wind), is read after the caller's queued writes."""
    import torch

    S = _stream(kind)
    ex, start, cols, dt = _stream_exec()
    old = _full_table(ex, start, cols, dt)
    rng = np.random.default_rng(3)
    new = {c: (a.copy() if c in GLOBALS else a * rng.uniform(0.5, 1.5, a.shape)) for c, a in old.items()}
    new[WORLD_POS] = old[WORLD_POS].copy()
    new[WORLD_POS][..., 4:] += rng.normal(0, 10, (SM, SN, 3))  # the attitude stays a unit quaternion
    want = _invoke_reference(new, 3)
    with ex:
        ex.set_stream(S.cuda_stream)
        ins, outs, ptr = _stream_buffers(ex, old, 0.0)
        upd = [(a, _device(new[c])) for c, a in zip(ex.input_ids, ins) if c not in GLOBALS]
        torch.cuda.synchronize()
        ev, _ = _delayed(S, sleep_cycles, lambda: [a.copy_(b) for a, b in upd])
        _pending(ev, f"invoke_batch read-after-write ({kind})")
        ex.invoke_batch_ptrs([ptr(b) for b in ins], [ptr(b) for b in outs], 3)
        got = {c: _host(b) for c, b in zip(ex.output_ids, outs)}
    for c, b in want.items():
        assert np.array_equal(got[c], b), f"{kind}: output {c:#x} differs from the undelayed run (an input read too early)"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAMS)
def test_invoke_batch_writes_outputs_after_queued_reads(kind, sleep_cycles):
    """invoke_batch on a caller stream writes no output (pass-through copies included) before the caller's queued
    reads of it: a snapshot queued before the call sees the old contents, the call returns the new ones."""
    import torch

    S = _stream(kind)
    ex, start, cols, dt = _stream_exec()
    table = _full_table(ex, start, cols, dt)
    want = _invoke_reference(table, 2)
    with ex:
        ex.set_stream(S.cuda_stream)
        ins, outs, ptr = _stream_buffers(ex, table, -3.0)
        dev = [(c, b) for c, b in zip(ex.output_ids, outs) if c not in GLOBALS]
        torch.cuda.synchronize()
        ev, snaps = _delayed(S, sleep_cycles, lambda: [b.clone() for _, b in dev])
        _pending(ev, f"invoke_batch write-after-read ({kind})")
        ex.invoke_batch_ptrs([ptr(b) for b in ins], [ptr(b) for b in outs], 2)
        got = {c: _host(b) for c, b in zip(ex.output_ids, outs)}
        torch.cuda.synchronize()
        snap = {c: t.cpu().numpy() for (c, _), t in zip(dev, snaps)}
    for c in ex.output_ids:
        assert c not in snap or np.all(snap[c] == -3.0), f"{kind}: output {c:#x} was written before the caller's queued read of it"
        assert np.array_equal(got[c], want[c]), f"{kind}: output {c:#x} differs from the undelayed run"


def _plane(ex, cid, k):
    import torch

    class _P:
        __cuda_array_interface__ = {"shape": (ex.plane_stride,), "typestr": "<f8", "data": (ex.device_plane(cid, k), False),
                                    "version": 3}

    return torch.as_tensor(_P(), device="cuda")[:SM * SN]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAMS)
def test_step_is_ordered_with_caller_work_on_its_stream(kind, sleep_cycles):
    """step() on a caller stream runs after a plane write queued there, and caller work queued after it reads the
    new state through device_plane with no sync in between."""
    import torch

    S = _stream(kind)
    ex, start, cols, dt = _stream_exec()
    vx = np.random.default_rng(4).normal(0, 10, SM * SN)
    ref_vel = start[1].copy()
    ref_vel[..., 3] = vx.reshape(SM, SN)
    ref, _, _, _ = _stream_exec()
    with ref:
        ref.set_state(start[0], ref_vel, start[2], **cols)
        ref.step(3, sync=True)
        want = ref.download(WORLD_POS)[..., 4].ravel()
    with ex:
        ex.set_stream(S.cuda_stream)
        ex.set_state(*start, **cols)
        vplane, xplane, vxd = _plane(ex, WORLD_VEL, 3), _plane(ex, WORLD_POS, 4), _device(vx)
        torch.cuda.synchronize()
        ev, _ = _delayed(S, sleep_cycles, lambda: vplane.copy_(vxd))
        _pending(ev, f"step ({kind})")
        ex.step(3)
        with torch.cuda.stream(S):
            snap = xplane.clone()
        torch.cuda.synchronize()
        got = snap.cpu().numpy()
    assert np.array_equal(got, want), f"{kind}: the state read on the caller's stream after step() is not step()'s result"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAMS)
def test_device_destinations_written_after_queued_reads(kind, sleep_cycles):
    """download, trajectory_download, state_stats and state_download_worlds into device destinations on a caller
    stream: a read of the destination queued before the call sees the old contents, and the call leaves what the
    host-destination entry returns."""
    import torch

    from elodin_b200 import _lib

    S = _stream(kind)
    ex, start, cols, dt = _stream_exec(traj=True)
    worlds = np.array([SM - 1, 0, 17, 17])
    with ex:
        ex.set_state(*start, **cols)
        ex.step(3, sync=True)
        ex.set_stream(S.cuda_stream)
        stats_shape = ex._rows(ring=False) + (_lib.STATS_FIELDS,)
        entries = {
            "download": (lambda p, n: ex.download_ptr(WORLD_VEL, p, n), ex.download(WORLD_VEL)),
            "trajectory_download": (ex.trajectory_to_ptr, ex.trajectory()),
            "state_stats": (lambda p, n: ex._reduce("stats", False, (), stats_shape, p, n), ex.state_stats()),
            "state_download_worlds": (lambda p, n: ex.state_worlds(worlds, p, n), ex.state_worlds(worlds)),
        }
        for name, (call, want) in entries.items():
            dst = torch.full(want.shape, -5.0, dtype=torch.float64, device="cuda")
            torch.cuda.synchronize()
            ev, snap = _delayed(S, sleep_cycles, lambda: dst.clone())
            _pending(ev, f"{name} ({kind})")
            call(dst.data_ptr(), dst.numel() * 8)
            got = dst.cpu().numpy()
            torch.cuda.synchronize()
            assert torch.all(snap == -5.0).item(), f"{kind} {name}: the destination was written before the caller's queued read"
            assert np.array_equal(got, want, equal_nan=True), f"{kind} {name}: device destination differs from the host one"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STREAMS)
def test_back_to_the_own_stream_in_the_middle_of_a_run(kind, sleep_cycles):
    """set_stream(None) in the middle of a run waits for the caller stream it leaves: a plane write queued there is
    in the state the next step() on the handle's own stream starts from."""
    import torch

    S = _stream(kind)
    ex, start, cols, dt = _stream_exec()
    vx = np.random.default_rng(6).normal(0, 10, SM * SN)
    ref, _, _, _ = _stream_exec()
    with ref:
        ref.set_state(*start, **cols)
        ref.step(2, sync=True)
        v = ref.download(WORLD_VEL)
        v[..., 3] = vx.reshape(SM, SN)
        ref.upload(WORLD_VEL, v)
        ref.step(3, sync=True)
        want = tuple(ref.download(c) for c in STATE)
    with ex:
        ex.set_stream(S.cuda_stream)
        ex.set_state(*start, **cols)
        ex.step(2)
        vplane, vxd = _plane(ex, WORLD_VEL, 3), _device(vx)
        torch.cuda.synchronize()
        ev, _ = _delayed(S, sleep_cycles, lambda: vplane.copy_(vxd))
        _pending(ev, f"set_stream(None) ({kind})")
        ex.set_stream(None)
        ex.step(3)
        got = tuple(ex.download(c) for c in STATE)
    for q, a, b in zip(("pos", "vel", "accel", "force"), got, want):
        assert np.array_equal(a, b), f"{kind} {q}: the run after set_stream(None) differs from the reference"
