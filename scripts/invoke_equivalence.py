"""Two builds of the package, byte for byte, through invoke_batch and step.

    python scripts/invoke_equivalence.py --other DIR [--out DIR]

DIR holds another built copy of the package (DIR/elodin_b200, e.g. the parent commit's).  Each side runs the seeded
cases below in a process of its own and writes every output column of every call, tick_count, trajectory() where the
handle has a ring, and timings()["kernel_launches"] to one .npz; the two files must then hold the same arrays with the
same bytes.  The cases walk the host runtime's branches: the packed small path and the pipelined path (whole-batch and
ragged world ranges), both math modes and integrators, inputs that are not dirty, outputs nobody reads, pass-through
outputs with their input present, absent and aliasing the output, caller buffers in device memory, the one-launch n-body
tick over odd and even tick counts, small worlds, a sparse graph, EGM08, a masked effector, Inertia uploaded between
calls.  Needs a GPU: there is no CPU fallback, so without one the first create fails.
"""
import argparse
import os
import subprocess
import sys
import tempfile

import numpy as np

DT = 1.0 / 120.0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def world(seed, M, N, scale=1e3):
    rng = np.random.default_rng(seed)
    q = rng.normal(size=(M, N, 4))
    q /= np.linalg.norm(q, axis=-1, keepdims=True)
    pos = np.concatenate([q, rng.uniform(-scale, scale, (M, N, 3))], -1)
    vel = np.concatenate([rng.normal(0, 0.5, (M, N, 3)), rng.normal(0, 10, (M, N, 3))], -1)
    ine = np.concatenate([rng.uniform(0.1, 10, (M, N, 3)), np.zeros((M, N, 3)), rng.uniform(0.5, 50, (M, N, 1))], -1)
    return pos, vel, ine


def effectors(el, kind, N):
    """(effector list, {column name: width}) of one kind of world."""
    if kind == "free":
        return [el.GravityConst(), el.ThrustBody((1.0, 0.0, 0.0), "thrust"), el.WrenchBody("aero")], {"thrust": 1, "aero": 6}
    if kind == "masked":
        mask = (np.arange(N) % 2).astype(np.uint8)
        return [el.GravityConst(), el.WrenchWorld("ext").with_mask(mask), el.DragQuadratic(column="wind")], {"ext": 6, "wind": 3}
    if kind == "wheels":
        return [el.GravityJ2(), el.TorqueBodyFold("wheels", 3)], {"wheels": 9}
    if kind == "dense":
        return [el.GravityEdges("softened", k_squared=1e-3, softening=1e-6, edges=el.all_pairs_edges(N))], {}
    if kind == "sparse":
        ring = np.array([[i, (i + k) % N] for i in range(N) for k in (1, 2, 5)], dtype=np.uint32)
        return [el.GravityEdges("newton", G=6.6743e-3, edges=ring), el.ThrustBody((0.0, 0.0, 1.0), "thrust")], {"thrust": 1}
    if kind == "egm08":
        rng = np.random.default_rng(77)
        c, s = rng.normal(0, 1e-6, (7, 7)), rng.normal(0, 1e-6, (7, 7))
        c[0, 0] = 1.0
        return [el.GravityEGM08(c, s, 6), el.ThrustBody((1.0, 0.0, 0.0), "thrust")], {"thrust": 1}
    raise ValueError(kind)


# kind, N, M, math, integrator, invoke_chunk_bodies, max_fused_ticks, trajectory ring, position scale
CASES = [
    ("free", 1, 1, "exact", "rk4", 0, 1, True, 1e3),
    ("free", 3, 100, "fast", "rk4", 0, 4, False, 1e3),
    ("free", 3, 100, "exact", "semi_implicit", 0, 1, True, 1e3),
    ("free", 3, 1000, "fast", "rk4", 231, 4, True, 1e3),            # 77 worlds a range, ragged last range
    ("free", 1, 1025, "exact", "rk4", 200, 1, False, 1e3),          # 128-world ranges of single bodies
    ("free", 5, 60000, "fast", "semi_implicit", 0, 2, False, 1e3),  # past the small path: default ranges
    ("masked", 4, 64, "exact", "rk4", 0, 1, False, 1e3),
    ("masked", 4, 640, "fast", "rk4", 1000, 1, False, 1e3),
    ("wheels", 2, 300, "fast", "rk4", 128, 3, True, 7e6),
    ("dense", 48, 6, "fast", "rk4", 0, 1, True, 30.0),              # one-launch n-body tick, small path
    ("dense", 48, 7, "fast", "rk4", 96, 1, True, 30.0),             # the same through ranges of 2 worlds (last: 1)
    ("dense", 48, 6, "exact", "rk4", 0, 1, False, 30.0),            # two launches per tick
    ("dense", 3, 50, "fast", "rk4", 0, 8, True, 30.0),              # small worlds: n ticks per launch
    ("dense", 8, 500, "exact", "semi_implicit", 800, 8, False, 30.0),
    ("sparse", 40, 9, "fast", "rk4", 80, 1, False, 30.0),
    ("sparse", 40, 9, "exact", "rk4", 0, 1, True, 30.0),
    ("egm08", 2, 40, "exact", "rk4", 0, 4, True, 7e6),
    ("egm08", 2, 400, "fast", "rk4", 100, 4, False, 7e6),
]

# One call of a case: ticks, which inputs are not dirty, which outputs nobody reads, which pass-through outputs alias their
# input buffer, and whether the caller's buffers are device memory.  Column names; "state" = pos, vel, accel, force.
CALLS = [
    dict(ticks=1),
    dict(ticks=3, not_dirty=("inertia", "effector"), unread=("force",)),
    dict(ticks=2, alias=True, unread=("world_accel", "tick")),
    dict(ticks=5, not_dirty=("inertia", "tick", "simulation_time_step"), device=True),
    dict(ticks=4, device=True, alias=True, not_dirty=("effector",)),
    dict(ticks=1, not_dirty=("world_pos", "world_vel", "world_accel", "force", "inertia", "effector")),
]


def run_side(out_path):
    import elodin_b200 as el
    import torch
    from elodin_b200.executor import FORCE, INERTIA, SIMULATION_TIME_STEP, TICK, WORLD_ACCEL, WORLD_POS, WORLD_VEL

    names = {WORLD_POS: "world_pos", WORLD_VEL: "world_vel", WORLD_ACCEL: "world_accel", FORCE: "force", INERTIA: "inertia",
             TICK: "tick", SIMULATION_TIME_STEP: "simulation_time_step"}
    rec = {}
    for ci, (kind, N, M, math, integ, chunk, fuse, ring, scale) in enumerate(CASES):
        effs, cols = effectors(el, kind, N)
        ex = el.B200Exec(N, M, DT, None, effs, integ, math, max_fused_ticks=fuse, invoke_chunk_bodies=chunk,
                         trajectory_every=2 if ring else 0, trajectory_capacity=6 if ring else 0)
        rng = np.random.default_rng(1000 + ci)
        pos, vel, ine = world(ci, M, N, scale)
        val = {WORLD_POS: pos, WORLD_VEL: vel, INERTIA: ine, WORLD_ACCEL: rng.normal(size=(M, N, 6)), FORCE: rng.normal(size=(M, N, 6)),
               TICK: np.array([7], dtype=np.uint64), SIMULATION_TIME_STEP: np.array([DT])}
        for name, w in cols.items():
            names[el.component_id(name)] = "effector"
            val[el.component_id(name)] = rng.normal(size=(M, N, w))
        key = lambda what: f"case{ci:02d}.{what}"

        def snapshot(tag):
            rec[key(f"{tag}.tick_count")] = np.array([ex.tick], dtype=np.uint64)
            rec[key(f"{tag}.launches")] = np.array([ex.timings()["kernel_launches"]], dtype=np.uint64)
            if ring:
                rec[key(f"{tag}.trajectory")] = ex.trajectory()

        for k, call in enumerate(CALLS):
            dev = call.get("device", False)
            ins, outs, keep = [], {}, []
            for c in ex.input_ids:
                if names[c] in call.get("not_dirty", ()):
                    ins.append(None)
                    continue
                a = np.ascontiguousarray(val[c])
                if dev and c not in (TICK, SIMULATION_TIME_STEP):
                    a = torch.from_numpy(a.view(np.uint8).reshape(-1)).cuda()
                keep.append(a)
                ins.append(a)
            for j, c in enumerate(ex.output_ids):
                if names[c] in call.get("unread", ()):
                    continue
                same = ins[ex.input_ids.index(c)]
                if call.get("alias") and names[c] in ("inertia", "effector") and same is not None:
                    outs[c] = same  # the pass-through output is the input buffer itself
                elif dev and c not in (TICK, SIMULATION_TIME_STEP):
                    outs[c] = torch.full((ex.column_bytes(c),), 0xAB, dtype=torch.uint8, device="cuda")
                else:
                    outs[c] = np.full(ex.column_shape(c), 0xAB, dtype=np.uint8).repeat(8, -1).view(
                        np.uint64 if c == TICK else np.float64)
            ptr = lambda a: None if a is None else (a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data)
            torch.cuda.synchronize()
            ex.invoke_batch_ptrs([ptr(a) for a in ins], [ptr(outs.get(c)) for c in ex.output_ids], call["ticks"])
            torch.cuda.synchronize()
            for c, a in outs.items():
                host = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
                host = host.view(np.uint64 if c == TICK else np.float64).reshape(ex.column_shape(c))
                rec[key(f"call{k}.out.{c:016x}")] = host.copy()
                if names[c] not in ("inertia", "effector"):
                    val[c] = host.copy()  # the next call's input, as a host would feed it back
            snapshot(f"call{k}")
            if k == 2:  # between calls: new masses through upload(), odd and even tick counts through step()
                val[INERTIA] = val[INERTIA] * 1.5
                ex.upload(INERTIA, val[INERTIA])
                for n in (3, 2):
                    ex.step(n, sync=True)
                    for c in (WORLD_POS, WORLD_VEL, WORLD_ACCEL, FORCE):
                        rec[key(f"step{n}.{c:016x}")] = ex.download(c)
                    snapshot(f"step{n}")
                ex.trajectory_reset()
        ex.close()
        print(f"case {ci:2d} {kind:7s} {M} x {N} {math} {integ} chunk {chunk}: done", flush=True)
    np.savez(out_path, **rec)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--other", help="directory holding the other build's elodin_b200 package")
    ap.add_argument("--out", help="directory for the two .npz files (default: a temporary one)")
    ap.add_argument("--side", nargs=2, metavar=("PACKAGE_ROOT", "NPZ"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.side:
        sys.path.insert(0, a.side[0])
        return run_side(a.side[1])
    if not a.other or not os.path.isdir(os.path.join(a.other, "elodin_b200")):
        ap.error("--other DIR must hold an elodin_b200 package")
    out = a.out or tempfile.mkdtemp(prefix="invoke_equivalence_")
    os.makedirs(out, exist_ok=True)
    files = {}
    for side, root in (("other", os.path.abspath(a.other)), ("this", ROOT)):
        files[side] = os.path.join(out, f"{side}.npz")
        env = {k: v for k, v in os.environ.items() if k != "PYTHONPATH"}
        subprocess.run([sys.executable, os.path.abspath(__file__), "--side", root, files[side]], check=True, env=env)
    x, y = np.load(files["other"]), np.load(files["this"])
    bad = [k for k in sorted(set(x.files) | set(y.files))
           if k not in x.files or k not in y.files or x[k].dtype != y[k].dtype or x[k].shape != y[k].shape
           or x[k].tobytes() != y[k].tobytes()]
    nbytes = sum(x[k].nbytes for k in x.files)
    if bad:
        print(f"DIFFERENT: {len(bad)} of {len(x.files)} arrays, first {bad[:8]}")
        return 1
    print(f"identical: {len(x.files)} arrays, {nbytes} bytes, {len(CASES)} cases x {len(CALLS)} calls")
    return 0


if __name__ == "__main__":
    sys.exit(main())
