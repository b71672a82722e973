"""Run scores (b200_sixdof_summary_start moments and dwells, Exec moments= / dwells= in ensemble mode) on one GPU.

    python scripts/scores_perf.py [--parent path/to/parent/libb200_sixdof.so] [--worlds 1048576] [--reps 3] [--out r.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query) and the device copy probe;
  2. summary_add_trajectory over 2^22 bodies x 1 sample and 2^20 x 16 samples with moments of 4 planes, with 2 dwells
     as well, and with extrema and the 4 moments together: the fold kernel's time from torch.profiler (median over
     the calls), and the bytes the fold must move (8 B per sample and plane read; 32 B read and 32 B written per body
     and moment plane; 48 B per world and dwell; extrema as scripts/summary_perf.py counts them) over that time,
     against the copy probe;
  3. Exec.run wall time per 10-tick telemetry cycle for the rocket set at 2^20 worlds with ensemble=True alone, with 4
     moment planes and 2 dwells, and with extrema as well; the arms alternate, --reps times;
  4. with --parent: scripts/summary_perf.py's fold shapes (extrema + 1 threshold, 1 threshold alone) on the parent's
     library and on this one, in alternating child processes: the tables' bits and the fold kernel times.
"""
import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np

KERNEL = "summary_fold_kernel"
MOMENTS = [4, 5, 6, 10]
DWELLS = [(0, 6, False, 6.4e6), (0, 10, True, 0.0)]
THRESHOLD = [(0, 6, False, 6.4e6)]


def fold_kernel_ms(ex, calls):
    """median device time of the fold kernel per call, from torch.profiler"""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ex.summary_add_trajectory()
        torch.cuda.synchronize()
    ms = [(e.end_ns() - e.start_ns()) / 1e6 for e in prof.profiler.kineto_results.events()
          if e.device_type() == DeviceType.CUDA and KERNEL in e.name()]
    return (float(np.median(ms)) if ms else float("nan")), len(ms)


def fold_handle(M, S):
    import elodin_b200 as el

    ex = el.B200Exec(1, M, 1e-3, None, [], "rk4", "fast", trajectory_every=1, trajectory_capacity=S, trajectory_full=True)
    rng = np.random.default_rng(1)
    pos = np.zeros((M, 1, 7))
    pos[..., 3] = 1.0
    pos[..., 4:] = rng.normal(6.4e6, 10.0, (M, 1, 3))
    vel = np.zeros((M, 1, 6))
    vel[..., 3:] = rng.normal(0.0, 7.6e3, (M, 1, 3))
    ine = np.tile(np.array([1.0, 1.0, 1.0, 0, 0, 0, 1.0]), (M, 1, 1))
    ex.set_state(pos, vel, ine)
    ex.step(S)
    return ex


def fold_bytes(M, S, extrema, n_thr, moments, dwells):
    planes = set(range(25)) if extrema else {p for _, p, _, _ in THRESHOLD[:n_thr]} | set(moments) | \
        {p for _, p, _, _ in dwells}
    b = M * S * len(planes) * 8 + M * len(moments) * 64 + M * len(dwells) * 48
    if extrema:
        b += M * 125 * 16
    elif n_thr:
        b += M * 8
    return b


def fold_case(M, S, calls, probe, extrema, n_thr, moments, dwells):
    ex = fold_handle(M, S)
    ex.summary_begin(extrema, THRESHOLD[:n_thr], moments, dwells)
    for _ in range(5):  # warm-up
        ex.summary_add_trajectory()
    k_ms, n_prof = fold_kernel_ms(ex, calls)
    ex.close()
    nbytes = fold_bytes(M, S, extrema, n_thr, moments, dwells)
    r = {"extrema": extrema, "thresholds": n_thr, "moments": len(moments), "dwells": len(dwells), "bodies": M,
         "samples": S, "bytes_moved": nbytes, "kernel_ms_median": k_ms, "profiled_kernels": n_prof,
         "kernel_gbs": nbytes / (k_ms * 1e-3) / 1e9}
    r["kernel_over_copy_probe"] = r["kernel_gbs"] / probe
    return r


def exec_case(M, cycles, arm):
    import elodin_b200 as el
    from ensemble_perf import rocket_world

    w, sys_, params = rocket_world(M)
    scores = {"moments": [("world_pos", (4, 5, 6)), ("world_vel", (3,))],
              "dwells": [el.Threshold("rocket.world_pos", 6, below=0.0), el.Threshold("rocket.world_vel", 3, above=0.0)]}
    kw = {"alone": {}, "scores": scores, "scores+extrema": dict(scores, extrema=True)}[arm]
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=12.0, math="fast", n_worlds=M, world_params=params,
                 ensemble=True, **kw)
    ex.run(10)  # warm-up cycle
    t0 = time.perf_counter()
    ex.run(10 * cycles)
    wall = time.perf_counter() - t0
    r = {"arm": arm, "worlds": M, "ticks_per_cycle": ex.ticks_per_telemetry, "cycles": cycles,
         "ms_per_cycle": wall * 1e3 / cycles}
    if arm != "alone":
        m = ex.moments("rocket.world_pos")
        r["rms_z_median_m"] = float(np.median(m["rms"][:, 2]))
        r["rows_below_ground_median"] = float(np.median(ex.dwell(0)["rows"]))
    ex.backend.close()
    return r


def child(lib_path, calls):
    """summary_perf.py's fold shapes on the library at lib_path: table digests and fold kernel times, as JSON."""
    from elodin_b200 import _lib

    class Tolerant(ctypes.CDLL):  # a parent library lacks the newer symbols: bind what it has
        def __getattr__(self, name):
            try:
                return super().__getattr__(name)
            except AttributeError:
                if not name.startswith("b200_"):
                    raise
                return type("Missing", (), {})()

    _lib.LIB_PATH = lib_path
    ctypes.CDLL = Tolerant
    out = []
    for M, S, ext in ((1 << 22, 1, True), (1 << 20, 16, True), (1 << 20, 1, False)):
        ex = fold_handle(M, S)
        ex.summary_begin(ext, THRESHOLD)
        ex.summary_add_trajectory()
        digest = hashlib.sha256((ex.extrema().tobytes() if ext else b"") + ex.thresholds().tobytes()).hexdigest()
        k_ms, _ = fold_kernel_ms(ex, calls)
        ex.close()
        out.append({"bodies": M, "samples": S, "extrema": ext, "digest": digest, "kernel_ms_median": k_ms})
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cycles", type=int, default=50)
    ap.add_argument("--worlds", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--parent", default=None, help="the parent commit's libb200_sixdof.so, for part 4")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    if a.child:
        return child(a.child, a.calls)
    import elodin_b200 as el
    from elodin_b200 import _lib
    from ensemble_perf import card

    if el.device_count() < 1:
        raise SystemExit("scores_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["fold"] = []
    arms = (("extrema + 1 threshold", True, 1, [], []), ("4 moments", False, 0, MOMENTS, []),
            ("4 moments + 2 dwells", False, 0, MOMENTS, DWELLS), ("extrema + 4 moments", True, 0, MOMENTS, []))
    for M, S in ((1 << 22, 1), (1 << 20, 16)):
        for what, ext, n_thr, mom, dw in arms:
            r = fold_case(M, S, a.calls, probe, ext, n_thr, mom, dw)
            r["arm"] = what
            res["fold"].append(r)
            print(f"summary_add_trajectory, {what:22s}, {M} bodies x {S:2d} samples ({r['bytes_moved'] / 1e9:.3f} GB): "
                  f"{KERNEL} {r['kernel_ms_median'] * 1e3:.1f} us = {r['kernel_gbs']:.0f} GB/s = "
                  f"{r['kernel_over_copy_probe']:.2f} of the copy probe ({r['profiled_kernels']} kernels profiled)")
    res["exec"] = []
    for rep in range(a.reps):
        for arm in ("alone", "scores", "scores+extrema"):
            r = exec_case(a.worlds, a.cycles, arm)
            r["rep"] = rep
            res["exec"].append(r)
            print(f"Exec.run rocket set, {a.worlds} worlds, ensemble=True, {arm:14s} rep {rep}: "
                  f"{r['ms_per_cycle']:.3f} ms per {r['ticks_per_cycle']}-tick cycle over {a.cycles} cycles")
    for arm in ("alone", "scores", "scores+extrema"):
        v = [r["ms_per_cycle"] for r in res["exec"] if r["arm"] == arm]
        print(f"  {arm:14s}: median {np.median(v):.3f} ms, min {np.min(v):.3f}, max {np.max(v):.3f}")
    if a.parent:
        res["parent"] = []
        libs = (("parent", os.path.abspath(a.parent)), ("this", _lib.LIB_PATH))
        for rep in range(a.reps):
            for name, path in libs:
                q = subprocess.run([sys.executable, __file__, "--child", path, "--calls", str(a.calls)],
                                   capture_output=True, text=True, check=True)
                for r in json.loads(q.stdout.strip().splitlines()[-1]):
                    r.update(lib=name, rep=rep)
                    res["parent"].append(r)
        for M, S, ext in ((1 << 22, 1, True), (1 << 20, 16, True), (1 << 20, 1, False)):
            rs = [r for r in res["parent"] if (r["bodies"], r["samples"], r["extrema"]) == (M, S, ext)]
            same = len({r["digest"] for r in rs}) == 1
            t = {n: [r["kernel_ms_median"] * 1e3 for r in rs if r["lib"] == n] for n, _ in libs}
            print(f"parent vs this, {'extrema + 1 threshold' if ext else '1 threshold alone':22s} {M} x {S:2d}: "
                  f"same bits {same}; fold kernel us parent {['%.1f' % x for x in t['parent']]} "
                  f"this {['%.1f' % x for x in t['this']]}")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
