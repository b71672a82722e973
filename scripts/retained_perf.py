"""Retained worlds (b200_sixdof_{trajectory,state}_download_worlds, World.build(..., ensemble=True, retain=...)) on one
GPU.

    python scripts/retained_perf.py [--calls 30] [--reps 3] [--cycles 20] [--worlds 1048576] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query) and the device copy probe;
  2. trajectory_worlds call time with CUDA events on the handle's stream, the host set-up included (median, min and max
     of --calls calls after warm-up), into a device tensor and into a host array: k = 1, 64, 1024 and 65 536 worlds of
     2^20 worlds x 1 entity, over 1 and 16 samples, and 1024 of 1024 worlds x 64 entities over 64 samples.  Bytes moved
     = read + write of the gathered rows (2 x k x entities x 25 x 8 per sample) over the call time, against the probe;
  3. Exec.run per 10-tick telemetry cycle for the rocket set at --worlds worlds, FAST math: ensemble=True alone and with
     retain= 1024 spread worlds, the arms alternating --reps times, each one run() of --cycles cycles after a warm-up
     cycle; the median and range of the per-cycle times (step, reductions and retained rows of a cycle), the run's wall
     time per cycle, and each arm's host RSS growth and retained-row bytes over its cycles.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

import elodin_b200 as el
from elodin_b200 import _lib
from ensemble_perf import card, rocket_world
from group_stats_perf import ring


def rss_mb() -> float:
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) / 1024.0
    return float("nan")


def timed(st, fn, calls):
    for _ in range(3):
        fn()
    ms = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        fn()
        b.record(st)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))


def call_cases(probe, calls):
    out = []
    for M, E, S, ks in ((1 << 20, 1, 1, (1, 64, 1024, 65536)), (1 << 20, 1, 16, (1, 64, 1024, 65536)),
                        (1024, 64, 64, (1024,))):
        ex, st = ring(M, E, S)
        full = ex.trajectory()[-1] if M * E <= 1 << 16 else None
        with torch.cuda.stream(st):
            for k in ks:
                ws = np.random.default_rng(k).permutation(M)[:k]
                dev = torch.empty((S, k, E, 25), dtype=torch.float64, device="cuda")
                host = np.empty((S, k, E, 25))
                moved = 2 * k * E * 25 * 8 * S
                for dst, fn in (("device", lambda: ex.trajectory_worlds(ws, dev.data_ptr(), dev.numel() * 8)),
                                ("host", lambda: ex.trajectory_worlds(ws, host.ctypes.data, host.nbytes))):
                    n0 = ex.timings()["kernel_launches"]
                    fn()
                    launches = ex.timings()["kernel_launches"] - n0
                    t = timed(st, fn, calls)
                    gbs = moved / t[0] / 1e6
                    r = {"worlds": M, "entities": E, "samples": S, "k": k, "dst": dst, "ms": t, "bytes": moved,
                         "gbs": gbs, "of_probe": gbs / probe, "launches": launches}
                    out.append(r)
                    print(f"trajectory_worlds {M} x {E} x {S} samples, k = {k:6d}, {dst:6s}: {t[0] * 1e3:9.1f} us "
                          f"(min {t[1] * 1e3:.1f}, max {t[2] * 1e3:.1f}) = {gbs:7.1f} GB/s = {gbs / probe:.3f} of the "
                          f"copy probe, {launches} launch(es)")
                assert np.array_equal(dev.cpu().numpy(), host)
                if full is not None:
                    assert host[-1].tobytes() == np.ascontiguousarray(full[ws]).tobytes()
                del dev, host
        ex.close()
        torch.cuda.synchronize()
    return out


def history_mb(ex) -> float:
    """Host memory held by the recorded rows of the retained worlds (arrays shared between rows counted once)."""
    seen = {}
    for rows in getattr(ex, "_history", {}).values():
        for r in rows:
            seen[id(r)] = r.nbytes
    return sum(seen.values()) / 2 ** 20


def exec_case(M, cycles, arm):
    w, sys_, params = rocket_world(M)
    kw = {"retain": list(np.linspace(0, M - 1, 1024).astype(np.int64))} if arm == "retain1024" else {}
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=12.0, math="fast", n_worlds=M, world_params=params,
                 ensemble=True, **kw)
    del params
    ex.run(10)  # warm-up cycle
    r0, h0, n0 = rss_mb(), history_mb(ex), len(ex._prof["execute_buffers"])
    t0 = time.perf_counter()
    ex.run(10 * cycles)
    wall = time.perf_counter() - t0
    # per cycle: step, reductions and retained rows of that cycle (Exec._run_ensemble's own timer; the run's one upload
    # of the inputs and one download of the final state are in `wall` only)
    per = ex._prof["execute_buffers"][n0:]
    assert len(per) == cycles
    r = {"arm": arm, "worlds": M, "cycles": cycles, "ms": per, "wall_ms_per_cycle": wall * 1e3 / cycles,
         "rss_growth_mb": rss_mb() - r0, "history_growth_mb": history_mb(ex) - h0}
    ex.backend.close()
    del ex
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cycles", type=int, default=20)
    ap.add_argument("--worlds", type=int, default=1 << 20)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    if el.device_count() < 1:
        raise SystemExit("retained_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["call"] = call_cases(probe, a.calls)
    res["exec"] = []
    arms = ("alone", "retain1024")
    for rep in range(a.reps):
        for arm in arms:
            r = exec_case(a.worlds, a.cycles, arm)
            r["rep"] = rep
            res["exec"].append(r)
            print(f"Exec.run rocket set, {a.worlds} worlds, ensemble=True, {arm:10s} rep {rep}: median "
                  f"{np.median(r['ms']):.3f} ms per 10-tick cycle [{np.min(r['ms']):.3f}, {np.max(r['ms']):.3f}] over "
                  f"{a.cycles} cycles ({r['wall_ms_per_cycle']:.3f} ms of run() wall time per cycle), host RSS "
                  f"+{r['rss_growth_mb']:.1f} MB, retained rows +{r['history_growth_mb']:.2f} MB")
    for arm in arms:
        v = np.concatenate([r["ms"] for r in res["exec"] if r["arm"] == arm])
        g = [r["rss_growth_mb"] for r in res["exec"] if r["arm"] == arm]
        print(f"  {arm:10s}: median {np.median(v):.3f} ms, min {np.min(v):.3f}, max {np.max(v):.3f}; "
              f"RSS growth {min(g):.1f} to {max(g):.1f} MB over {a.cycles} cycles")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
