"""Ensemble quantiles (b200_sixdof_trajectory_quantiles, Exec.quantiles in ensemble mode) on one GPU.

    python scripts/quantile_perf.py [--cycles 50] [--worlds 1048576] [--calls 50] [--reps 3] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query);
  2. the device copy probe (b200_probe_copy_gbs);
  3. trajectory_quantiles at 2^22 worlds x 1 entity x 1 sample, 2^20 x 1 x 16 and 8 x 1024 x 64 (25 planes), for 1 and
     16 levels: the summed device time of the call's kernels from torch.profiler (median over the calls), the reads of
     the planes the call made (b200_sixdof_quantile_reads, counted from the pass plan), those bytes over kernel time
     against the copy probe, and the call's launches;
  4. Exec.run wall time per 10-tick telemetry cycle for the rocket set at 2^20 worlds with ensemble=True alone, with
     quantiles=(0.01, 0.5, 0.99) and with 16 levels, and the growth of the process's resident memory over the run; the
     three arms alternate, --reps times.
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

LEVELS16 = tuple(np.linspace(0.0, 1.0, 16))


def rss_mb():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) / 1024.0
    return float("nan")


def kernel_ms(ex, q, calls):
    """median over the calls of the summed device time of the quantile kernels of one call, from torch.profiler"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ex.trajectory_quantiles(q)
        torch.cuda.synchronize()
    ev = sorted((e.start_ns(), e.end_ns()) for e in prof.profiler.kineto_results.events()
                if e.device_type() == DeviceType.CUDA and "quantile" in e.name())
    per = len(ev) // calls if calls else 0
    sums = [sum(b - a for a, b in ev[c * per:(c + 1) * per]) / 1e6 for c in range(calls)] if per else []
    return (float(np.median(sums)) if sums else float("nan")), per


def call_case(M, N, S, q, calls, probe):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        ex = el.B200Exec(N, M, 1e-3, None, [], "rk4", "fast", trajectory_every=1, trajectory_capacity=S, trajectory_full=True)
        ex.set_stream(st.cuda_stream)
        rng = np.random.default_rng(1)
        pos = np.zeros((M, N, 7))
        pos[..., 3] = 1.0
        pos[..., 4:] = rng.normal(6.4e6, 10.0, (M, N, 3))
        vel = np.zeros((M, N, 6))
        vel[..., 3:] = rng.normal(0.0, 7.6e3, (M, N, 3))
        ine = np.tile(np.array([1.0, 1.0, 1.0, 0, 0, 0, 1.0]), (M, N, 1))
        ex.set_state(pos, vel, ine)
        del pos, vel, ine
        ex.step(S)
        for _ in range(3):
            ex.trajectory_quantiles(q)
        n0 = ex.timings()["kernel_launches"]
        ex.trajectory_quantiles(q)
        launches = ex.timings()["kernel_launches"] - n0
        reads = ex.quantile_reads()
        k_ms, per = kernel_ms(ex, q, calls)
        ex.close()
    plane_bytes = M * N * 25 * S * 8
    r = {"worlds": M, "entities": N, "samples": S, "levels": len(q), "calls": calls, "launches": launches,
         "reads": reads, "bytes_read": reads * plane_bytes, "kernel_ms_median": k_ms, "profiled_kernels_per_call": per}
    r["kernel_gbs"] = r["bytes_read"] / (k_ms * 1e-3) / 1e9
    r["kernel_over_copy_probe"] = r["kernel_gbs"] / probe
    return r


def exec_case(M, cycles, arm):
    w, sys_, params = rocket_world(M)
    kw = {"alone": {}, "q3": {"quantiles": (0.01, 0.5, 0.99)}, "q16": {"quantiles": LEVELS16}}[arm]
    rss0 = rss_mb()
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=12.0, math="fast", n_worlds=M, world_params=params,
                 ensemble=True, **kw)
    ex.run(10)  # warm-up cycle (module load, first launches, staging buffers)
    t0 = time.perf_counter()
    ex.run(10 * cycles)
    wall = time.perf_counter() - t0
    r = {"arm": arm, "worlds": M, "ticks_per_cycle": ex.ticks_per_telemetry, "cycles": cycles,
         "ms_per_cycle": wall * 1e3 / cycles, "rss_growth_mb": rss_mb() - rss0}
    if arm != "alone":
        r["altitude_last_row"] = ex.quantiles("rocket.world_pos")[-1, :, 6].tolist()[:3]
    ex.backend.close()
    del ex
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cycles", type=int, default=50)
    ap.add_argument("--worlds", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    if el.device_count() < 1:
        raise SystemExit("quantile_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["call"] = []
    for M, N, S in ((1 << 22, 1, 1), (1 << 20, 1, 16), (8, 1024, 64)):
        for q in ((0.5,), LEVELS16):
            r = call_case(M, N, S, q, a.calls, probe)
            res["call"].append(r)
            print(f"trajectory_quantiles, {M} worlds x {N} entities x {S} samples, {len(q):2d} levels: "
                  f"{r['reads']:.2f} reads ({r['bytes_read'] / 1e9:.3f} GB), kernels {r['kernel_ms_median'] * 1e3:.1f} us "
                  f"= {r['kernel_gbs']:.0f} GB/s = {r['kernel_over_copy_probe']:.2f} of the copy probe, "
                  f"{r['launches']} launches")
    res["exec"] = []
    for rep in range(a.reps):
        for arm in ("alone", "q3", "q16"):
            r = exec_case(a.worlds, a.cycles, arm)
            r["rep"] = rep
            res["exec"].append(r)
            print(f"Exec.run rocket set, {a.worlds} worlds, ensemble=True, {arm:5s} rep {rep}: "
                  f"{r['ms_per_cycle']:.3f} ms per {r['ticks_per_cycle']}-tick cycle over {a.cycles} cycles, "
                  f"RSS +{r['rss_growth_mb']:.0f} MB")
    for arm in ("alone", "q3", "q16"):
        v = [r["ms_per_cycle"] for r in res["exec"] if r["arm"] == arm]
        print(f"  {arm:5s}: median {np.median(v):.3f} ms, min {np.min(v):.3f}, max {np.max(v):.3f}")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
