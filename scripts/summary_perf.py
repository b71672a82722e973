"""Run summaries (b200_sixdof_summary_*, Exec extrema / thresholds in ensemble mode) on one GPU.

    python scripts/summary_perf.py [--cycles 50] [--worlds 1048576] [--reps 3] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query);
  2. the device copy probe (b200_probe_copy_gbs);
  3. summary_add_trajectory with extrema and one threshold over 2^22 bodies x 1 sample and 2^20 x 16 samples: the
     fold kernel's own time from torch.profiler (summary_fold_kernel, median over the calls) and the call's device time
     from CUDA events; bytes moved (every sample of the 25 planes read once, the 125 extrema planes read and written
     once: 200 B per sample + 2000 B per body) over kernel time, against the copy probe; and the same for one
     threshold alone at 2^20 bodies x 1 sample (its plane and its tick: 16 B per body);
  4. Exec.run wall time per 10-tick telemetry cycle for the rocket set at 2^20 worlds with ensemble=True alone, with
     extrema=True, and with one threshold (rocket z below 0) only; the three arms alternate, --reps times.
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

KERNEL = "summary_fold_kernel"


def fold_kernel_ms(ex, calls):
    """median device time of the fold kernel per call, from torch.profiler"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ex.summary_add_trajectory()
        torch.cuda.synchronize()
    ms = [(e.end_ns() - e.start_ns()) / 1e6 for e in prof.profiler.kineto_results.events()
          if e.device_type() == DeviceType.CUDA and KERNEL in e.name()]
    return (float(np.median(ms)) if ms else float("nan")), len(ms)


def fold_case(M, S, calls, probe, extrema=True):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        ex = el.B200Exec(1, M, 1e-3, None, [], "rk4", "fast", trajectory_every=1, trajectory_capacity=S, trajectory_full=True)
        ex.set_stream(st.cuda_stream)
        rng = np.random.default_rng(1)
        pos = np.zeros((M, 1, 7))
        pos[..., 3] = 1.0
        pos[..., 4:] = rng.normal(6.4e6, 10.0, (M, 1, 3))
        vel = np.zeros((M, 1, 6))
        vel[..., 3:] = rng.normal(0.0, 7.6e3, (M, 1, 3))
        ine = np.tile(np.array([1.0, 1.0, 1.0, 0, 0, 0, 1.0]), (M, 1, 1))
        ex.set_state(pos, vel, ine)
        del pos, vel, ine
        ex.summary_begin(extrema, [(0, 6, False, 6.4e6)])
        ex.step(S)
        for _ in range(5):  # warm-up; folding the same rows again leaves every bit as it is
            ex.summary_add_trajectory()
        ms = []
        for _ in range(calls):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            ex.summary_add_trajectory()
            b.record(st)
            b.synchronize()
            ms.append(a.elapsed_time(b))
        k_ms, n_prof = fold_kernel_ms(ex, calls)
        ex.close()
    # extrema: 25 planes per sample read, 125 accumulator planes read and written; one threshold alone: its plane per
    # sample and its tick per world (read as part of a 32-byte sector: the table is world-major, 208 B per world)
    nbytes = M * (S * 25 * 8 + 125 * 8 * 2) if extrema else M * (S * 8 + 8)
    r = {"extrema": extrema, "bodies": M, "samples": S, "bytes_moved": nbytes, "calls": calls,
         "call_ms_median": float(np.median(ms)),
         "kernel_ms_median": k_ms, "profiled_kernels": n_prof, "kernel_gbs": nbytes / (k_ms * 1e-3) / 1e9}
    r["kernel_over_copy_probe"] = r["kernel_gbs"] / probe
    return r


def exec_case(M, cycles, arm):
    w, sys_, params = rocket_world(M)
    kw = {"alone": {}, "extrema": {"extrema": True},
          "threshold": {"thresholds": [el.Threshold("rocket.world_pos", 6, below=0.0)]}}[arm]
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=12.0, math="fast", n_worlds=M, world_params=params,
                 ensemble=True, **kw)
    ex.run(10)  # warm-up cycle (module load, first launches, staging buffers)
    t0 = time.perf_counter()
    ex.run(10 * cycles)
    wall = time.perf_counter() - t0
    r = {"arm": arm, "worlds": M, "ticks_per_cycle": ex.ticks_per_telemetry, "cycles": cycles,
         "ms_per_cycle": wall * 1e3 / cycles}
    if arm == "extrema":
        x = ex.extrema("rocket.world_pos")
        r["max_altitude_median_m"] = float(np.median(x["max"][:, 6]))
        r["max_altitude_tick_median"] = float(np.median(x["max_tick"][:, 6]))
    elif arm == "threshold":
        t = ex.threshold(0)["tick"]
        r["impacted_worlds"] = int(np.sum(t >= 0))
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
        raise SystemExit("summary_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["fold"] = []
    for M, S, ext in ((1 << 22, 1, True), (1 << 20, 16, True), (1 << 20, 1, False)):
        r = fold_case(M, S, a.calls, probe, ext)
        res["fold"].append(r)
        what = "extrema + 1 threshold" if ext else "1 threshold alone"
        print(f"summary_add_trajectory, {what}, {M} bodies x {S} samples ({r['bytes_moved'] / 1e9:.3f} GB "
              f"moved): {KERNEL} {r['kernel_ms_median'] * 1e3:.1f} us = {r['kernel_gbs']:.0f} GB/s = "
              f"{r['kernel_over_copy_probe']:.2f} of the copy probe; call (events, median of {a.calls}) "
              f"{r['call_ms_median'] * 1e3:.1f} us")
    res["exec"] = []
    for rep in range(a.reps):
        for arm in ("alone", "extrema", "threshold"):
            r = exec_case(a.worlds, a.cycles, arm)
            r["rep"] = rep
            res["exec"].append(r)
            extra = {k: v for k, v in r.items() if k.startswith(("max_", "impacted"))}
            print(f"Exec.run rocket set, {a.worlds} worlds, ensemble=True, {arm:9s} rep {rep}: "
                  f"{r['ms_per_cycle']:.3f} ms per {r['ticks_per_cycle']}-tick cycle over {a.cycles} cycles {extra or ''}")
    for arm in ("alone", "extrema", "threshold"):
        v = [r["ms_per_cycle"] for r in res["exec"] if r["arm"] == arm]
        print(f"  {arm:9s}: median {np.median(v):.3f} ms, min {np.min(v):.3f}, max {np.max(v):.3f}")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
