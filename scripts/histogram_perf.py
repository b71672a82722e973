"""Ensemble histograms (b200_sixdof_trajectory_histograms, Exec.histogram in ensemble mode) on one GPU.

    python scripts/histogram_perf.py [--cycles 50] [--worlds 1048576] [--calls 50] [--reps 3] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query);
  2. the device copy probe (b200_probe_copy_gbs);
  3. trajectory_histograms of one sample at 2^20 and 2^22 worlds x 1 entity and 1024 worlds x 1024 entities, with 1
     spec of 64 bins, 8 specs of 64 bins, 8 specs of 4096 bins and one 64 x 64 2D spec, each on spread data and on
     data with every world in one bin (the contention case): the call's time with CUDA events (median over the calls,
     one event pair per call), the bytes the specs need (worlds x 8 per axis and spec) over that time against the copy
     probe, and the call's launches;
  4. Exec.run wall time per 10-tick telemetry cycle for the rocket set at 2^20 worlds with ensemble=True alone and with
     4 histograms (world_pos z, downrange x crossrange 2D, two velocity components); the arms alternate, --reps times.
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

# (name, specs, axes read): planes 4, 5, 6 (world_pos x, y, z) of entity 0, range (-4, 4)
SETS = {
    "1x64": [(0, 6, 64, -4.0, 4.0)],
    "8x64": [(0, 4 + k % 3, 64, -4.0 + k * 0.01, 4.0) for k in range(8)],
    "8x4096": [(0, 4 + k % 3, 4096, -4.0 + k * 0.01, 4.0) for k in range(8)],
    "2d64x64": [(0, (4, 5), (64, 64), (-4.0, -4.0), (4.0, 4.0))],
}
ARMS = {"alone": None, "hist4": lambda: [
    el.Histogram("rocket.world_pos", 6, range=(0.0, 200.0), bins=100),
    el.Histogram("rocket.world_pos", (4, 5), range=((-100.0, 400.0), (-50.0, 50.0)), bins=(64, 64)),
    el.Histogram("rocket.world_vel", 3, range=(-50.0, 150.0), bins=100),
    el.Histogram("rocket.world_vel", 5, range=(-50.0, 150.0), bins=100)]}


def axes_of(specs):
    return sum(len(np.atleast_1d(s[1])) for s in specs)


def call_case(M, N, probe, calls, one_bin):
    """every spec set on one handle: [result per set]"""
    st = torch.cuda.Stream()
    out = []
    with torch.cuda.stream(st):
        ex = el.B200Exec(N, M, 1e-3, None, [], "rk4", "fast", trajectory_every=1, trajectory_capacity=1, trajectory_full=True)
        ex.set_stream(st.cuda_stream)
        rng = np.random.default_rng(1)
        pos = np.zeros((M, N, 7))
        pos[..., 3] = 1.0
        pos[..., 4:] = 0.5 if one_bin else rng.normal(0.0, 1.5, (M, N, 3))
        ine = np.tile(np.array([1.0, 1.0, 1.0, 0, 0, 0, 1.0]), (M, N, 1))
        ex.set_state(pos, np.zeros((M, N, 6)), ine)
        del pos, ine
        ex.step(1)
        for name, specs in SETS.items():
            args, row = ex._hist_specs(specs)
            dst = torch.empty((1, row), dtype=torch.float64, device="cuda")
            for _ in range(3):
                ex.trajectory_histograms(specs, out_ptr=dst.data_ptr())
            n0 = ex.timings()["kernel_launches"]
            ex.trajectory_histograms(specs, out_ptr=dst.data_ptr())
            launches = ex.timings()["kernel_launches"] - n0
            ms = []
            for _ in range(calls):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                ex.trajectory_histograms(specs, out_ptr=dst.data_ptr())
                b.record(st)
                b.synchronize()
                ms.append(a.elapsed_time(b))
            k_ms = float(np.median(ms))
            nbytes = M * 8 * axes_of(specs)
            r = {"worlds": M, "entities": N, "specs": name, "one_bin": one_bin, "launches": launches, "calls": calls,
                 "bytes": nbytes, "call_ms_median": k_ms, "call_ms_min": float(np.min(ms))}
            r["gbs"] = nbytes / (k_ms * 1e-3) / 1e9
            r["over_copy_probe"] = r["gbs"] / probe
            out.append(r)
        ex.close()
    return out


def exec_case(M, cycles, arm):
    w, sys_, params = rocket_world(M)
    kw = {} if ARMS[arm] is None else {"histograms": ARMS[arm]()}
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=12.0, math="fast", n_worlds=M, world_params=params,
                 ensemble=True, **kw)
    ex.run(10)  # warm-up cycle (module load, first launches, staging buffers)
    t0 = time.perf_counter()
    ex.run(10 * cycles)
    wall = time.perf_counter() - t0
    r = {"arm": arm, "worlds": M, "ticks_per_cycle": ex.ticks_per_telemetry, "cycles": cycles,
         "ms_per_cycle": wall * 1e3 / cycles}
    if ARMS[arm] is not None:
        h = ex.histogram(0)
        r["last_row_in_bins"] = int(h["counts"][-1].sum())
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
        raise SystemExit("histogram_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["call"] = []
    for M, N in ((1 << 20, 1), (1 << 22, 1), (1024, 1024)):
        for one_bin in (False, True):
            for r in call_case(M, N, probe, a.calls, one_bin):
                res["call"].append(r)
                print(f"trajectory_histograms, {M} worlds x {N} entities x 1 sample, {r['specs']:8s} "
                      f"{'one bin' if one_bin else 'spread '}: {r['call_ms_median'] * 1e3:.1f} us "
                      f"(min {r['call_ms_min'] * 1e3:.1f}) for {r['bytes'] / 1e6:.1f} MB = {r['gbs']:.0f} GB/s = "
                      f"{r['over_copy_probe']:.2f} of the copy probe, {r['launches']} launches")
    res["exec"] = []
    for rep in range(a.reps):
        for arm in ARMS:
            r = exec_case(a.worlds, a.cycles, arm)
            r["rep"] = rep
            res["exec"].append(r)
            print(f"Exec.run rocket set, {a.worlds} worlds, ensemble=True, {arm:5s} rep {rep}: "
                  f"{r['ms_per_cycle']:.3f} ms per {r['ticks_per_cycle']}-tick cycle over {a.cycles} cycles")
    med = {arm: float(np.median([r["ms_per_cycle"] for r in res["exec"] if r["arm"] == arm])) for arm in ARMS}
    for arm in ARMS:
        v = [r["ms_per_cycle"] for r in res["exec"] if r["arm"] == arm]
        print(f"  {arm:5s}: median {med[arm]:.3f} ms, min {np.min(v):.3f}, max {np.max(v):.3f}, "
              f"extra over alone {med[arm] - med['alone']:+.3f} ms per cycle")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
