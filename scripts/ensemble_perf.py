"""Ensemble statistics (b200_sixdof_trajectory_stats, Exec ensemble mode) on one GPU.

    python scripts/ensemble_perf.py [--cycles 50] [--worlds 1048576] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query);
  2. the device copy probe (b200_probe_copy_gbs);
  3. trajectory_stats over 2^22 worlds x 1 entity x 25 planes x 4 samples, 2^20 x 1 x 25 x 16 and 8 x 1024 x 25 x 64:
     the call's device time from CUDA events (each call ends in a stream synchronise, so the window of one call also
     holds its launch latency), and the reduction kernels' own time from torch.profiler in a separate pass; bytes read
     (every sampled value once) over kernel time against the copy probe;
  4. Exec.run wall time per telemetry cycle for the rocket set at 2^20 worlds, 10 ticks per cycle: ensemble=True
     against the default mode (per-cycle invoke_batch there), with the host RSS growth of each.
"""
import argparse
import json
import os
import resource
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import elodin_b200 as el
from elodin_b200 import _lib


def rss_mb():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) / 1024.0
    return float("nan")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[1] if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def stats_kernel_times(ex, out, calls):
    """median per-call sum of the reduction kernels' device time, from torch.profiler"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ex.trajectory_stats_to_ptr(out.data_ptr(), out.numel() * 8)
        torch.cuda.synchronize()
    evs = sorted((e for e in prof.profiler.kineto_results.events()
                  if e.device_type() == DeviceType.CUDA and "world_stats" in e.name()), key=lambda e: e.start_ns())
    per_call, cur, last_chunk = [], 0.0, None
    for e in evs:  # a call = one chunk kernel (+ one merge kernel)
        if "chunk" in e.name() and last_chunk is not None:
            per_call.append(cur)
            cur = 0.0
        if "chunk" in e.name():
            last_chunk = e
        cur += (e.end_ns() - e.start_ns()) / 1e6
    if last_chunk is not None:
        per_call.append(cur)
    return float(np.median(per_call)) if per_call else float("nan"), len(per_call)


def ring_case(M, E, S, calls, probe):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        ex = el.B200Exec(E, M, 1e-3, None, [], "rk4", "fast", trajectory_every=1, trajectory_capacity=S, trajectory_full=True)
        ex.set_stream(st.cuda_stream)
        rng = np.random.default_rng(1)
        pos = np.zeros((M, E, 7))
        pos[..., 3] = 1.0
        pos[..., 4:] = rng.normal(6.4e6, 10.0, (M, E, 3))
        vel = np.zeros((M, E, 6))
        vel[..., 3:] = rng.normal(0.0, 7.6e3, (M, E, 3))
        ine = np.tile(np.array([1.0, 1.0, 1.0, 0, 0, 0, 1.0]), (M, E, 1))
        ex.set_state(pos, vel, ine)
        del pos, vel, ine
        ex.step(S)
        out = torch.empty((S, E, 25, 5), dtype=torch.float64, device="cuda")
        for _ in range(5):  # warm-up
            ex.trajectory_stats_to_ptr(out.data_ptr(), out.numel() * 8)
        ms = []
        for _ in range(calls):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            ex.trajectory_stats_to_ptr(out.data_ptr(), out.numel() * 8)
            b.record(st)
            b.synchronize()
            ms.append(a.elapsed_time(b))
        host = ex.trajectory_stats()  # the same table through host memory
        assert np.array_equal(host, out.cpu().numpy(), equal_nan=True)
        k_ms, n_prof = stats_kernel_times(ex, out, calls)
        ex.close()
    nbytes = M * E * 25 * S * 8
    r = {"worlds": M, "entities": E, "planes": 25, "samples": S, "bytes_read": nbytes, "calls": calls,
         "call_ms_median": float(np.median(ms)), "call_ms_min": float(np.min(ms)),
         "kernel_ms_median": k_ms, "profiled_calls": n_prof,
         "kernel_gbs": nbytes / (k_ms * 1e-3) / 1e9, "call_gbs": nbytes / (np.median(ms) * 1e-3) / 1e9}
    r["kernel_over_copy_probe"] = r["kernel_gbs"] / probe
    return r


def rocket_world(M):
    Thrust = el.Annotated[np.ndarray, el.Component("thrust", el.ComponentType.F64)]
    Wind = el.Annotated[np.ndarray, el.Component("wind", el.ComponentType(el.PrimitiveType.F64, (3,)))]

    @el.dataclass
    class Rocket(el.Archetype):
        thrust: Thrust
        wind: Wind

    w = el.World()
    w.spawn([el.Body(world_pos=el.SpatialTransform(angular=el.Quaternion.from_euler([0.0, np.radians(70.0), 0.0]),
                                                   linear=np.array([0.0, 0.0, 1.0])),
                     inertia=el.SpatialInertia(3.0, np.array([0.1, 1.0, 1.0]))),
             Rocket(np.array([88.426]), np.zeros(3))], name="rocket")
    effs = el.GravityConst((0.0, 0.0, -9.81)) | el.ThrustBody((-1.0, 0.0, 0.0), "thrust") | el.DragQuadratic(0.6125, 0.0025, "wind")
    rng = np.random.default_rng(42)
    params = {"thrust": 88.426 * rng.uniform(0.8, 1.2, (M, 1, 1)),
              "wind": np.concatenate([rng.normal(0, 2, (M, 1, 1)), np.zeros((M, 1, 2))], -1),
              "inertia": np.concatenate([np.tile([0.1, 1.0, 1.0, 0, 0, 0], (M, 1, 1)), rng.uniform(2.5, 3.5, (M, 1, 1))], -1)}
    return w, el.six_dof(sys=effs), params


def exec_case(M, cycles, ensemble):
    w, sys_, params = rocket_world(M)
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=12.0, math="fast", n_worlds=M, world_params=params,
                 ensemble=ensemble)
    ex.run(10)  # warm-up cycle (module load, first launches, staging buffers)
    rss0 = rss_mb()
    t0 = time.perf_counter()
    ex.run(10 * cycles)
    wall = time.perf_counter() - t0
    rss1 = rss_mb()
    r = {"ensemble": ensemble, "worlds": M, "ticks_per_cycle": ex.ticks_per_telemetry, "cycles": cycles,
         "ms_per_cycle": wall * 1e3 / cycles, "rss_growth_mb": rss1 - rss0, "rss_mb_after": rss1}
    if ensemble:
        x = ex.ensemble("rocket.world_pos")
        r["final_downrange_mean_m"] = float(x["mean"][-1, 4])
        r["final_downrange_std_m"] = float(x["std"][-1, 4])
        r["final_count"] = float(x["count"][-1, 4])
    else:
        x = ex.world.columns[el.component_id("world_pos")].buffer[:, 0, 4]
        r["final_downrange_mean_m"] = float(np.mean(x))
        r["final_downrange_std_m"] = float(np.std(x))
    final = ex.world.columns[el.component_id("world_pos")].buffer.copy()
    ex.backend.close()
    del ex
    return r, final


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cycles", type=int, default=50)
    ap.add_argument("--worlds", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    if el.device_count() < 1:
        raise SystemExit("ensemble_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["trajectory_stats"] = []
    for M, E, S in ((1 << 22, 1, 4), (1 << 20, 1, 16), (8, 1024, 64)):
        r = ring_case(M, E, S, a.calls, probe)
        res["trajectory_stats"].append(r)
        print(f"trajectory_stats {M} worlds x {E} entities x 25 planes x {S} samples ({r['bytes_read'] / 1e9:.3f} GB): "
              f"kernels {r['kernel_ms_median'] * 1e3:.1f} us = {r['kernel_gbs']:.0f} GB/s = {r['kernel_over_copy_probe']:.2f} "
              f"of the copy probe; call (events, median of {a.calls}) {r['call_ms_median'] * 1e3:.1f} us")
    res["exec"] = []
    finals = {}
    for ens in (True, False):
        r, finals[ens] = exec_case(a.worlds, a.cycles, ens)
        res["exec"].append(r)
        print(f"Exec.run rocket set, {a.worlds} worlds, {r['ticks_per_cycle']} ticks per cycle, {a.cycles} cycles, "
              f"{'ensemble=True' if ens else 'default mode'}: {r['ms_per_cycle']:.2f} ms per cycle, host RSS "
              f"+{r['rss_growth_mb']:.0f} MB; final downrange mean {r['final_downrange_mean_m']:.4f} m, "
              f"std {r['final_downrange_std_m']:.4f} m")
    res["final_state_identical"] = bool(np.array_equal(finals[True], finals[False]))
    print("final world_pos identical between the two modes:", res["final_state_identical"])
    res["max_rss_mb"] = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
