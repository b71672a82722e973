"""Derived channels (b200_sixdof_set_channels, channel_kernels.cu, World.build(..., channels=...)) on one GPU.

    python scripts/channels_perf.py [--parent-lib PATH] [--calls 20] [--reps 3] [--cycles 10] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query) and the device copy probe;
  2. channel_kernel's device time (torch.profiler, median over --calls calls of b200_sixdof_trajectory_channels) for 4
     channels (speed, range, altitude, angle of attack) of 2^20 worlds x 16 samples and 2^22 x 4: the bytes it must move
     (10 planes read, 4 written, 8 B each per body and sample) over that time, against the copy probe;
  3. Exec.run per 10-tick telemetry cycle for the rocket set at 2^20 worlds, FAST math, ensemble=True with 0 and with
     4 channels (speed, range, pitch from vertical, angle of attack), the arms alternating --reps times, each one run()
     of --cycles cycles after a warm-up cycle;
  4. with --parent-lib (the parent commit's libb200_sixdof.so, built into a separate directory): the zero-channel path
     against the parent on the DESIGN section 6 shapes of trajectory_stats, trajectory_quantiles,
     trajectory_covariance, trajectory_histograms and the summary fold, parent and this tree's library alternating
     --reps times, with the median, min and max of the per-rep medians, and whether both give the same bits.
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
from group_stats_perf import parent_lib, reduce_into, ring, timed

# speed, range from the pad, altitude over a sphere, angle of attack (the velocity in the body frame's x axis)
KERNEL_CHANNELS = [(_lib.CHANNEL_NORM, 3, (10, 11, 12)), (_lib.CHANNEL_NORM, 2, (4, 5), (1.0, 2.0)),
                   (_lib.CHANNEL_NORM, 3, (4, 5, 6), (), (), 6.371e6),
                   (_lib.CHANNEL_AXIS_ANGLE, 3, (10,), (-1.0, 0.0, 0.0))]
PLANES_READ, PLANES_WRITTEN = 10, 4  # q (0-3), x (4-6), v (10-12); one plane per channel


def kernel_ms(ex, out, calls):
    """median device time of channel_kernel per trajectory_channels call, from torch.profiler"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ex.trajectory_channels(out.data_ptr())
        torch.cuda.synchronize()
    evs = [e for e in prof.profiler.kineto_results.events()
           if e.device_type() == DeviceType.CUDA and "channel_kernel" in e.name()]
    return float(np.median([(e.end_ns() - e.start_ns()) / 1e6 for e in evs])), len(evs)


def kernel_cases(probe, calls):
    out = []
    for M, S in ((1 << 20, 16), (1 << 22, 4)):
        ex, st = ring(M, 1, S)
        ex.set_channels(KERNEL_CHANNELS)
        with torch.cuda.stream(st):
            dst = torch.empty((S, M, 1, len(KERNEL_CHANNELS)), dtype=torch.float64, device="cuda")
            ex.trajectory_channels(dst.data_ptr())  # warm-up
            torch.cuda.synchronize()
            ms, n = kernel_ms(ex, dst, calls)
        nbytes = (PLANES_READ + PLANES_WRITTEN) * 8 * M * S
        gbs = nbytes / ms / 1e6
        out.append({"worlds": M, "samples": S, "channels": len(KERNEL_CHANNELS), "kernel_ms": ms, "kernels": n,
                    "bytes": nbytes, "gbs": gbs, "of_probe": gbs / probe})
        print(f"channel_kernel, {len(KERNEL_CHANNELS)} channels, {M} worlds x {S} samples: {ms * 1e3:8.1f} us "
              f"(median of {n}) for {nbytes / 1e6:.0f} MB = {gbs:6.0f} GB/s = {gbs / probe:.2f} of the copy probe")
        ex.close()
        del ex, dst
        torch.cuda.synchronize()
    return out


def exec_case(M, cycles, arm):
    w, sys_, params = rocket_world(M)
    kw = {}
    if arm == "4 channels":
        kw["channels"] = [el.Norm("speed", "world_vel", (3, 4, 5)), el.Norm("range", "world_pos", (4, 5)),
                          el.AxisAngle("pitch", (-1.0, 0.0, 0.0), (0.0, 0.0, 1.0)),
                          el.AxisAngle("aoa", (-1.0, 0.0, 0.0), ("world_vel", (3, 4, 5)))]
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=12.0, math="fast", n_worlds=M, world_params=params,
                 ensemble=True, **kw)
    del params
    ex.run(10)  # warm-up cycle
    n0 = len(ex._prof["execute_buffers"])
    t0 = time.perf_counter()
    ex.run(10 * cycles)
    wall = time.perf_counter() - t0
    per = ex._prof["execute_buffers"][n0:]
    assert len(per) == cycles
    ex.backend.close()
    del ex
    return {"arm": arm, "worlds": M, "cycles": cycles, "ms": per, "wall_ms_per_cycle": wall * 1e3 / cycles}


def regression(parent, calls, reps):
    cases = [(1 << 22, 1, 4, "stats", ()), (1 << 20, 1, 16, "stats", ()), (8, 1024, 64, "stats", ()),
             (1 << 20, 1, 16, "quantiles", (0.01, 0.5, 0.99)), (5000, 1, 16, "quantiles", tuple(np.linspace(0, 1, 16))),
             (1 << 20, 1, 16, "covariance", (4, 5, 6, 10, 11, 12)), (1 << 20, 1, 16, "covariance", tuple(range(25))),
             (1 << 20, 1, 16, "histograms", [(0, 6, 64, -4.0, 4.0)]), (1 << 20, 1, 16, "summary", ())]
    out = []
    for M, N, S, kind, k in cases:
        per = {"parent": [], "new": []}
        tables = {}
        for rep in range(reps):
            for arm in ("parent", "new"):
                ex, st = ring(M, N, S, parent if arm == "parent" else None)
                with torch.cuda.stream(st):
                    if kind == "summary":
                        ex.summary_begin(True, [(0, 6, False, 0.0)])
                        fold = lambda: _lib.check(ex._L.b200_sixdof_summary_add_trajectory(ex._h))  # noqa: E731
                        per[arm].append(timed(st, fold, calls)[0])
                        ext = np.empty((M, N, 25, 5))  # the parent's library has no channels to ask about
                        _lib.check(ex._L.b200_sixdof_extrema_download(ex._h, ext.ctypes.data, ext.nbytes))
                        tables[arm] = ext.tobytes() + ex.thresholds().tobytes()
                    else:
                        if kind == "stats":
                            args, rec = (), (N, 25, 5)
                        elif kind == "quantiles":
                            args, rec = ex._levels(k), (N, 25, len(k))
                        elif kind == "covariance":
                            args, rec = ex._selection(k), (N, 1 + len(k) + len(k) ** 2)
                        else:
                            args, row = ex._hist_specs(k)
                            rec = (row,)
                        dst = torch.empty((S,) + rec, dtype=torch.float64, device="cuda")
                        per[arm].append(timed(st, reduce_into(ex, kind, args, dst), calls)[0])
                        tables[arm] = dst.cpu().numpy().tobytes()
                        del dst
                ex.close()
                del ex
                torch.cuda.synchronize()
        label = f"{kind} {M} x {N} x {S}" + (f" ({len(k)})" if kind in ("quantiles", "covariance") else "")
        same = tables["parent"] == tables["new"]
        r = {"case": label, "same_bits": same}
        for arm, v in per.items():
            r[arm] = {"median_us": float(np.median(v)) * 1e3, "min_us": float(np.min(v)) * 1e3,
                      "max_us": float(np.max(v)) * 1e3}
        out.append(r)
        print(f"zero channels, {label:40s}: parent {r['parent']['median_us']:9.1f} us [{r['parent']['min_us']:.1f}, "
              f"{r['parent']['max_us']:.1f}], new {r['new']['median_us']:9.1f} us [{r['new']['min_us']:.1f}, "
              f"{r['new']['max_us']:.1f}], same bits: {same}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cycles", type=int, default=10)
    ap.add_argument("--worlds", type=int, default=1 << 20)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    if el.device_count() < 1:
        raise SystemExit("channels_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["kernel"] = kernel_cases(probe, a.calls)
    res["exec"] = []
    arms = ("0 channels", "4 channels")
    for rep in range(a.reps):
        for arm in arms:
            r = exec_case(a.worlds, a.cycles, arm)
            r["rep"] = rep
            res["exec"].append(r)
            print(f"Exec.run rocket set, {a.worlds} worlds, ensemble=True, {arm} rep {rep}: median "
                  f"{np.median(r['ms']):.3f} ms per 10-tick cycle [{np.min(r['ms']):.3f}, {np.max(r['ms']):.3f}] over "
                  f"{a.cycles} cycles ({r['wall_ms_per_cycle']:.3f} ms of run() wall time per cycle)")
    for arm in arms:
        v = np.concatenate([r["ms"] for r in res["exec"] if r["arm"] == arm])
        print(f"  {arm}: median {np.median(v):.3f} ms, min {np.min(v):.3f}, max {np.max(v):.3f}")
    if a.parent_lib:
        res["zero_channels"] = regression(parent_lib(a.parent_lib), a.calls, a.reps)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
