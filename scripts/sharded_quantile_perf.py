"""World-sharded quantiles (b200_sixdof_sharded_quantiles_*) against the unsharded trajectory quantiles, on one GPU.

    python scripts/sharded_quantile_perf.py [--worlds 1048576] [--samples 16] [--reps 3] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query);
  2. trajectory_quantiles at --worlds rocket worlds x 1 entity x --samples samples x 25 planes x 3 levels: call time
     (host clock around the call, which ends in a stream synchronise), summed kernel time (torch.profiler), reads;
  3. the sharded protocol over the same worlds at R = 1 (the sum is the identity), 2 and 4 ranks simulated on the one
     GPU (R handles holding consecutive world ranges, driven in lockstep; each round's partials are device buffers
     summed with one torch add per extra rank, as an all-reduce would leave them): the whole call's time, the summed
     kernel time of every rank, the rounds per slice, the reads, the bytes of every round and the host time per round
     (every rank's round call plus the sum).  Every table is checked bit for bit against the unsharded one.
Times across GPUs (NVLink all-reduce of the rounds) cannot be measured on one GPU and are not reported.
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
from ensemble_perf import card

LEVELS = (0.01, 0.5, 0.99)
HIST_BYTES = ((1 << 14) + 64) * 4  # a triple's bytes in a histogram round


def rocket_handles(M, S, bounds):
    """One handle per world range [bounds[k], bounds[k + 1]) of the same rocket campaign, stepped S ticks."""
    rng = np.random.default_rng(1)
    pos = np.zeros((M, 1, 7))
    pos[..., 3] = 1.0
    pos[..., 6] = rng.uniform(0.0, 10.0, (M, 1))
    vel = np.zeros((M, 1, 6))
    vel[..., 3:] = rng.normal(0.0, 5.0, (M, 1, 3))
    ine = np.tile(np.array([0.1, 1.0, 1.0, 0, 0, 0, 3.0]), (M, 1, 1))
    thrust = 88.4 * rng.uniform(0.8, 1.2, (M, 1, 1))
    wind = np.concatenate([rng.normal(0.0, 2.0, (M, 1, 1)), np.zeros((M, 1, 2))], -1)
    out = []
    for a, b in zip(bounds[:-1], bounds[1:]):
        effs = [el.GravityConst((0.0, 0.0, -9.81)), el.ThrustBody((-1.0, 0.0, 0.0), "thrust"),
                el.DragQuadratic(0.6125, 0.0025, "wind")]
        ex = el.B200Exec(1, b - a, 1.0 / 120.0, None, effs, "rk4", "exact", trajectory_every=1, trajectory_capacity=S,
                         trajectory_full=True)
        ex.set_state(pos[a:b], vel[a:b], ine[a:b], thrust=thrust[a:b], wind=wind[a:b])
        ex.step(S)
        out.append(ex)
    return out


def kernel_ms(call):
    """summed device time of the quantile kernels of one call, from torch.profiler"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    return sum((e.end_ns() - e.start_ns()) for e in prof.profiler.kineto_results.events()
               if e.device_type() == DeviceType.CUDA and "quantile" in e.name()) / 1e6


def sharded(exs):
    """One sharded call over the handles: (tables, round sizes, host seconds per round)."""
    bound = [ex.sharded_quantiles_begin(LEVELS, "ring") for ex in exs][0]
    bufs = [torch.zeros(max(bound // 4, 1), dtype=torch.int32, device="cuda") for _ in exs]
    sizes, times, n, red = [], [], 0, None
    while True:
        t0 = time.perf_counter()
        got = [ex.sharded_quantiles_round(red, n, b) for ex, b in zip(exs, bufs)]
        n = got[0]
        assert len(set(got)) == 1
        if n:
            red = bufs[0][: n // 4].clone()
            for b in bufs[1:]:
                red += b[: n // 4]
            torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        sizes.append(n)
        if n == 0:
            break
    return [ex.sharded_quantiles_end() for ex in exs], sizes, times


def per_slice(sizes):
    out = []
    for n in sizes[:-1]:
        if n < HIST_BYTES:
            out.append(0)
        out[-1] += 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, default=1 << 20)
    ap.add_argument("--samples", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    if el.device_count() < 1:
        raise SystemExit("sharded_quantile_perf.py needs a CUDA device")
    M, S = a.worlds, a.samples
    res = {"card": card(), "worlds": M, "samples": S, "planes": 25, "levels": len(LEVELS)}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    one = rocket_handles(M, S, [0, M])[0]
    want = one.trajectory_quantiles(LEVELS)  # warm-up
    calls = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        one.trajectory_quantiles(LEVELS)
        calls.append((time.perf_counter() - t0) * 1e3)
    res["unsharded"] = {"call_ms": float(np.median(calls)), "kernel_ms": kernel_ms(lambda: one.trajectory_quantiles(LEVELS)),
                        "reads": one.quantile_reads()}
    print("unsharded:", res["unsharded"])
    one.close()
    for R in (1, 2, 4):
        exs = rocket_handles(M, S, [M * k // R for k in range(R + 1)])
        tabs, sizes, times = sharded(exs)  # warm-up
        assert all(t.tobytes() == want.tobytes() for t in tabs), f"R = {R}: not the unsharded table"
        walls = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            tabs, sizes, times = sharded(exs)
            walls.append((time.perf_counter() - t0) * 1e3)
        assert all(t.tobytes() == want.tobytes() for t in tabs), f"R = {R}: not the unsharded table"
        r = {"ranks": R, "call_ms": float(np.median(walls)), "kernel_ms_all_ranks": kernel_ms(lambda: sharded(exs)),
             "rounds": len(sizes) - 1, "rounds_per_slice": per_slice(sizes), "reads": exs[0].quantile_reads(),
             "round_bytes": sizes[:-1], "host_ms_per_round": [round(t * 1e3, 3) for t in times]}
        print(f"sharded R={R}:", r)
        res[f"sharded_R{R}"] = r
        for ex in exs:
            ex.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
