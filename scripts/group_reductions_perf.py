"""Grouped quantiles and covariance (b200_sixdof_trajectory_group_quantiles / _group_covariance, World.build(...,
groups=..., quantiles=..., covariance=...)) on one GPU.

    python scripts/group_reductions_perf.py [--parent-lib PATH] [--calls 10] [--reps 3] [--cycles 10] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query);
  2. with --parent-lib (the parent commit's libb200_sixdof.so, built into a separate directory): the ungrouped
     trajectory_quantiles and trajectory_covariance on the sort, block and radix routes and the chunked covariance,
     parent and this tree's library alternating --reps times, with the median, min and max of the per-rep medians, and
     whether both give the same bits;
  3. trajectory_quantiles (3 and 16 levels) and trajectory_covariance (p = 6 and 25) against their grouped entries at
     2^20 worlds x 1 entity x 16 samples and 2^22 x 1 x 4, with G = 1, 12, 256 and 1024 equal groups and one skewed split
     (half the worlds in one group, the rest in 63): the call time with CUDA events (median over --calls calls after
     warm-up), the ratio to the ungrouped call and the launches;
  4. Exec.run wall time per 10-tick telemetry cycle for the rocket set at 2^20 worlds: ensemble=True alone, then with
     groups=[12 equal groups], then also quantiles=(0.01, 0.5, 0.99) and covariance of world_pos[4:7] + world_vel[3:6];
     the arms alternate, --reps times.
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
from ensemble_perf import card, rocket_world
from group_stats_perf import parent_lib, reduce_into, ring, splits, timed

LEVELS = {3: (0.01, 0.5, 0.99), 16: tuple(np.linspace(0.0, 1.0, 16))}
SELECTIONS = {6: (4, 5, 6, 10, 11, 12), 25: tuple(range(25))}


def entry_args(ex, kind, k):
    """(entry, argument tuple, record shape after [samples, (G,)]) of a quantile call of k levels or a covariance call of
    p = k planes."""
    if kind == "quantiles":
        lv = ex._levels(LEVELS[k])
        return "quantiles", lv, (ex.n_entities, 25, k)
    sel = ex._selection(SELECTIONS[k])
    return "covariance", sel, (ex.n_entities, 1 + k + k * k)


def call_cases(calls):
    out = []
    for M, S in ((1 << 20, 16), (1 << 22, 4)):
        ex, st = ring(M, 1, S)
        with torch.cuda.stream(st):
            for kind, k in (("quantiles", 3), ("quantiles", 16), ("covariance", 6), ("covariance", 25)):
                entry, args, rec = entry_args(ex, kind, k)
                dst = torch.empty((S,) + rec, dtype=torch.float64, device="cuda")
                base = timed(st, reduce_into(ex, entry, args, dst), calls)
                label = f"trajectory_{entry} {'q' if kind == 'quantiles' else 'p'}={k}"
                out.append({"worlds": M, "samples": S, "call": label, "groups": "none", "ms": base})
                print(f"{label:28s} {M} x 1 x {S} samples, ungrouped    : {base[0] * 1e3:9.1f} us "
                      f"(min {base[1] * 1e3:.1f}, max {base[2] * 1e3:.1f})")
                for gname, sizes in splits(M).items():
                    ex.set_world_groups(sizes)
                    gdst = torch.empty((S, len(sizes)) + rec, dtype=torch.float64, device="cuda")
                    n0 = ex.timings()["kernel_launches"]
                    reduce_into(ex, f"group_{entry}", args, gdst)()
                    launches = ex.timings()["kernel_launches"] - n0
                    t = timed(st, reduce_into(ex, f"group_{entry}", args, gdst), calls)
                    if gname == "G=1":
                        assert torch.equal(gdst[:, 0].nan_to_num(-7.0), dst.nan_to_num(-7.0)), "G = 1 differs"
                    out.append({"worlds": M, "samples": S, "call": label, "groups": gname, "ms": t,
                                "launches": launches})
                    print(f"{'  grouped':28s} {gname:14s}: {t[0] * 1e3:9.1f} us (min {t[1] * 1e3:.1f}, max "
                          f"{t[2] * 1e3:.1f}), {t[0] / base[0]:.2f}x ungrouped, {launches} launches")
                    del gdst
                ex.set_world_groups([])
                del dst
        ex.close()
        torch.cuda.synchronize()
    return out


def exec_case(M, cycles, arm):
    w, sys_, params = rocket_world(M)
    kw = {}
    if arm != "alone":
        kw["groups"] = splits(M)["G=12"]
    if arm == "groups12+q+cov":
        kw["quantiles"] = LEVELS[3]
        kw["covariance"] = [("world_pos", (4, 5, 6)), ("world_vel", (3, 4, 5))]
    ex = w.build(sys_, simulation_rate=120.0, telemetry_rate=12.0, math="fast", n_worlds=M, world_params=params,
                 ensemble=True, **kw)
    ex.run(10)  # warm-up cycle
    t0 = time.perf_counter()
    ex.run(10 * cycles)
    wall = time.perf_counter() - t0
    r = {"arm": arm, "worlds": M, "cycles": cycles, "ms_per_cycle": wall * 1e3 / cycles}
    ex.backend.close()
    del ex
    return r


def regression(parent, calls, reps):
    cases = [(200, 1, 64, "quantiles", 16), (5000, 1, 16, "quantiles", 16), (1 << 20, 1, 16, "quantiles", 3),
             (1 << 22, 1, 4, "quantiles", 16), (8, 1024, 64, "covariance", 25), (1 << 20, 1, 16, "covariance", 6),
             (1 << 20, 1, 16, "covariance", 25)]
    out = []
    for M, N, S, kind, k in cases:
        per = {"parent": [], "new": []}
        tables = {}
        for rep in range(reps):
            for arm in ("parent", "new"):
                ex, st = ring(M, N, S, parent if arm == "parent" else None)
                with torch.cuda.stream(st):
                    entry, args, rec = entry_args(ex, kind, k)
                    dst = torch.empty((S,) + rec, dtype=torch.float64, device="cuda")
                    per[arm].append(timed(st, reduce_into(ex, entry, args, dst), calls)[0])
                    tables[arm] = dst.cpu().numpy()
                ex.close()
                del ex, dst
                torch.cuda.synchronize()
        label = f"trajectory_{kind} {'q' if kind == 'quantiles' else 'p'}={k} {M} x {N} x {S}"
        same = tables["parent"].tobytes() == tables["new"].tobytes()
        r = {"case": label, "same_bits": same}
        for arm, v in per.items():
            r[arm] = {"median_us": float(np.median(v)) * 1e3, "min_us": float(np.min(v)) * 1e3,
                      "max_us": float(np.max(v)) * 1e3}
        out.append(r)
        print(f"one group, {label:46s}: parent {r['parent']['median_us']:9.1f} us [{r['parent']['min_us']:.1f}, "
              f"{r['parent']['max_us']:.1f}], new {r['new']['median_us']:9.1f} us [{r['new']['min_us']:.1f}, "
              f"{r['new']['max_us']:.1f}], same bits: {same}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cycles", type=int, default=10)
    ap.add_argument("--worlds", type=int, default=1 << 20)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    if el.device_count() < 1:
        raise SystemExit("group_reductions_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    if a.parent_lib:
        res["one_group"] = regression(parent_lib(a.parent_lib), a.calls, a.reps)
    res["call"] = call_cases(a.calls)
    res["exec"] = []
    arms = ("alone", "groups12", "groups12+q+cov")
    for rep in range(a.reps):
        for arm in arms:
            r = exec_case(a.worlds, a.cycles, arm)
            r["rep"] = rep
            res["exec"].append(r)
            print(f"Exec.run rocket set, {a.worlds} worlds, ensemble=True, {arm:15s} rep {rep}: "
                  f"{r['ms_per_cycle']:.3f} ms per 10-tick cycle over {a.cycles} cycles")
    for arm in arms:
        v = [r["ms_per_cycle"] for r in res["exec"] if r["arm"] == arm]
        print(f"  {arm:15s}: median {np.median(v):.3f} ms, min {np.min(v):.3f}, max {np.max(v):.3f}")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
