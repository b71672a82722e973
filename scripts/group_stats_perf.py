"""Grouped ensembles (b200_sixdof_trajectory_group_stats / _group_histograms, World.build(..., groups=...)) on one GPU.

    python scripts/group_stats_perf.py [--parent-lib PATH] [--calls 40] [--reps 3] [--cycles 20] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query) and the device copy probe;
  2. trajectory_stats against trajectory_group_stats at 2^20 worlds x 1 entity x 16 samples x 25 planes and at 2^22 x 1
     x 4, with G = 1, 12, 256 and 1024 equal groups and one skewed split (half the worlds in one group, the rest in 63):
     the call time with CUDA events (median over --calls calls after warm-up), the planes' bytes over that time against
     the copy probe, and the ratio to the ungrouped call;
  3. the same for trajectory_histograms against trajectory_group_histograms, with 1 spec of 64 bins and one 64 x 64 2D
     spec;
  4. Exec.run wall time per 10-tick telemetry cycle for the rocket set at 2^20 worlds: ensemble=True alone, with one 2D
     histogram, and with the histogram and groups=[12 equal groups]; the arms alternate, --reps times;
  5. with --parent-lib (the parent commit's libb200_sixdof.so, built into a separate directory): the ungrouped
     trajectory_stats on the DESIGN section 6 shapes and trajectory_histograms on one shape, parent and this tree's
     library alternating --reps times, with the median, min and max of the per-rep medians, and whether both give the
     same bits.
"""
import argparse
import ctypes
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

HIST_SETS = {"1x64": [(0, 6, 64, -4.0, 4.0)], "2d64x64": [(0, (4, 5), (64, 64), (-4.0, -4.0), (4.0, 4.0))]}


def splits(M):
    eq = lambda G: [M // G + (1 if g < M % G else 0) for g in range(G)]  # noqa: E731
    rest = M - M // 2
    return {"G=1": eq(1), "G=12": eq(12), "G=256": eq(256), "G=1024": eq(1024),
            "skew 1/2 + 63": [M // 2] + [rest // 63 + (1 if g < rest % 63 else 0) for g in range(63)]}


def ring(M, N, S, L=None):
    """A handle with a full ring of S samples of M worlds x N entities (spread data, FAST free bodies), on its own
    stream; with L (a loaded library) the handle lives in that library."""
    st = torch.cuda.Stream()
    old = _lib._lib
    if L is not None:
        _lib._lib = L
    try:
        ex = el.B200Exec(N, M, 1e-3, None, [], "rk4", "fast", trajectory_every=1, trajectory_capacity=S,
                         trajectory_full=True)
    finally:
        _lib._lib = old
    ex.set_stream(st.cuda_stream)
    rng = np.random.default_rng(1)
    pos = np.zeros((M, N, 7))
    pos[..., 3] = 1.0
    pos[..., 4:] = rng.normal(0.0, 1.5, (M, N, 3))
    vel = rng.normal(0.0, 1.0, (M, N, 6))
    ine = np.tile(np.array([1.0, 1.0, 1.0, 0, 0, 0, 1.0]), (M, N, 1))
    ex.set_state(pos, vel, ine)
    del pos, vel, ine
    ex.step(S)
    ex.sync()
    return ex, st


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


def reduce_into(ex, entry, args, dst):
    fn = getattr(ex._L, f"b200_sixdof_trajectory_{entry}")
    return lambda: _lib.check(fn(ex._h, *args, ctypes.c_void_p(dst.data_ptr()), dst.numel() * 8))


def call_cases(probe, calls):
    out = []
    for M, S in ((1 << 20, 16), (1 << 22, 4)):
        ex, st = ring(M, 1, S)
        nbytes = M * 25 * S * 8
        with torch.cuda.stream(st):
            for kind in ("stats", "histograms"):
                for hname, specs in (HIST_SETS.items() if kind == "histograms" else [("", None)]):
                    args, row = ex._hist_specs(specs) if specs else ((), None)
                    rec = (1, 25, 5) if specs is None else (row,)
                    read = nbytes if specs is None else M * 8 * S * sum(len(np.atleast_1d(s[1])) for s in specs)
                    dst = torch.empty((S,) + rec, dtype=torch.float64, device="cuda")
                    base = timed(st, reduce_into(ex, kind, args, dst), calls)
                    label = f"trajectory_{kind} {hname}".strip()
                    r = {"worlds": M, "samples": S, "call": label, "groups": "none", "ms": base, "bytes": read}
                    out.append(r)
                    print(f"{label:32s} {M} x 1 x {S} samples, ungrouped    : {base[0] * 1e3:8.1f} us "
                          f"(min {base[1] * 1e3:.1f}, max {base[2] * 1e3:.1f}) = {read / base[0] / 1e6:6.0f} GB/s "
                          f"= {read / base[0] / 1e6 / probe:.2f} of the copy probe")
                    for gname, sizes in splits(M).items():
                        ex.set_world_groups(sizes)
                        gdst = torch.empty((S, len(sizes)) + rec, dtype=torch.float64, device="cuda")
                        n0 = ex.timings()["kernel_launches"]
                        reduce_into(ex, f"group_{kind}", args, gdst)()
                        launches = ex.timings()["kernel_launches"] - n0
                        t = timed(st, reduce_into(ex, f"group_{kind}", args, gdst), calls)
                        if gname == "G=1":
                            assert torch.equal(gdst[:, 0].nan_to_num(-7.0), dst.nan_to_num(-7.0)), "G = 1 differs"
                        out.append({"worlds": M, "samples": S, "call": label, "groups": gname, "ms": t, "bytes": read,
                                    "launches": launches})
                        print(f"{'  grouped':32s} {gname:14s}: {t[0] * 1e3:8.1f} us (min {t[1] * 1e3:.1f}, max "
                              f"{t[2] * 1e3:.1f}) = {read / t[0] / 1e6:6.0f} GB/s = {read / t[0] / 1e6 / probe:.2f} of "
                              f"the copy probe, {t[0] / base[0]:.2f}x ungrouped, {launches} launches")
                    ex.set_world_groups([])
        ex.close()
        torch.cuda.synchronize()
    return out


def exec_case(M, cycles, arm):
    w, sys_, params = rocket_world(M)
    kw = {}
    if arm != "alone":
        kw["histograms"] = [el.Histogram("rocket.world_pos", (4, 5), range=((-100.0, 400.0), (-50.0, 50.0)), bins=(64, 64))]
    if arm == "hist2d+groups12":
        kw["groups"] = splits(M)["G=12"]
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


def parent_lib(path):
    """The parent's library with the argtypes of this tree's binding for every symbol it has."""
    new, L = _lib.lib(), ctypes.CDLL(os.path.abspath(path))
    for name in _lib.SYMBOLS:
        if hasattr(L, name) and hasattr(new, name):
            f, g = getattr(L, name), getattr(new, name)
            f.argtypes, f.restype = g.argtypes, g.restype
    return L


def regression(parent, calls, reps):
    cases = [(1 << 22, 1, 4, None), (1 << 20, 1, 16, None), (8, 1024, 64, None), (1 << 20, 1, 16, "1x64")]
    out = []
    for M, N, S, hname in cases:
        per = {"parent": [], "new": []}
        tables = {}
        for rep in range(reps):
            for arm in ("parent", "new"):
                ex, st = ring(M, N, S, parent if arm == "parent" else None)
                with torch.cuda.stream(st):
                    if hname is None:
                        dst = torch.empty((S, N, 25, 5), dtype=torch.float64, device="cuda")
                        fn = reduce_into(ex, "stats", (), dst)
                    else:
                        args, row = ex._hist_specs(HIST_SETS[hname])
                        dst = torch.empty((S, row), dtype=torch.float64, device="cuda")
                        fn = reduce_into(ex, "histograms", args, dst)
                    per[arm].append(timed(st, fn, calls)[0])
                    tables[arm] = dst.cpu().numpy()
                ex.close()
                del ex, dst
                torch.cuda.synchronize()
        label = f"trajectory_{'stats' if hname is None else 'histograms ' + hname} {M} x {N} x {S}"
        same = tables["parent"].tobytes() == tables["new"].tobytes()
        r = {"case": label, "same_bits": same}
        for arm, v in per.items():
            r[arm] = {"median_us": float(np.median(v)) * 1e3, "min_us": float(np.min(v)) * 1e3,
                      "max_us": float(np.max(v)) * 1e3}
        out.append(r)
        print(f"one group, {label:44s}: parent {r['parent']['median_us']:8.1f} us [{r['parent']['min_us']:.1f}, "
              f"{r['parent']['max_us']:.1f}], new {r['new']['median_us']:8.1f} us [{r['new']['min_us']:.1f}, "
              f"{r['new']['max_us']:.1f}], same bits: {same}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cycles", type=int, default=20)
    ap.add_argument("--worlds", type=int, default=1 << 20)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    if el.device_count() < 1:
        raise SystemExit("group_stats_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    if a.parent_lib:
        res["one_group"] = regression(parent_lib(a.parent_lib), a.calls, a.reps)
    res["call"] = call_cases(probe, a.calls)
    res["exec"] = []
    arms = ("alone", "hist2d", "hist2d+groups12")
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
