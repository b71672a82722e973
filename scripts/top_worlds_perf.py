"""Worst worlds (b200_sixdof_outcome_[group_]top_worlds) on one GPU, against the host route.

    python scripts/top_worlds_perf.py [--calls 10] [--out r.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query) and the device copy probe;
  2. for 2^20 and 2^22 worlds with P = 8 and P = 25 outcomes (host values: continuous normal values, or a heavily
     tied plane of 4 distinct values, the way dwell row counts and saturated ticks look), G = 1, 12 and 256 groups and
     k = 16 and 1024 (both directions): the wall time of one call (each call ends in a stream synchronise, so a host
     clock measures it; median over the calls), the plane reads per task the call reports, and the bytes those reads
     move (8 B per world, outcome and read) over the call time, against the copy probe;
  3. for G = 1, the host route for the same answers: outcome_values into pinned memory, then np.lexsort per outcome;
     the records of both routes must be equal bit for bit.
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np

CASES = [(1 << 20, 8), (1 << 20, 25), (1 << 22, 8), (1 << 22, 25)]


def values_of(M, P, tied, seed=3):
    rng = np.random.default_rng(seed)
    if tied:
        return rng.integers(0, 4, (M, P)).astype(np.float64)
    v = rng.normal(0.0, 1.0, (M, P)) * rng.uniform(0.1, 100.0, (1, P))
    v[rng.random((M, P)) < 0.01] = np.nan
    return v


def host_records(values, k, largest):
    """[P, 1 + 2k]: the host route's records (numpy's totalOrder restatement and lexsort)."""
    M, P = values.shape
    out = np.empty((P, 1 + 2 * k))
    world = np.arange(M)
    for p in range(P):
        x = values[:, p]
        fin = np.isfinite(x)
        u = x[fin].view(np.uint64)
        key = np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))
        order = np.lexsort((world[fin], ~key if largest else key))[:k]
        out[p] = np.nan
        out[p, 0] = fin.sum()
        out[p, 1 + k:] = -1.0
        out[p, 1:1 + order.size] = x[fin][order]
        out[p, 1 + k:1 + k + order.size] = world[fin][order]
    return out


def bits(x):
    x = np.array(x)
    x[np.isnan(x)] = np.nan
    return x.view(np.uint64)


def median_ms(call, calls):
    call()
    t = []
    for _ in range(calls):
        t0 = time.perf_counter()
        call()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    import elodin_b200 as el
    from elodin_b200 import _lib
    from ensemble_perf import card

    if el.device_count() < 1:
        raise SystemExit("top_worlds_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["cases"] = []
    for M, P in CASES:
        for tied in (False, True):
            values = values_of(M, P, tied)
            ex = el.B200Exec(1, M, 0.01, None, [], "rk4", "fast")
            ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, values[:, p]) for p in range(P)])
            planes = list(range(P))
            # the host route: the per-world download into pinned memory, then numpy
            buf = el.pinned_empty((M, P))
            t0 = time.perf_counter()
            _lib.check(ex._L.b200_sixdof_outcome_values(ex._h, ctypes.c_void_p(buf.ctypes.data), buf.nbytes))
            dl_ms = (time.perf_counter() - t0) * 1e3
            host = {}
            for largest in (True, False):
                t0 = time.perf_counter()
                host[largest] = host_records(buf, 1024, largest)
                host[(largest, "ms")] = (time.perf_counter() - t0) * 1e3 + dl_ms
            el.pinned_free(buf)
            for G in (1, 12, 256):
                sizes = [M // G + (g < M % G) for g in range(G)]
                if G > 1:
                    ex.set_world_groups(sizes)
                for k in (16, 1024):
                    for largest in (True, False):
                        fn = ex.outcome_group_top_worlds if G > 1 else ex.outcome_top_worlds
                        ms = median_ms(lambda: fn(planes, k, largest), a.calls)
                        reads = ex.top_worlds_reads()
                        moved = reads * M * P * 8
                        row = {"worlds": M, "P": P, "data": "tied" if tied else "continuous", "G": G, "k": k,
                               "largest": largest, "call_ms": ms, "reads": reads,
                               "of_probe": moved / (ms * 1e-3) / 1e9 / probe}
                        line = (f"M=2^{M.bit_length() - 1} P={P} {row['data']:10s} G={G:3d} k={k:4d} "
                                f"{'largest ' if largest else 'smallest'}: {ms:8.2f} ms, {reads:.2f} reads, "
                                f"{row['of_probe']:.2f} of the probe")
                        if G == 1:
                            got = fn(planes, k, largest)
                            want = host[largest][:, np.r_[0:1 + k, 1 + 1024:1 + 1024 + k]]
                            assert np.array_equal(bits(got), bits(want)), (M, P, tied, k, largest)
                            row["host_ms"] = host[(largest, "ms")]
                            line += f"; host route {row['host_ms']:.0f} ms (download {dl_ms:.0f} ms), same records"
                        print(line, flush=True)
                        res["cases"].append(row)
            ex.close()
            del values
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
