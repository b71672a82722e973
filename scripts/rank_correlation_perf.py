"""Rank correlation (b200_sixdof_outcome_[group_]rank_correlation and _ranks) on one GPU, against the host route.

    python scripts/rank_correlation_perf.py [--calls 5] [--out r.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query) and the device copy probe;
  2. for 2^20 and 2^22 worlds, n_p = 4, 8 and 25 outcomes (host values: continuous normal values, a heavily tied plane
     of 4 distinct values, the way dwell row counts and saturated ticks look, or heavy-tailed Cauchy values with one
     1e300 outlier) and G = 1, 12 and 256 groups: the wall time of one correlation call and of one rank call into
     device memory (each call ends in a stream synchronise, so a host clock measures it; median over the calls), the
     plane reads per task the rank call reports, and the bytes the rank pass moves (the completeness read, the reads of
     the plane and the write of the rank plane, 8 B per world, outcome and pass) over the rank call's time, against the
     copy probe;
  3. for G = 1, the host route for the same answer: outcome_values into pinned memory, then scipy.stats.rankdata per
     outcome over the complete worlds and np.corrcoef; its rho must be within 1e-12 of the device's.
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

SIZES = (1 << 20, 1 << 22)
PLANES = (4, 8, 25)
DATA = ("continuous", "4-valued", "heavy-tailed")


def values_of(M, P, data, seed=3):
    rng = np.random.default_rng(seed)
    if data == "4-valued":
        return rng.integers(0, 4, (M, P)).astype(np.float64)
    if data == "heavy-tailed":
        v = rng.standard_cauchy((M, P))
        v[rng.integers(0, M), :] = 1e300
        return v
    v = rng.normal(0.0, 1.0, (M, P)) * rng.uniform(0.1, 100.0, (1, P))
    v[rng.random((M, P)) < 0.01] = np.nan
    return v


def host_rho(values):
    """The host route's rank correlation matrix over the complete worlds."""
    import scipy.stats

    x = values[np.all(np.isfinite(values), axis=1)]
    ranks = np.column_stack([scipy.stats.rankdata(x[:, j], method="average") for j in range(x.shape[1])])
    return np.corrcoef(ranks, rowvar=False)


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
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    import torch

    import elodin_b200 as el
    from elodin_b200 import _lib
    from ensemble_perf import card

    if el.device_count() < 1 or not torch.cuda.is_available():
        raise SystemExit("rank_correlation_perf.py needs a CUDA device")
    res = {"card": card()}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    probe = float(_lib.lib().b200_probe_copy_gbs(0, 1 << 30, 20))
    res["copy_probe_gbs"] = probe
    print(f"b200_probe_copy_gbs: {probe:.0f} GB/s")
    res["cases"] = []
    for M in SIZES:
        for data in DATA:
            values = values_of(M, max(PLANES), data)
            ex = el.B200Exec(1, M, 0.01, None, [], "rk4", "fast")
            ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, np.ascontiguousarray(values[:, p]))
                             for p in range(values.shape[1])])
            dev = torch.empty(M * max(PLANES), dtype=torch.float64, device="cuda")
            for P in PLANES:
                planes = list(range(P))
                host = None
                for G in (1, 12, 256):
                    sizes = [M // G + (g < M % G) for g in range(G)]
                    if G > 1:
                        ex.set_world_groups(sizes)
                    corr = ex.outcome_group_rank_correlation if G > 1 else ex.outcome_rank_correlation
                    name = "group_ranks" if G > 1 else "ranks"
                    corr_ms = median_ms(lambda: corr(planes), a.calls)
                    ranks_ms = median_ms(lambda: ex._reduce(name, "outcome", ex._selection(planes), (M, P),
                                                            dev.data_ptr()), a.calls)
                    reads = ex.rank_reads()
                    moved = (1 + reads + 1) * M * P * 8
                    row = {"worlds": M, "P": P, "data": data, "G": G, "corr_ms": corr_ms, "ranks_ms": ranks_ms,
                           "reads": reads, "of_probe": moved / (ranks_ms * 1e-3) / 1e9 / probe}
                    line = (f"M=2^{M.bit_length() - 1} n_p={P:2d} {data:12s} G={G:3d}: correlation {corr_ms:8.2f} ms, "
                            f"ranks {ranks_ms:8.2f} ms, {reads:.2f} reads, {row['of_probe']:.2f} of the probe")
                    if G == 1:
                        buf = el.pinned_empty((M, ex.n_outcomes))
                        t0 = time.perf_counter()
                        _lib.check(ex._L.b200_sixdof_outcome_values(ex._h, ctypes.c_void_p(buf.ctypes.data), buf.nbytes))
                        host = host_rho(buf[:, :P])
                        row["host_ms"] = (time.perf_counter() - t0) * 1e3
                        el.pinned_free(buf)
                        rho = corr(planes)[1:].reshape(P, P)
                        assert np.allclose(rho, host, atol=1e-12, rtol=0, equal_nan=True), (M, P, data)
                        line += f"; host route {row['host_ms']:.0f} ms, same rho to 1e-12"
                    print(line, flush=True)
                    res["cases"].append(row)
                ex.set_world_groups([])
            ex.close()
            del values, dev
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
