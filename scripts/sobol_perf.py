"""Time the Sobol entry (b200_sixdof_outcome_[group_]sobol) and its host route.

    python scripts/sobol_perf.py [out.json]

Per size (2^20 and 2^22 worlds), d (4, 8, 23), resamples B (0, 100, 1000) and (outputs, groups) ((1, 1), (8, 1),
(8, 12)): the wall time of a call (host destination, median of 3 after a warm-up) and, from one torch.profiler run of
the call, the kernel time of the plane pass, the covariance (chunk and merge), the bootstrap (list and resample
kernels) and the finish.  The host route, for B = 0 and 100 with one output and one group: the outcome_values
download, then the numpy formulas and a bootstrap with the same draws (tests/test_outcome_sobol.py's restatement).
The card's name and power limit are read in the same run and printed with the numbers.
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import elodin_b200 as el
from elodin_b200 import _lib
from elodin_b200.executor import sobol_indices
from tests.test_outcome_sobol import cov_record, layout, ref_bootstrap

KERNELS = {"plane": ("sobol_plane",), "covariance": ("cov_chunk", "cov_merge"), "bootstrap": ("sobol_list", "sobol_boot"),
           "finish": ("sobol_finish",)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def handle(W, d, p, G, rng):
    N = W // (d + 2)
    X = layout(rng.uniform(size=(N, d)), rng.uniform(size=(N, d)))
    c = rng.normal(size=d)
    Y = np.column_stack([np.sin(X @ c + k) + X[:, 0] * X[:, -1] for k in range(p)])
    ex = el.B200Exec(1, Y.shape[0], 0.01, None, [], "rk4", "fast")
    ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, np.ascontiguousarray(Y[:, k])) for k in range(p)])
    if G > 1:
        n = [N // G + (g < N % G) for g in range(G)]
        ex.set_world_groups([k * (d + 2) for k in n])
    return ex, Y


def kernel_ms(call):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in KERNELS}
    for e in prof.key_averages():
        for k, names in KERNELS.items():
            if any(n in e.key for n in names):
                out[k] += e.device_time_total / 1e3  # us -> ms
    return out


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    torch.cuda.init()
    info = card()
    print(f"card: {info}")
    rng = np.random.default_rng(0)
    results = []
    for W in (1 << 20, 1 << 22):
        for d in (4, 8, 23):
            W_d = W // (d + 2) * (d + 2)
            for p, G in ((1, 1), (8, 1), (8, 12)):
                ex, Y = handle(W_d, d, p, G, rng)
                fn = ex.outcome_group_sobol if G > 1 else ex.outcome_sobol
                for B in (0, 100, 1000):
                    call = lambda: fn(list(range(p)), d, B, 1)
                    call()
                    times = []
                    for _ in range(3):
                        t0 = time.perf_counter()
                        call()
                        times.append((time.perf_counter() - t0) * 1e3)
                    k = kernel_ms(call)
                    r = {"worlds": W_d, "d": d, "B": B, "outputs": p, "groups": G, "call_ms": float(np.median(times)),
                         **{f"{n}_ms": v for n, v in k.items()}}
                    if p == 1 and G == 1 and B <= 100:
                        t0 = time.perf_counter()
                        y = ex.outcome_values()[:, 0]
                        rec = cov_record(y, d)
                        sobol_indices(rec, d)
                        if B:
                            ref_bootstrap(y, d, B, 1, rec[1:d + 3])
                        r["host_ms"] = (time.perf_counter() - t0) * 1e3
                    print(json.dumps(r), flush=True)
                    results.append(r)
                del ex
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump({"card": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
