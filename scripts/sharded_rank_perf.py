"""World-sharded rank correlation (b200_sixdof_sharded_ranks_*) against the unsharded call and the gather route, on one GPU.

    python scripts/sharded_rank_perf.py [--worlds 1048576 4194304] [--reps 3] [--out results.json]

Prints, as one run:
  1. the card's name, power limit and max SM clock (nvidia-smi, read-only query);
  2. for every --worlds M and selection (4 and 25 continuous outcomes, and one outcome of 4 distinct values), on
     handles whose outcomes are VALUES planes:
       unsharded  outcome_rank_correlation on one handle holding the M worlds: call time (host clock around the call,
                  which ends in a stream synchronise) and reads per task;
       sharded    the protocol at R = 1, 2 and 4 ranks simulated on the one GPU (R handles holding consecutive world
                  ranges, driven in lockstep; each round's partials are device buffers summed with one torch add per
                  extra rank, as an all-reduce would leave them), ending with every rank's covariance records merged on
                  the host into rho (with one outcome, the ranks downloaded instead, as the other routes return them):
                  the whole call's time, the rounds, the exchanges, the total and largest round bytes
                  and the reads per task.  The ranks of every rank are checked bit for bit against the unsharded rows
                  once, and rho within 1e-12 of the unsharded rho;
       gather     every rank's outcome values downloaded and gathered into one handle, then ranked there (the route
                  without the protocol: per-world traffic to one place): the whole time.
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
from elodin_b200 import _lib
from elodin_b200.executor import merge_covariance, rank_correlation
from ensemble_perf import card

CAP = 32 << 20  # the largest round, in bytes (include/b200_sixdof.h)


def values_handle(v):
    ex = el.B200Exec(1, v.shape[0], 0.01, None, [], "rk4", "fast")
    ex.set_outcomes([(_lib.OUTCOME_VALUES, 0, 0, 0, 0, np.ascontiguousarray(v[:, j])) for j in range(v.shape[1])])
    return ex


def selection(M, kind, seed=1):
    rng = np.random.default_rng(seed)
    if kind == "4 values":
        return rng.integers(0, 4, (M, 1)).astype(np.float64)
    p = int(kind.split()[0])
    x = rng.normal(0.0, 1.0, (M, p))
    x[:, 1:] += 0.5 * x[:, :1]  # correlated outcomes
    return x


def sharded(exs, planes, ranks=False):
    """One sharded call over the handles: (rho or None, every rank's ranks or None, round sizes)."""
    R = len(exs)
    bound = [ex.sharded_ranks_begin(planes, False, r, R) for r, ex in enumerate(exs)][0]
    bufs = [torch.zeros(bound // 4, dtype=torch.int32, device="cuda") for _ in exs]
    sizes, n, red = [], 0, None
    while True:
        got = [ex.sharded_ranks_round(red, n, b) for ex, b in zip(exs, bufs)]
        n = got[0]
        assert len(set(got)) == 1
        sizes.append(n)
        if n == 0:
            break
        red = bufs[0][: n // 4].clone()
        for b in bufs[1:]:
            red += b[: n // 4]
        torch.cuda.synchronize()
    out = [ex.sharded_ranks_end(ranks, True) for ex in exs]
    rho = rank_correlation(merge_covariance([c for _, c in out]), len(planes))[0] if len(planes) > 1 else None
    return rho, [r for r, _ in out], sizes


def timed(fn, reps):
    fn()  # warm-up
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, nargs="+", default=[1 << 20, 1 << 22])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the figures as JSON to this file")
    a = ap.parse_args()
    if el.device_count() < 1:
        raise SystemExit("sharded_rank_perf.py needs a CUDA device")
    res = {"card": card(), "cases": []}
    print("card (name, power.limit, clocks.max.sm):", res["card"])
    for M in a.worlds:
        for kind in ("4 continuous", "25 continuous", "4 values"):
            v = selection(M, kind)
            p = v.shape[1]
            planes = list(range(p))
            one = values_handle(v)
            call = (lambda: one.outcome_rank_correlation(planes)) if p > 1 else (lambda: one.outcome_ranks(planes))
            case = {"worlds": M, "outcomes": kind,
                    "unsharded": {"call_ms": timed(call, a.reps), "reads": one.rank_reads()}}
            want_rho = one.outcome_rank_correlation(planes) if p > 1 else None
            want = one.outcome_ranks(planes)
            one.close()
            print(M, kind, "unsharded:", case["unsharded"])
            for R in (1, 2, 4):
                bounds = [M * k // R for k in range(R + 1)]
                exs = [values_handle(v[bounds[k]:bounds[k + 1]]) for k in range(R)]
                rho, ranks, sizes = sharded(exs, planes, ranks=True)
                for k in range(R):
                    assert ranks[k].tobytes() == want[bounds[k]:bounds[k + 1]].tobytes(), f"R = {R}: not the unsharded ranks"
                if p > 1:
                    assert np.allclose(rho, want_rho, atol=1e-12, rtol=0, equal_nan=True), f"R = {R}: rho"
                # one outcome: the unsharded and gather routes return the ranks, so this call downloads them too
                ms = timed(lambda: sharded(exs, planes, ranks=p == 1), a.reps)
                rounds = sizes[:-1]
                r = {"call_ms": ms, "rounds": len(rounds), "exchanges": sum(1 for n in rounds if n < CAP),
                     "round_bytes_total": int(sum(rounds)), "round_bytes_max": int(max(rounds)),
                     "reads": exs[0].rank_reads()}

                def gather():
                    vals = np.concatenate([ex.outcome_values() for ex in exs])
                    h = values_handle(vals)
                    h.outcome_rank_correlation(planes) if p > 1 else h.outcome_ranks(planes)
                    h.close()

                r["gather_ms"] = timed(gather, a.reps)
                case[f"sharded_R{R}"] = r
                print(M, kind, f"R={R}:", r)
                for ex in exs:
                    ex.close()
            res["cases"].append(case)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
