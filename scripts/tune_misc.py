"""Secondary kernels on one GPU (tuning build for the EXACT shapes: make -C elodin_b200/csrc TUNE=1):
  * EXACT body kernel launch shapes (B200_EXACT_CFG re-read per launch in a tuning build), 2^20 worlds
  * n-body 1024: pair kernel at M = 1 / 8 / 64 worlds, FP64-pipe fraction against b200_probe_fp64_gflops
Prints one JSON row per measurement and writes gpurun_out/tune_misc.json."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import elodin_b200 as el, bench
from elodin_b200 import _lib

L = _lib.lib()
fp64 = L.b200_probe_fp64_gflops(0, 20000)
st = torch.cuda.Stream()
rows = []

def timed(ex, ticks, warm, reps=3):
    ex.set_stream(st.cuda_stream)
    best = 1e30
    with torch.cuda.stream(st):
        ex.step(warm); torch.cuda.synchronize()
        for _ in range(reps):
            a, b = torch.cuda.Event(True), torch.cuda.Event(True)
            a.record(st); ex.step(ticks); b.record(st); torch.cuda.synchronize()
            best = min(best, a.elapsed_time(b) / ticks)
    return best

M = 1 << 20
pos, vel, ine = bench.synth_world(M, 1)
for cfg in [3, 12, 1, 0, 4, 5, 6, 7, 8, 9, 10, 11]:
    os.environ["B200_EXACT_CFG"] = str(cfg)
    ex = el.B200Exec(1, M, 1e-3, None, [], "rk4", "exact")
    ex.set_state(pos, vel, ine)
    ms = timed(ex, 10, 3)
    ex.close()
    rows.append({"what": "exact_body", "cfg": cfg, "us_per_tick": ms * 1e3, "entity_steps_per_s": M / (ms * 1e-3)})
    print(json.dumps(rows[-1]), flush=True)
os.environ["B200_EXACT_CFG"] = "3"

N = 1024
rng = np.random.default_rng(7)
g = el.GravityEdges("softened", k_squared=2.9591220828e-4 / 86400.0 ** 2, softening=1e-10, edges=el.all_pairs_edges(N))
for Mw in (1, 8, 64, 296):
    p = np.zeros((Mw, N, 7)); p[..., 3] = 1.0; p[..., 4:] = rng.uniform(-30, 30, (Mw, N, 3))
    v = np.zeros((Mw, N, 6)); v[..., 3:] = rng.normal(0, 1e-7, (Mw, N, 3))
    m = 10 ** rng.uniform(-10, -3, (Mw, N)); m[:, 0] = 1.0
    I = np.zeros((Mw, N, 7)); I[..., :3] = m[..., None]; I[..., 6] = m
    for math in ("fast", "exact"):
        if math == "exact" and Mw > 8:
            continue
        ex = el.B200Exec(N, Mw, 3600.0, None, [g], "rk4", math)
        ex.set_state(p, v, I)
        ms = timed(ex, 100 if math == "fast" else 20, 5)
        ex.close()
        pair = 3.0 * N * (N - 1) * Mw / (ms * 1e-3)
        rows.append({"what": "nbody_1024", "worlds": Mw, "math": math, "us_per_tick": ms * 1e3, "pair_evals_per_s": pair,
                     "pipe_frac": pair * 18.0 / (fp64 * 1e9 / 2.0) if math == "fast" else None})
        print(json.dumps(rows[-1]), flush=True)
os.makedirs("gpurun_out", exist_ok=True)
json.dump({"fp64_probe_GFLOPs": fp64, "rows": rows}, open("gpurun_out/tune_misc.json", "w"), indent=1)
