"""compute-sanitizer target for the kernels added late in round 1: small_world_kernel (FAST / EXACT, RK4 /
semi-implicit, ragged worlds per warp, sparse CSR graph), the full-telemetry trajectory ring and its
25-plane read-back, and the trajectory ring's slot rule on every tick route.  Small sizes where it can: the tool
slows every kernel by 10-50x."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import elodin_b200 as el

rng = np.random.default_rng(1)
for N in (3, 7, 32):
    M = 41
    p = np.zeros((M, N, 7)); p[..., 3] = 1.0; p[..., 4:] = rng.uniform(-5, 5, (M, N, 3))
    v = rng.normal(0, 0.1, (M, N, 6)); I = np.ones((M, N, 7)); I[..., 6] = rng.uniform(1, 2, (M, N))
    graphs = [el.all_pairs_edges(N)]
    if N > 3:
        graphs.append(np.array([(i, j) for i in range(0, N, 2) for j in rng.permutation(N)[:3] if i != j]))
    for edges in graphs:
        for integ in ("rk4", "semi_implicit"):
            for math in ("fast", "exact"):
                g = el.GravityEdges("softened", k_squared=0.3, softening=1e-6, edges=edges)
                with el.B200Exec(N, M, 0.01, None, [g, el.ThrustBody()], integ, math, max_fused_ticks=3,
                                 trajectory_every=2, trajectory_capacity=3, trajectory_full=True) as ex:
                    ex.set_state(p, v, I, thrust=rng.uniform(0, 1, (M, N, 1)))
                    ex.step(7, sync=True)
                    assert ex.trajectory().shape == (3, M, N, 25)
M = 1000
p = np.zeros((M, 1, 7)); p[..., 3] = 1.0
with el.B200Exec(1, M, 0.01, None, [el.GravityConst()], "rk4", "fast", max_fused_ticks=8, trajectory_every=4,
                 trajectory_capacity=4, trajectory_full=True) as ex:
    ex.set_state(p, rng.normal(0, 1, (M, 1, 6)), np.ones((M, 1, 7)))
    ex.step(16, sync=True)
    assert np.isfinite(ex.trajectory()).all()
# the trajectory ring's slot rule on every tick route (tests/test_trajectory_routes.py), a write past the last slot
# being what only this tool can see: every schedule on the small cases, and the one-tick schedule of the deferred
# 16-byte pair store and of the pipelined ranges past kPairMinBodies (one of them at an odd body)
from tests import test_trajectory_routes as T

for key in ("exact-g_thrust_drag-rk4", "spec-thrust_drag-rk4", "interp-egm08-semi_implicit", "small-irregular-exact-rk4",
            "small-dense-rk4", "csr-semi_implicit", "nbody-fused", "nbody-exact", "invoke-ranges", "pair-free-rk4",
            "invoke-pair"):
    for s, w in T.CASES[key]["runs"]:
        steps, _ = T.plan(T.SCHEDULES[s], T.CASES[key]["multi"], T.CASES[key]["per_launch"])
        for invoke in (False, True) if "chunk" in T.CASES[key] else (False,):
            out = T._record(key, s, w, invoke)
            assert list(out["len"]) == [st["len"] for st in steps], (key, s, w, invoke)
print("done")
