"""The worst runs of a rocket dispersion campaign: flagged on the device, then replayed with full telemetry.

    python examples/rocket_worst_runs.py [n_worlds] [ticks] [out_dir]

The campaign of rocket_dispersion.py (dispersed thrust gain, mass and wind, one world group per thrust gain) runs in
ensemble mode.  Exec.outcome_top_worlds then names the worst runs without a per-world table crossing PCIe: the 8
largest downrange misses over the campaign (the smallest impact x: the rocket flies toward -x) and the 8 lowest
apogees of each thrust gain (tied apogees, such as rockets too heavy to climb, come in world order).  The same campaign
is built again with retain= those worlds, so that their full telemetry rows are recorded, and each flagged run is
written to its own elodin-db under <out_dir>/runs/<run_id>/db with monte_carlo.write_run_databases.
"""
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import elodin_b200 as el
from elodin_b200 import monte_carlo

n = int(sys.argv[1]) if len(sys.argv) > 1 else 30000
ticks = int(sys.argv[2]) if len(sys.argv) > 2 else 1200
out_dir = sys.argv[3] if len(sys.argv) > 3 else tempfile.mkdtemp(prefix="rocket_worst_runs_")
gains = (0.9, 1.0, 1.1)
sizes = [n // 3 + (g < n % 3) for g in range(3)]  # the worlds of each gain are contiguous: one group per sweep point
rng = np.random.default_rng(42)
gain = np.repeat(gains, sizes)
mass = rng.uniform(2.5, 3.5, n)
wind_x = rng.normal(0.0, 2.0, n)

Thrust = el.Annotated[np.ndarray, el.Component("thrust", el.ComponentType.F64)]
Wind = el.Annotated[np.ndarray, el.Component("wind", el.ComponentType(el.PrimitiveType.F64, (3,)))]


@el.dataclass
class Rocket(el.Archetype):
    thrust: Thrust
    wind: Wind


def campaign(retain=None):
    """rocket_dispersion.py's campaign, run for `ticks` ticks; with `retain`, the full rows of those worlds too."""
    w = el.World()
    w.spawn([el.Body(world_pos=el.SpatialTransform(angular=el.Quaternion.from_euler([0.0, np.radians(20.0), 0.0]),
                                                   linear=np.array([0.0, 0.0, 1.0])),
                     inertia=el.SpatialInertia(3.0, np.array([0.1, 1.0, 1.0]))),
             Rocket(np.array([88.426]), np.zeros(3))], name="rocket")
    effectors = (el.GravityConst((0.0, 0.0, -9.81)) | el.ThrustBody((-1.0, 0.0, 0.0), "thrust")
                 | el.DragQuadratic(0.6125, 0.0025, "wind"))
    params = {"thrust": (88.426 * gain)[:, None, None],
              "wind": np.stack([wind_x, np.zeros(n), np.zeros(n)], -1)[:, None, :],
              "inertia": np.stack([np.full(n, 0.1), np.ones(n), np.ones(n), np.zeros(n), np.zeros(n), np.zeros(n), mass],
                                  -1)[:, None, :]}
    O = el.Outcome
    outcomes = [O("apogee", "rocket.world_pos", 6, "max"), O.threshold("impact_tick", 0, "tick"),
                O.threshold("impact_x", 0, "world_pos", 4), O.threshold("impact_y", 0, "world_pos", 5),
                O("mass", "rocket.inertia", 6), O("thrust", "rocket.thrust", 0), O("wind", "rocket.wind", 0)]
    ex = w.build(el.six_dof(sys=effectors), simulation_rate=120.0, telemetry_rate=120.0, math="fast", n_worlds=n,
                 world_params=params, ensemble=True, groups=sizes, extrema=True,
                 thresholds=[el.Threshold("rocket.world_pos", 6, below=0.0)], outcomes=outcomes, retain=retain)
    ex.run(ticks)
    return ex


ex = campaign()
# the rocket flies toward -x, so the farthest impacts downrange have the smallest impact_x
miss = ex.outcome_top_worlds(8, names=["impact_x"], largest=False)
print(f"the 8 largest downrange misses ({int(miss['count'][0])} impacts):")
for x, wd in zip(miss["value"][0], miss["world"][0]):
    if wd >= 0:
        print(f"  world {wd:6d}: impact x = {x:.3f} m (gain {gain[wd]}, mass {mass[wd]:.3f} kg, wind {wind_x[wd]:+.3f} m/s)")
low = ex.outcome_top_worlds(8, names=["apogee"], largest=False, groups=True)
for g, gn in enumerate(gains):
    print(f"thrust gain {gn}: the 8 lowest apogees " + ", ".join(
        f"{a:.2f} m (world {wd})" for a, wd in zip(low["value"][g, 0], low["world"][g, 0]) if wd >= 0))

flagged = sorted(set(int(wd) for wd in np.concatenate([miss["world"].ravel(), low["world"].ravel()]) if wd >= 0))
replay = campaign(retain=flagged)
z = replay.history_worlds("rocket.world_pos")[..., 6]  # [rows, flagged]
apogee = ex.outcome_values()["apogee"] if n <= 1 << 16 else None  # a per-world download: small campaigns only
for slot, wd in enumerate(flagged[:4]):
    top = np.nanmax(z[:, slot])
    note = "" if apogee is None else f" (outcome {apogee[wd]:.6f} m)"
    print(f"replayed world {wd}: {z.shape[0]} rows, apogee {top:.6f} m{note}")
rows = [{"run_id": f"run_{k:07}"} for k in range(n)]
paths = monte_carlo.write_run_databases(replay, rows, out_dir, keep=flagged)
print(f"wrote {len(paths)} run databases under {os.path.join(out_dir, 'runs')}")
