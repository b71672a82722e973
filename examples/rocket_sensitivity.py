"""Which dispersed input drives the miss: rank correlation and partial rank correlation of a rocket dispersion campaign.

    python examples/rocket_sensitivity.py [n_worlds] [ticks]

The campaign of rocket_dispersion.py (dispersed mass and wind, swept over three thrust gains).  The outcomes are ranked
on the device, within each sweep point with groups=True, and their Spearman correlation comes back as one small table;
outcome_sensitivity adds the partial rank correlation (PRCC), which separates inputs that act together.  Prints the
Spearman rho and the PRCC of apogee and of the downrange impact point against mass, wind and thrust gain: over all
worlds (thrust takes 3 values, so its ranks are heavily tied), per gain (thrust is constant within a sweep point, so
its row is NaN), and next to the Pearson correlation of outcome_covariance that rocket_dispersion.py prints.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import elodin_b200 as el

n = int(sys.argv[1]) if len(sys.argv) > 1 else 30000
ticks = int(sys.argv[2]) if len(sys.argv) > 2 else 1200
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


w = el.World()
w.spawn([el.Body(world_pos=el.SpatialTransform(angular=el.Quaternion.from_euler([0.0, np.radians(20.0), 0.0]),
                                               linear=np.array([0.0, 0.0, 1.0])),
                 inertia=el.SpatialInertia(3.0, np.array([0.1, 1.0, 1.0]))),
         Rocket(np.array([88.426]), np.zeros(3))], name="rocket")
effectors = el.GravityConst((0.0, 0.0, -9.81)) | el.ThrustBody((-1.0, 0.0, 0.0), "thrust") | el.DragQuadratic(0.6125, 0.0025, "wind")
params = {"thrust": (88.426 * gain)[:, None, None],
          "wind": np.stack([wind_x, np.zeros(n), np.zeros(n)], -1)[:, None, :],
          "inertia": np.stack([np.full(n, 0.1), np.ones(n), np.ones(n), np.zeros(n), np.zeros(n), np.zeros(n), mass], -1)[:, None, :]}
O = el.Outcome
outcomes = [O("apogee", "rocket.world_pos", 6, "max"), O.threshold("impact_tick", 0, "tick"),
            O.threshold("impact_x", 0, "world_pos", 4), O.threshold("impact_y", 0, "world_pos", 5),
            O("mass", "rocket.inertia", 6), O("thrust", "rocket.thrust", 0), O("wind", "rocket.wind", 0)]
ex = w.build(el.six_dof(sys=effectors), simulation_rate=120.0, telemetry_rate=120.0, math="fast", n_worlds=n,
             world_params=params, ensemble=True, groups=sizes, extrema=True,
             thresholds=[el.Threshold("rocket.world_pos", 6, below=0.0)], outcomes=outcomes)
ex.run(ticks)

inputs = ["mass", "wind", "thrust"]


def table(title, s, pearson=None):
    print(f"{title} ({int(s['count'])} complete worlds)")
    print("  " + " " * 10 + "".join(f"{'rho ' + i:>14s}{'prcc ' + i:>14s}" for i in s["inputs"]) +
          ("".join(f"{'pearson ' + i:>17s}" for i in s["inputs"]) if pearson is not None else ""))
    for y, out in enumerate(s["outputs"]):
        row = "".join(f"{s['rho'][y, i]:+14.3f}{s['prcc'][y, i]:+14.3f}" for i in range(len(s["inputs"])))
        if pearson is not None:
            row += "".join(f"{pearson[y, i]:+17.3f}" for i in range(len(s["inputs"])))
        print(f"  {out:10s}{row}")


# apogee: every world; impact_x: the worlds that came down (a tick that never happened is NaN, so the others drop out)
for outputs in (["apogee"], ["impact_x"]):
    s = ex.outcome_sensitivity(inputs, outputs)
    c = ex.outcome_covariance(inputs + outputs)
    with np.errstate(invalid="ignore", divide="ignore"):
        corr = c["cov"] / np.sqrt(np.outer(np.diag(c["cov"]), np.diag(c["cov"])))
    table(f"all gains, {outputs[0]}: Spearman, PRCC and Pearson", s, corr[len(inputs):, :len(inputs)])

g = ex.outcome_sensitivity(inputs, ["apogee", "impact_x"], groups=True)
for k, gn in enumerate(gains):
    table(f"thrust gain {gn} (thrust constant: NaN)", {key: (v[k] if key in ("count", "rho", "prcc") else v)
                                                      for key, v in g.items()})
