"""A rocket dispersion analysis in ensemble mode: outcome tables reduced on the device, per thrust gain.

    python examples/rocket_dispersion.py [n_worlds] [ticks]

The campaign of rocket_monte_carlo.py (dispersed thrust, mass and wind), launched at a low angle so that the heavier,
weaker rockets come back down, swept over three thrust gains.  Ensemble mode keeps every run on the device; the
per-run outcomes (apogee, impact point and tick, and the dispersed inputs) are reduced over the worlds on the device
too, so no per-world table crosses PCIe.  Prints the apogee percentiles per gain, the impact ellipse, the impact
probability and the correlations between the downrange miss and the inputs.
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

q = ex.outcome_quantiles([0.01, 0.5, 0.99], groups=True)  # [G, 3, P]
k = ex.outcomes.index("apogee")
for g, gn in enumerate(gains):
    print(f"thrust gain {gn}: apogee 1% / 50% / 99% = {q[g, 0, k]:.2f} / {q[g, 1, k]:.2f} / {q[g, 2, k]:.2f} m")

hit = ex.outcome_stats(groups=True)["count"][:, ex.outcomes.index("impact_tick")]
for g, gn in enumerate(gains):
    print(f"thrust gain {gn}: impact probability {hit[g] / sizes[g]:.3f} ({int(hit[g])} of {sizes[g]} runs)")

c = ex.outcome_covariance(["impact_x", "impact_y"])
if c["count"] > 1:
    val, vec = np.linalg.eigh(c["cov"])
    ang = np.degrees(np.arctan2(vec[1, 1], vec[0, 1]))
    print(f"impact ellipse ({int(c['count'])} impacts): centre ({c['mean'][0]:.2f}, {c['mean'][1]:.2f}) m, 1-sigma "
          f"semi-axes {np.sqrt(max(val[1], 0.0)):.3f} and {np.sqrt(max(val[0], 0.0)):.3f} m, major axis at {ang:.1f} deg")

c = ex.outcome_covariance(["impact_x", "mass", "thrust", "wind"])
with np.errstate(invalid="ignore", divide="ignore"):
    corr = c["cov"] / np.sqrt(np.outer(np.diag(c["cov"]), np.diag(c["cov"])))
print("correlation of the downrange miss with " + ", ".join(f"{nm} {corr[0, j]:+.3f}" for j, nm in
                                                              enumerate(c["planes"]) if j))
