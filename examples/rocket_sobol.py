"""Which dispersed input drives the miss, non-monotone effects included: Sobol indices of a rocket campaign.

    python examples/rocket_sobol.py [n_base] [ticks]

The rocket of rocket_sensitivity.py with dispersed mass, wind speed and a wind azimuth uniform over [0, 2 pi) (measured
from the y axis), swept over three thrust gains.  monte_carlo.saltelli lays the campaign out as blocks of d + 2 worlds
per base sample (world k = plan row k), one group per thrust gain; Exec.outcome_sobol returns the first-order (S1) and
total (ST) indices of each output with bootstrap confidence half-widths, and outcome_sensitivity the PRCC of the same
worlds.  The crossrange impact point (impact_y) goes as cos(azimuth), so the azimuth's PRCC is about 0 and only ST
shows its effect.  In this model the mass sets apogee and the downrange impact point (the wind's share of those is
below 0.1 %), many worlds do not come down within the run (a sample counts only if its d + 2 worlds all land), and the
crossrange intervals are wide: read the half-widths before the indices.
"""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import elodin_b200 as el
from elodin_b200 import monte_carlo

GAINS = (0.9, 1.0, 1.1)
SPEC = {
    "sim_sweep": {"thrust_gain": list(GAINS)},
    "monte_carlo": {"n_samples": 2048, "method": "random", "seed": 7, "variables": {
        "mass": {"dist": "uniform", "min": 2.5, "max": 3.5},
        "wind_speed": {"dist": "uniform", "min": 0.0, "max": 4.0},
        "wind_az": {"dist": "uniform", "min": 0.0, "max": 2.0 * math.pi},
        "pitch_deg": {"dist": "fixed", "value": 20.0},
    }},
}

Thrust = el.Annotated[np.ndarray, el.Component("thrust", el.ComponentType.F64)]
Wind = el.Annotated[np.ndarray, el.Component("wind", el.ComponentType(el.PrimitiveType.F64, (3,)))]


@el.dataclass
class Rocket(el.Archetype):
    thrust: Thrust
    wind: Wind


def campaign(n_base=None, ticks=3600, bootstrap=200, seed=0, math_mode="fast"):
    """(design, Exec, Sobol dict, sensitivity dict) of the campaign: Sobol indices per thrust gain with groups=True,
    and the PRCC of the same worlds over every gain."""
    design = monte_carlo.saltelli(SPEC, n_base)
    rows, sizes, _ = monte_carlo.plan_groups(design.rows, ["param.thrust_gain"])
    p = monte_carlo.plan_params(rows)
    n = len(rows)
    col = lambda k: np.array([r[k] for r in p], dtype=np.float64)
    mass, speed, az, gain = col("mass"), col("wind_speed"), col("wind_az"), col("thrust_gain")
    pitch = np.radians(p[0]["pitch_deg"])
    w = el.World()
    w.spawn([el.Body(world_pos=el.SpatialTransform(angular=el.Quaternion.from_euler([0.0, pitch, 0.0]),
                                                   linear=np.array([0.0, 0.0, 1.0])),
                     inertia=el.SpatialInertia(3.0, np.array([0.1, 1.0, 1.0]))),
             Rocket(np.array([88.426]), np.zeros(3))], name="rocket")
    effectors = (el.GravityConst((0.0, 0.0, -9.81)) | el.ThrustBody((-1.0, 0.0, 0.0), "thrust")
                 | el.DragQuadratic(0.6125, 0.0025, "wind"))
    params = {"thrust": (88.426 * gain)[:, None, None],
              "wind": np.stack([speed * np.sin(az), speed * np.cos(az), np.zeros(n)], -1)[:, None, :],
              "inertia": np.stack([np.full(n, 0.1), np.ones(n), np.ones(n), np.zeros(n), np.zeros(n), np.zeros(n),
                                   mass], -1)[:, None, :]}
    O = el.Outcome
    values = {"mass": mass, "wind_speed": speed, "wind_az": az}  # the inputs as outcomes, for the PRCC
    outcomes = [O("apogee", "rocket.world_pos", 6, "max"), O.threshold("impact_x", 0, "world_pos", 4),
                O.threshold("impact_y", 0, "world_pos", 5)] + [O.values(k, values[k]) for k in design.inputs]
    ex = w.build(el.six_dof(sys=effectors), simulation_rate=120.0, telemetry_rate=120.0, math=math_mode, n_worlds=n,
                 world_params=params, ensemble=True, groups=sizes, extrema=True,
                 thresholds=[el.Threshold("rocket.world_pos", 6, below=0.0)], outcomes=outcomes)
    ex.run(ticks)
    outputs = ["apogee", "impact_x", "impact_y"]
    sobol = ex.outcome_sobol(design.inputs, outputs, groups=True, bootstrap=bootstrap, seed=seed)
    sens = ex.outcome_sensitivity(design.inputs, outputs)
    return design, ex, sobol, sens


def main():
    n_base = int(sys.argv[1]) if len(sys.argv) > 1 else None
    ticks = int(sys.argv[2]) if len(sys.argv) > 2 else 3600
    design, ex, s, sens = campaign(n_base, ticks)
    d = len(design.inputs)
    print(f"Saltelli design: {design.n_base} base samples x {d + 2} worlds x {len(GAINS)} thrust gains "
          f"= {ex.n_worlds} worlds; inputs {design.inputs}")
    for k, gain in enumerate(GAINS):
        print(f"thrust gain {gain}")
        print("  " + " " * 10 + "".join(f"{i:>36s}" for i in design.inputs))
        for y, out in enumerate(s["outputs"]):
            cells = "".join(f"  S1 {s['S1'][k, y, i]:+.3f}±{s['S1_conf'][k, y, i]:.3f} ST {s['ST'][k, y, i]:+.3f}"
                            f"±{s['ST_conf'][k, y, i]:.3f}" for i in range(d))
            print(f"  {out:10s}{cells}   (n = {int(s['count'][k, y])})")
    print(f"PRCC of the same worlds, every gain ({int(sens['count'])} complete worlds)")
    for y, out in enumerate(sens["outputs"]):
        print(f"  {out:10s}" + "".join(f"{i:>14s} {sens['prcc'][y, j]:+.3f}" for j, i in enumerate(design.inputs)))


if __name__ == "__main__":
    main()
