"""examples/grids/Fluid_Logo.ipynb on the H100 path: smoke rising from three weighted inflows around the PhiFlow logo, an obstacle made
of eight boxes, the whole step as ONE library call per step.
python examples/fluid_logo.py [--res 128] [--steps 200]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403


def main(res=128, steps=200):
    domain = dict(x=res, y=res, bounds=Box(x=100, y=100))
    geometries = [Box(x=(15 + x * 7, 15 + (x + 1) * 7), y=(41, 83)) for x in range(1, 10, 2)] + \
                 [Box(x=(43, 50), y=(41, 48)), Box(x=(15, 43), y=(83, 90)), Box(x=(50, 85), y=(83, 90))]   # Box['x,y', 43:50, 41:48], ...
    geometry = union(geometries)
    inflow = CenteredGrid(Box(x=(14, 21), y=(6, 10)), ZERO_GRADIENT, **domain) + \
             CenteredGrid(Box(x=(81, 88), y=(6, 10)), ZERO_GRADIENT, **domain) * 0.9 + \
             CenteredGrid(Box(x=(44, 47), y=(49, 51)), ZERO_GRADIENT, **domain) * 0.4
    v = StaggeredGrid(0, boundary=0, **domain)
    smoke = CenteredGrid(0, boundary=ZERO_GRADIENT, **domain)
    pressure = None
    iterations = []
    with SolveTape() as solves:
        for _ in range(steps):
            # smoke = advect.semi_lagrangian(smoke, v, 1) + inflow; v = advect.semi_lagrangian(v, v, 1) + resample(smoke * (0, 0.1), to=v);
            # v, pressure = fluid.make_incompressible(v, geometry, Solve('CG-adaptive', 1e-5, x0=pressure))
            v, smoke, pressure = fluid.incompressible_step(v, smoke, pressure, 1., inflow=inflow, inflow_rate=1., buoyancy=(0, 0.1),
                                                           solve=Solve('CG-adaptive', 1e-5), obstacles=geometry)
            iterations.append(int(solves[-1].iterations[0]))
    s = smoke.numpy()
    inside = geometry.lies_inside(smoke.points())
    print(f"fluid logo {res}x{res}, {steps} steps: smoke {float(s.sum()):.2f}, smoke inside the obstacle {float(np.abs(s[inside]).sum()):.3e}, "
          f"CG-adaptive iterations first / last {iterations[0]} / {iterations[-1]}")
    return smoke, v, pressure, iterations


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, default=128)
    ap.add_argument('--steps', type=int, default=200)
    a = ap.parse_args()
    main(a.res, a.steps)
