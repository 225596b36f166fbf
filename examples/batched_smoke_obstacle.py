"""examples/grids/Batched_Smoke.ipynb on the H100 path: three inflow settings as one batch, an obstacle in the flow.
python examples/batched_smoke_obstacle.py [--res 64] [--steps 100]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403


def main(res=64, steps=100):
    domain = Box(x=100, y=100)
    inflow_rate = (.1, .2, .3)
    inflow_x = (40, 50, 60)
    obstacle = Box(x=(35, 65), y=(50, 70))                      # Cuboid(vec(x=50, y=60), half_size=vec(x=15, y=10))
    v = StaggeredGrid(0, 0, domain, batch=3, x=res, y=res)
    s = CenteredGrid(0, ZERO_GRADIENT, domain, batch=3, x=res, y=res)
    # inflow_rate * resample(inflow, to=s, soft=True) per setting, baked into one batched mask
    masks = np.stack([r * resample(Sphere(x=cx, y=9.5, radius=5), to=CenteredGrid(0, ZERO_GRADIENT, domain, x=res, y=res), soft=True).numpy()
                      for r, cx in zip(inflow_rate, inflow_x)])
    inflow = CenteredGrid(masks, ZERO_GRADIENT, domain, batch=3, x=res, y=res)
    p = None
    for _ in range(steps):
        s = advect.mac_cormack(s, v, 1.) + inflow
        buoyancy = resample(s * (0, 0.1), to=v)
        v = advect.semi_lagrangian(v, v, 1.) + buoyancy * 1.
        v, p = fluid.make_incompressible(v, obstacle, Solve(x0=p))
    smoke = s.numpy()
    inside = obstacle.lies_inside(s.points()) if hasattr(s, 'points') else None
    print(f"batched smoke {res}x{res} x 3 settings, {steps} steps: smoke per setting {[round(float(a.sum()), 2) for a in smoke]}"
          + (f", smoke inside the obstacle {float((smoke * inside).sum()):.3e}" if inside is not None else ""))
    return v, s, p


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, default=64)
    ap.add_argument('--steps', type=int, default=100)
    a = ap.parse_args()
    main(a.res, a.steps)
