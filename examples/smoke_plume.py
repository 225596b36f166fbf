"""examples/grids/Smoke_Plume.ipynb on the H100 path (cells :39-68).  python examples/smoke_plume.py [--res 128] [--steps 50] [--scene DIR]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403


def main(res=128, steps=50, scene_dir=None, fused=True):
    domain = Box(x=100, y=100)
    inflow = Sphere(x=50, y=9.5, radius=5)
    inflow_rate = 0.2
    v = StaggeredGrid(0, 0, domain, x=res, y=res)
    s = CenteredGrid(0, ZERO_GRADIENT, domain, x=res, y=res)
    inflow_mask = resample(inflow, to=s, soft=True)
    p = None
    scene = Scene.create(scene_dir) if scene_dir else None

    def step(v, s, p, dt):                                          # the notebook's step(), function by function
        s = advect.mac_cormack(s, v, dt) + inflow_rate * inflow_mask
        buoyancy = resample(s * (0, 0.1), to=v)
        v = advect.semi_lagrangian(v, v, dt) + buoyancy * dt
        v, p = fluid.make_incompressible(v, (), Solve('CG', 1e-3, x0=p))
        return v, s, p

    for i in range(steps):
        if fused:                                                   # the same step as ONE library call (5 kernel launches)
            v, s, p = fluid.incompressible_step(v, s, p, 0.5, inflow=inflow_mask, inflow_rate=inflow_rate, buoyancy=(0, 0.1),
                                                solve=Solve('CG', 1e-3), smoke_advection='mac_cormack')
        else:
            v, s, p = step(v, s, p, 0.5)
        if scene is not None and i % 10 == 0:
            scene.write({'smoke': s, 'velocity': v}, frame=i)
    smoke = s.numpy()
    print(f"smoke plume {res}x{res}, {steps} steps: total smoke {float(smoke.sum()):.3f}, highest smoke cell y = "
          f"{int(np.nonzero(smoke.max(axis=0) > 1e-3)[0].max())}, max|div v| = {float(np.abs(field.divergence(v).numpy()).max()):.2e}")
    return v, s, p


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, default=128)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--scene', default=None)
    ap.add_argument('--unfused', action='store_true')
    a = ap.parse_args()
    main(a.res, a.steps, a.scene, not a.unfused)
