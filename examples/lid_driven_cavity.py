"""examples/grids/Lid_Driven_Cavity.ipynb on the H100 path.  python examples/lid_driven_cavity.py [--steps 300]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403


@jit_compile
def step(v, p, dt=1., viscosity=.1):
    v = advect.semi_lagrangian(v, v, dt)
    v = diffuse.explicit(v, viscosity, dt)
    v, p = fluid.make_incompressible(v, solve=Solve(x0=p))
    return v, p


def main(steps=300, x=50, y=32):
    boundary = {'x': 0, 'y-': 0, 'y+': vec(x=1, y=0)}
    v0 = StaggeredGrid(0, boundary, x=x, y=y)
    v, p = iterate(step, steps, v0, None)           # the notebook records the trajectory: iterate(step, batch(time=300), v0, None)
    vx, vy = v.numpy()
    print(f"lid-driven cavity {x}x{y}, {steps} steps: max|v_x| = {float(np.abs(vx).max()):.4f} (lid speed 1), "
          f"return flow min v_x = {float(vx.min()):.4f}, max|div v| = {float(np.abs(field.divergence(v).numpy()).max()):.2e}")
    return v, p


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=300)
    a = ap.parse_args()
    main(a.steps)
