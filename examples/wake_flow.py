"""examples/grids/Wake_Flow.ipynb on the H100 path: flow past a cylinder that spans the periodic z extent, inflow from x-.
python examples/wake_flow.py [--res 128] [--nz 8] [--steps 200]
--res sets the x resolution (y takes half of it), --nz the z resolution; the notebook runs 128 x 64 x 8.

The notebook projects the initial velocity with Solve('scipy-direct').  There is no direct solver here, so that first
projection runs CG-adaptive at rel_tol = abs_tol = 1e-5; every step then uses Solve(x0=p) = CG-adaptive, as in the notebook."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403


def main(res=128, nz=8, steps=200, dt=1.):
    cylinder = geom.infinite_cylinder(x=20, y=50, radius=10, inf_dim='z')
    boundary = {'x-': vec(x=2, y=0, z=0), 'x+': ZERO_GRADIENT, 'y': PERIODIC, 'z': PERIODIC}
    v0 = StaggeredGrid((8., 0, 0), boundary, x=res, y=res // 2, z=nz, bounds=Box(x=200, y=100, z=5))
    v0, p0 = fluid.make_incompressible(v0, cylinder, Solve('CG-adaptive', 1e-5, 1e-5))

    def step(v, p):
        v = advect.semi_lagrangian(v, v, dt)
        return fluid.make_incompressible(v, cylinder, Solve(x0=p))

    v, p = iterate(step, steps, v0, p0)
    vx = v.numpy()[0]
    print(f"wake flow {res}x{res // 2}x{nz}, {steps} steps: max|v_x| {float(abs(vx).max()):.3f}, max|p| {float(abs(p.numpy()).max()):.3f}")
    return v, p


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--res', type=int, default=128)
    ap.add_argument('--nz', type=int, default=8)
    ap.add_argument('--steps', type=int, default=200)
    a = ap.parse_args()
    main(a.res, a.nz, a.steps)
