"""examples/grids/Taylor_Green.ipynb on the H100 path (without plotting).  python examples/taylor_green.py [--steps N]

The notebook in double precision: math.set_global_precision(64), a 25 x 25 periodic grid on Box(x=2 pi, y=2 pi), viscosity 0.1 and
199 steps at dt = 10 / 199 of  diffuse.explicit -> advect.semi_lagrangian -> fluid.make_incompressible(Solve('CG', 1e-12, 1e-12,
x0=pressure)), started from the analytic velocity and pressure.  Every operation of the step runs on the fp64 kernels.  The analytic
fields are sampled at the face and cell centres with NumPy in float64 (the notebook passes callables to the grid constructors); the
script prints the notebook's RMSE and relative error against the analytic velocity per frame.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403

PI = np.pi
N = 25
VISCOSITY = 0.1
FRAMES = 200                                  # time = math.linspace(0, 10., batch(time=200))
DT = 10. / (FRAMES - 1)


def domain():
    return dict(x=N, y=N, boundary=PERIODIC, bounds=Box(x=2 * PI, y=2 * PI))


def analytic_velocity(t):
    """taylor_green_velocity at the stored faces of the periodic staggered grid: the x component at (i dx, (j + 1/2) dx), the y
    component at ((i + 1/2) dx, j dx)."""
    h = 2 * PI / N
    faces, centres = np.arange(N) * h, (np.arange(N) + 0.5) * h
    decay = np.exp(-2 * VISCOSITY * t)
    xu, yu = np.meshgrid(faces, centres, indexing='ij')
    xv, yv = np.meshgrid(centres, faces, indexing='ij')
    return [np.cos(xu) * np.sin(yu) * decay, -np.sin(xv) * np.cos(yv) * decay]


def analytic_pressure(t):
    """taylor_green_pressure at the cell centres."""
    c = (np.arange(N) + 0.5) * 2 * PI / N
    x, y = np.meshgrid(c, c, indexing='ij')
    return -1 / 4 * (np.cos(2 * x) + np.cos(2 * y)) * np.exp(-4 * VISCOSITY * t)


def step(velocity, pressure, dt):
    velocity = diffuse.explicit(velocity, VISCOSITY, dt)
    velocity = advect.semi_lagrangian(velocity, velocity, dt)
    return fluid.make_incompressible(velocity, (), Solve('CG', 1e-12, 1e-12, x0=pressure))


def errors(v, t):
    """The notebook's rmse = sqrt(mean((analytic_v - sim_v)^2)) and relative_err = rmse / mean(|analytic_v|) of one frame."""
    exact = np.concatenate([c.ravel() for c in analytic_velocity(t)])
    sim = np.concatenate([c.ravel() for c in v])
    rmse = np.sqrt(np.mean((exact - sim) ** 2))
    return rmse, rmse / np.mean(np.abs(exact))


def run(steps=FRAMES - 1, verbose=False):
    """The notebook's trajectory.  Returns (final velocity components, final pressure, per-frame (rmse, relative error) for frames
    0 .. steps, CG iterations per step)."""
    with math.precision(64):
        v = StaggeredGrid(analytic_velocity(0.), **domain())
        p = CenteredGrid(analytic_pressure(0.), **domain())
    errs, iters = [errors(v.numpy(), 0.)], []
    with math.SolveTape() as solves:
        for k in range(steps):
            v, p = step(v, p, DT)
            errs.append(errors(v.numpy(), (k + 1) * DT))
            iters.append(int(solves[-1].iterations[0]))
            if verbose:
                print(f"frame {k + 1:3d}  t = {(k + 1) * DT:6.3f}  RMSE = {errs[-1][0]:.3e}  relative error = {errs[-1][1]:.3e}  "
                      f"CG iterations = {iters[-1]}")
    return v.numpy(), p.numpy(), np.array(errs), iters


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=FRAMES - 1)
    args = ap.parse_args()
    run(args.steps, verbose=True)
