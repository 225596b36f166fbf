"""examples/grids/Heat_Flow.ipynb on the H100 path.  python examples/heat_flow.py [--steps 100]"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403

domain = Box(x=10, y=5)
boundary = {'x-': 1, 'x+': ZERO_GRADIENT, 'y': PERIODIC}
bars = union(Box(x=(0, 10), y=(2, 3)), Box(x=(4.5, 5.5), y=(1, 4)))
conductivity = CenteredGrid(bars, ZERO_GRADIENT, domain, x=100, y=50) + .01


@jit_compile
def step(t, dt):
    return diffuse.implicit(t, conductivity, dt)


def run(steps=100):
    """The notebook's trajectory (without plotting).  Returns the final temperature, the CG iterations of every step, and what a
    check needs to repeat the steps: the conductivity values, the boundary as an ops-level spec, the cell size."""
    t0 = CenteredGrid(0, boundary, domain, x=100, y=50)
    iterations = []
    with math.SolveTape() as tape:
        t_trj = iterate(step, batch(time=steps), t0, dt=1)          # the notebook passes range=trange (a progress bar)
    for s in range(len(tape)):
        iterations.append(int(tape[s].iterations[0]))
    t = t_trj[-1]
    return dict(t=t.numpy(), iterations=iterations, conductivity=conductivity.numpy(), spec=t.spec, dx=t.dx)


def main(steps=100):
    out = run(steps)
    t = out['t']
    print(f"heat flow 100x50, {steps} steps at dt = 1: mean temperature {float(t.mean()):.4f}, at x- {float(t[0].mean()):.4f}, "
          f"at x+ {float(t[-1].mean()):.4f}; CG iterations per step {min(out['iterations'])} .. {max(out['iterations'])}")
    return out


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=100)
    a = ap.parse_args()
    main(a.steps)
