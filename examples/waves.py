"""examples/grids/Waves.ipynb on the H100 path (without plotting).  python examples/waves.py [--frames N] [--cell]

Each frame is ONE call of the fused step with substeps=16: the moving source disc of each substep is evaluated on the host, and all
16 substeps (stamp + explicit wave update) run in one kernel launch.  `--cell` runs the notebook's own cell instead (`step` below,
verbatim), on the mirror's field arithmetic: about a dozen launches and a host-built disc mask per substep.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403
from phiflow_b200.flow import wave_step  # noqa: E402

DT = 1 / 60. / 16
SUBSTEPS = 16


def wave_displace(sphere: Sphere, *fields, mag=.5, t=-math.PI * 0.5):
    return [field.where(sphere, mag * math.sin(t), f) for f in fields]


@jit_compile
def step(h_c, h_p, time, dt=1/60./16, k_speed=1.0, k_damp=0.0):
    sphere = Sphere(center=h_c.bounds.center + math.rotate_vector(vec(x=0, y=-12.8/3), time), radius=1.)
    h_c, h_p = wave_displace(sphere, h_c, h_p)
    h_n = 2.0 * h_c - h_p + dt * dt * (k_speed * h_c.laplace() - k_damp * (h_c - h_p))  # wave_solve
    return h_n, h_c, time + dt


def source(bounds):
    """The notebook's disc and value as a function of time, for the fused step."""
    return lambda time: (Sphere(center=bounds.center + math.rotate_vector(vec(x=0, y=-12.8/3), time), radius=1.), .5 * math.sin(-math.PI * .5))


def initial_state():
    return CenteredGrid(x=128, y=128, bounds=Box(x=12.8, y=12.8), boundary=ZERO_GRADIENT)


def frame(h_c, h_p, time):
    """One recorded frame of the notebook: 16 substeps in one call."""
    return wave_step(h_c, h_p, time, DT, substeps=SUBSTEPS, source=source(h_c.bounds))


def run(frames=300, cell=False):
    """The notebook's trajectory.  Returns the h trajectory as a numpy array (frames + 1, 128, 128) and the final time."""
    h_initial = initial_state()
    if cell:
        h_trj, _, t_trj = iterate(step, batch(time=frames), h_initial, h_initial, 0, substeps=SUBSTEPS)
    else:
        h_trj, _, t_trj = iterate(frame, batch(time=frames), h_initial, h_initial, 0)
    return np.stack([h.numpy() for h in h_trj]), t_trj[-1]


def main(frames=300, cell=False):
    h, t = run(frames, cell)
    print(f"{'cell' if cell else 'fused'}: {h.shape[0] - 1} frames of {SUBSTEPS} substeps, 128x128, t = {t:.4f}: "
          f"h in [{h[-1].min():.4f}, {h[-1].max():.4f}]")
    return h


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=300)
    ap.add_argument('--cell', action='store_true', help="run the notebook's own cell on the mirror's field arithmetic")
    a = ap.parse_args()
    main(a.frames, a.cell)
