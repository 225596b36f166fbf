"""examples/grids/Reaction_Diffusion.ipynb on the H100 path (without plotting).  python examples/reaction_diffusion.py [--frames N]

The notebook's first initialisation is `Noise(scale=20, smoothness=1.3)`, which the mirror does not have: `smooth_noise` below stands
in for it with seeded Gaussian-filtered white noise of unit standard deviation.  Each frame is ONE call of the fused step with
substeps=20 (all 20 Gray-Scott substeps in one kernel launch); `reaction_diffusion_cell` is the notebook's own cell, which runs
unmodified on the mirror's field arithmetic (about 20 launches per substep) and serves as a cross-check.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403
from phiflow_b200.flow import reaction_diffusion  # noqa: E402

PARAMS = {'maze': {'du': 0.19, 'dv': 0.05, 'f': 0.06, 'k': 0.062},
          'coral': {'du': 0.16, 'dv': 0.08, 'f': 0.06, 'k': 0.062},
          'dots': {'du': 0.19, 'dv': 0.03, 'f': 0.04, 'k': 0.061}}
FRAMES = {'maze': 100, 'coral': 200, 'dots': 100}
N = 100


@jit_compile
def reaction_diffusion_cell(u, v, du, dv, f, k, dt):
    uvv = u * v**2
    su = du * field.laplace(u) - uvv + f * (1 - u)
    sv = dv * field.laplace(v) + uvv - (f + k) * v
    return u + dt * su, v + dt * sv


def smooth_noise(n=N, scale=20.0, seed=0):
    """Stand-in for Noise(scale=20): white noise low-pass filtered at wavelengths around `scale` cells, unit standard deviation."""
    white = np.random.default_rng(seed).standard_normal((n, n))
    kx, ky = np.meshgrid(np.fft.fftfreq(n), np.fft.fftfreq(n), indexing='ij')
    a = np.fft.ifft2(np.fft.fft2(white) * np.exp(-0.5 * (np.hypot(kx, ky) * scale) ** 2)).real
    return ((a - a.mean()) / a.std()).astype(np.float32)


def initial_state(n=N):
    """The notebook's three initialisations stacked along the batch: noise * .2 + .1, a Gaussian blob, concentric rings."""
    x = (np.arange(n) + 0.5).astype(np.float32)
    X, Y = np.meshgrid(x, x, indexing='ij')
    r2 = (X - 50) ** 2 + (Y - 50) ** 2
    values = np.stack([smooth_noise(n) * .2 + .1, np.exp(-0.5 * r2 / 3 ** 2), np.cos(np.sqrt(r2) / 3) * .5]).astype(np.float32)
    return CenteredGrid(values, x=n, y=n, batch=3)


def run(params='maze', frames=None, substeps=20, dt=.5, fused=True):
    """One trajectory of the notebook (u0 serves as both u and v, as there).  Returns the u and v trajectories as numpy arrays
    (frames + 1, 3, n, n)."""
    frames = FRAMES[params] if frames is None else frames
    u0 = initial_state()
    if fused:
        frame = lambda u, v, **kw: reaction_diffusion(u, v, dt=dt, substeps=substeps, **kw)
        u_trj, v_trj = iterate(frame, batch(time=frames), u0, u0, f_kwargs=PARAMS[params])
    else:
        u_trj, v_trj = iterate(reaction_diffusion_cell, batch(time=frames), u0, u0, dt=dt, f_kwargs=PARAMS[params], substeps=substeps)
    return np.stack([u.numpy() for u in u_trj]), np.stack([v.numpy() for v in v_trj])


def main(frames=None):
    out = {}
    for name in PARAMS:
        u, v = run(name, frames)
        out[name] = (u, v)
        print(f"{name}: {u.shape[0] - 1} frames of 20 substeps, 100x100, batch 3: u in [{u[-1].min():.3f}, {u[-1].max():.3f}], "
              f"v in [{v[-1].min():.3f}, {v[-1].max():.3f}]")
    return out


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=None, help='frames per parameter set (default: the notebook\'s 100 / 200 / 100)')
    main(ap.parse_args().frames)
