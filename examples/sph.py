"""examples/particles/SPH.ipynb on the H100 path (without plotting).  python examples/sph.py [--nx 25 --ny 100 --nz 25] [--frames 480] [--cell]

The notebook's dam break: 25 x 100 x 25 particles on a lattice of spacing h = 0.8 in the corner of Box(x=80, y=80, z=80), 480 frames
of int(32 / h) = 40 substeps of apply_bounds(sph_step(v)).  The cells run on the mirror API, with two differences:
  * `math.random_normal` is PhiML's own generator: the jitter of the initial lattice is seeded NumPy noise of the same size;
  * Sphere(volume=h ** 3) is not in the mirror: `particle_volume` states the volume the notebook's Sphere reports, in float32.
By default one `sph_step(..., substeps=40)` call runs each frame in one kernel launch; --cell runs the notebook's own loop,
iterate(step, batch(t=frames), x, v, substeps=40), one launch per substep.  Both give the same bits.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403

SMOOTHING_LENGTH = 0.8


def particle_volume(h, d=3):
    """Sphere(center, volume=h ** d).volume as the notebook's PhiML tensors give it: volume_from_radius(radius_from_volume(h ** d))."""
    f32 = np.float32
    if d == 3:
        return f32(4 / 3 * np.pi) * np.power(np.power(f32(.75 / np.pi) * np.asarray(h ** 3, f32), 1 / 3), 3)
    return f32(np.pi) * np.power(np.sqrt(np.asarray(h ** 2, f32) / f32(np.pi)), 2)


def initial_state(nx=25, ny=100, nz=25, h=SMOOTHING_LENGTH, seed=0):
    """pack_dims(meshgrid(x=nx, y=ny, z=nz), spatial, instance('particles')) * h + 0.001 h N(0, 1), and zero velocities."""
    grid = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing='ij'), -1).reshape(-1, 3).astype(np.float32)
    x = grid * np.float32(h)
    x = (x + np.float32(0.001 * h) * np.random.default_rng(seed).standard_normal(x.shape).astype(np.float32)).astype(np.float32)
    return x, np.zeros_like(x)


def run(nx=25, ny=100, nz=25, frames=480, cell=False, seed=0):
    h = SMOOTHING_LENGTH
    domain = Box(x=80, y=80, z=80)
    x, v = initial_state(nx, ny, nz, h, seed)
    particle_mass = np.float32(0.01) * particle_volume(h)
    dt = 0.01 * h
    gravity = vec(x=0, y=0, z=-0.1)
    substeps = int(32 / h)

    def step(x, v, substeps=1):
        return sph_step(x, v, domain, h, particle_mass, dt, gravity, dynamic_visc=0.025, damping_coef=-0.95, substeps=substeps)

    if cell:
        return iterate(step, frames, x, v, substeps=substeps)
    for _ in range(frames):
        x, v = step(x, v, substeps)
    return x, v


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--nx', type=int, default=25)
    ap.add_argument('--ny', type=int, default=100)
    ap.add_argument('--nz', type=int, default=25)
    ap.add_argument('--frames', type=int, default=480)
    ap.add_argument('--cell', action='store_true', help="the notebook's iterate loop, one launch per substep")
    args = ap.parse_args(argv)
    x, v = run(args.nx, args.ny, args.nz, args.frames, args.cell)
    inside = bool(np.all((x >= 0) & (x <= 80)))
    print(f"{len(x)} particles after {args.frames} frames x {int(32 / SMOOTHING_LENGTH)} substeps: all inside the domain: {inside}, "
          f"finite: {bool(np.isfinite(x).all() and np.isfinite(v).all())}, extent x [{x[:, 0].min():.2f}, {x[:, 0].max():.2f}] "
          f"y [{x[:, 1].min():.2f}, {x[:, 1].max():.2f}] z [{x[:, 2].min():.2f}, {x[:, 2].max():.2f}], max |v| {np.abs(v).max():.3f}")


if __name__ == '__main__':
    main()
