"""examples/particles/Streamlines.ipynb on the H100 path (without plotting).  python examples/streamlines.py [--n 256]

The notebook's cells run on the mirror API, with three differences:
  * `Noise(vector='x,y')` is not in the mirror: `smooth_noise` below stands in for it with seeded Gaussian-filtered white noise per
    component, as examples/reaction_diffusion.py does; `fluid.make_incompressible` then projects it as in the notebook;
  * the 8 x 8 start points are the cell centres of CenteredGrid(0, 0, domain, x=8, y=8) from `axis_centres()` (PhiML's float32
    centres bit for bit; `points()` forms them in float64 and can differ by one ulp);
  * plotting and the named-dimension post-processing (`x_trj.iter[1:] - x_trj.iter[:-1]`, `math.vec_length`, `math.sum(.., 'iter')`)
    are done in NumPy on the stacked trajectory.
Both trajectories are computed twice: with `iterate` over `advect.points` (one kernel launch per step) and with `streamlines` (all 50
steps in one launch); the two must agree bit for bit.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403


def smooth_noise(shape, scale=20.0, seed=0):
    """Stand-in for one component of Noise(): white noise low-pass filtered at wavelengths around `scale` cells, unit std."""
    white = np.random.default_rng(seed).standard_normal(shape)
    k = np.meshgrid(*[np.fft.fftfreq(n) for n in shape], indexing='ij')
    a = np.fft.ifftn(np.fft.fftn(white) * np.exp(-0.5 * (np.hypot(*k) * scale) ** 2)).real
    return ((a - a.mean()) / a.std()).astype(np.float32)


def run(n=256, iterations=50, step_size=.1):
    domain = Box(x=10, y=10)
    v = StaggeredGrid([smooth_noise((n - 1, n), seed=1), smooth_noise((n, n - 1), seed=2)], 0, domain, x=n, y=n)
    v, _ = fluid.make_incompressible(v)

    def move_along_field(x, step_size=step_size):
        return advect.points(geom.Point(x), v, step_size, integrator=advect.rk4).center

    x0 = vec(x=5, y=5)
    x_trj = np.array(iterate(move_along_field, spatial(iter=iterations), x0), np.float32)
    cx, cy = CenteredGrid(0, 0, domain, x=8, y=8).axis_centres()
    X, Y = np.meshgrid(cx, cy, indexing='ij')
    starts = np.stack([X.ravel(), Y.ravel()], -1)
    s_trj = np.stack(iterate(move_along_field, spatial(iter=iterations), starts))
    fused_one = streamlines(x0, v, step_size, iterations)
    fused = streamlines(starts, v, step_size, iterations)
    assert np.array_equal(fused_one, x_trj) and np.array_equal(fused, s_trj), "streamlines differs from iterate over advect.points"
    distance = np.linalg.norm(np.diff(s_trj, axis=0), axis=-1).sum(0)
    return x_trj, s_trj, distance


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=256)
    args = ap.parse_args()
    x_trj, s_trj, distance = run(args.n)
    print(f"(5, 5) -> ({x_trj[-1, 0]:.4f}, {x_trj[-1, 1]:.4f}) after {len(x_trj) - 1} RK4 steps; 64 streamlines, distance travelled "
          f"min {distance.min():.3f} mean {distance.mean():.3f} max {distance.max():.3f}; streamlines == iterate bit for bit")


if __name__ == '__main__':
    main()
