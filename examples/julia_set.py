"""examples/grids/Julia_Set.ipynb on the H100 path (without plotting).  python examples/julia_set.py

The notebook's constants cell runs unmodified on the mirror (complex64 NumPy, as PhiML computes it); `belongs_to_julia_set` sampled
through CenteredGrid(lambda re, im: ...) is replaced by flow.julia_set, which counts all 100 Julia sets in one kernel launch.  The
grid's axes x and y stand for the notebook's re and im.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from phiflow_b200.flow import *  # noqa: E402,F401,F403
from phiflow_b200.flow import julia_set  # noqa: E402


def constants():
    c = 0.7885 * math.exp(1j*math.linspace(0, 2*PI, batch(time=100)))
    return c


def sample(c, iter_count=50):
    return julia_set(c, iter_count, Box(x=(-2, 2), y=(-2, 2)), x=256, y=256)


def main():
    c = constants()
    sampled = sample(c)
    counts = sampled.numpy()
    print(f"{counts.shape[0]} Julia sets at {counts.shape[1]}x{counts.shape[2]}, 50 iterations: mean count {counts.mean():.3f}, "
          f"cells that never reach |z| = 2: {np.mean(counts == 50):.4f}")
    return c, sampled


if __name__ == '__main__':
    main()
