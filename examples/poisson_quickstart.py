""" The reference README's first example (README.md:25-60), unchanged apart from the import: on an H100 the fit
runs in the fused kernel; without a GPU it falls back to the autograd path.

    python examples/poisson_quickstart.py            # 1500 steps of batch 100, like the README
"""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pydens import Solver, D                                   # noqa: E402  (drop-in alias of pydens_b200)


def pde(f, x, y):
    return D(D(f, x), x) + D(D(f, y), y) - 5 * torch.sin(np.pi * (x + y))


solver = Solver(equation=pde, ndims=2, boundary_condition=1,
                layout='fa fa fa f', activation='Tanh', units=[10, 12, 15, 1])
start = time.time()
solver.fit(batch_size=100, niters=1500)
print('fit: %.3f s, loss %.4f -> %.4f' % (time.time() - start, float(solver.losses[0]), float(solver.losses[-1])))

grid = np.linspace(0, 1, 100)
xs, ys = (a.reshape(-1) for a in np.meshgrid(grid, grid))
approx = solver.predict(xs, ys).reshape(100, 100)
print('u on a 100 x 100 grid: min %.3f max %.3f (boundary value 1 on the edges: %.3f)'
      % (approx.min(), approx.max(), approx[0].mean()))
