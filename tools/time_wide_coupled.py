""" Whole `Solver.fit` steps of a coupled system on the usual flow-PINN size — 2-D steady incompressible Navier-Stokes in
(u, v, p) on four hidden layers of 100 units (tests/problems_wide_coupled.py: navier_stokes2d_wide), which the coupled
form of the 128-wide tile kernel trains — against the autograd path, at 100 k and 500 k points per batch, in one call:

    python tools/time_wide_coupled.py [--steps K] [--out FILE.json]

Each configuration is warmed up (graph capture, optimizer state, autograd's first pass), then timed over K steps between
two device synchronisations; the card name and its power limit are printed beside the numbers. """
import argparse
import json
import os
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
os.environ.setdefault('PYDENS_B200_PROGRESS', '0')

import torch                                            # noqa: E402

import problems_wide_coupled as PWC                     # noqa: E402
from pydens_b200 import Solver, D, V                    # noqa: E402
from time_coupled import card                           # noqa: E402

NAME = 'navier_stokes2d_wide'


def make(backend):
    cfg = PWC.PROBLEMS[NAME]
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        return Solver(PWC.bind(NAME, D, lambda n, init: V(n, data=torch.Tensor([init]))), ndims=cfg['ndims'],
                      boundary_condition=cfg['bc'], domain=cfg['domain'], layout=cfg['layout'], features=cfg['features'],
                      activation=cfg['activation'], device='cuda', backend=backend, seed=1)


def ms_per_step(backend, batch, steps):
    solver = make(backend)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        solver.fit(niters=max(8, steps // 4), batch_size=batch, lr=0.001)        # warm-up: capture, state, allocator
        if backend == 'fused':
            assert solver._engine is not None and solver._engine.info.tensor_core == 2, 'not on the 128-wide tile kernel'
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        solver.fit(niters=steps, batch_size=batch, lr=0.001, optimizer=None)
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    rows = []
    for batch in (100_000, 500_000):
        fused = ms_per_step('fused', batch, args.steps)
        autograd = ms_per_step('torch', batch, max(5, args.steps // 5))
        rows.append(dict(batch=batch, fused_ms=fused, autograd_ms=autograd, speedup=autograd / fused))
        print('%s k=3 batch %7d: fused %8.3f ms/step  autograd %9.3f ms/step  (x%.1f)'
              % (NAME, batch, fused, autograd, autograd / fused))
    info = card()
    print('card: %s' % info)
    if args.out:
        json.dump(dict(card=info, rows=rows), open(args.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
