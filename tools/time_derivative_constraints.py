""" Whole `Solver.fit` steps of fits with a constraint that differentiates the solution at its points, fused against the
same constraint added by autograd (PYDENS_B200_FUSED_CONSTRAINTS=0, which is how every such constraint ran before):

- the oscillator u'' + (2 pi)^2 u = 0, u(0) = 1 by the ansatz, u'(0) = 0 by a constraint, batch 100 and 1 000: the
  fused fit runs in the persistent kernels (50 steps per launch), the autograd one a step launch, the constraint's
  autograd graph and torch's Adam per step;
- Poisson on the unit square with a 16-point Neumann flux constraint on x = 1, batch 100 000: one launch per step
  either way, the constraint a fused launch or an autograd graph.

    python tools/time_derivative_constraints.py [--steps K] [--runs R] [--out FILE.json]

The two paths alternate, R runs each; every run is warmed up and then timed over K steps (the Poisson fit: K / 5)
between two device synchronisations.  The card name and its power limit are read in the same call. """
import argparse
import json
import os
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
os.environ.setdefault('PYDENS_B200_PROGRESS', '0')

import numpy as np                                      # noqa: E402
import torch                                            # noqa: E402

from pydens_b200 import Solver, D                       # noqa: E402
from time_coupled import card                           # noqa: E402


def velocity(u, t):
    t0 = torch.tensor([0.0], requires_grad=True, device='cuda')
    return D(u(t0), t0)


def flux(u, x, y):
    x0 = torch.ones(16, requires_grad=True, device='cuda')
    return D(u(x0, torch.linspace(0.05, 0.95, 16, device='cuda')), x0) - 0.3


def oscillator():
    torch.manual_seed(0)
    return Solver(lambda u, t: D(D(u, t), t) + (2 * np.pi) ** 2 * u, ndims=1, initial_condition=1.0, layout='fafaf',
                  features=[12, 10, 1], activation='Tanh', constraints=velocity, device='cuda')


def poisson():
    torch.manual_seed(0)
    return Solver(lambda u, x, y: D(D(u, x), x) + D(D(u, y), y) - 5 * torch.sin(np.pi * (x + y)), ndims=2,
                  boundary_condition=1, layout='fa fa fa f', units=[10, 12, 15, 1], activation='Tanh',
                  constraints=flux, device='cuda')


def ms_per_step(make, batch, fused, steps):
    os.environ['PYDENS_B200_FUSED_CONSTRAINTS'] = '1' if fused else '0'
    solver = make()
    terms = ['equation', 'constraint_0']
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        solver.fit(niters=100, batch_size=batch, lr=0.005, loss_terms=terms)              # warm-up
        assert (solver._lower_constraint(0) is not None) == fused, 'not on the intended path'
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        solver.fit(niters=steps, batch_size=batch, lr=0.005, loss_terms=terms, optimizer=None)
        torch.cuda.synchronize()
    persistent = fused and not solver._engine._graphs        # an autograd constraint never runs persistent or captured
    return (time.perf_counter() - t0) * 1e3 / steps, persistent


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=1500)
    ap.add_argument('--runs', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    info = card()
    rows = []
    for name, make, batch, steps in (('oscillator', oscillator, 100, args.steps), ('oscillator', oscillator, 1000, args.steps),
                                     ('poisson_flux', poisson, 100000, max(1, args.steps // 5))):
        times = {'fused': [], 'autograd': []}
        paths = {}
        for _ in range(args.runs):
            for mode in ('fused', 'autograd'):
                t, persistent = ms_per_step(make, batch, mode == 'fused', steps)
                times[mode].append(t)
                paths[mode] = 'persistent' if persistent else 'stepwise'
        rows.append(dict(name=name, batch=batch, steps=steps, paths=paths, **{k + '_ms': v for k, v in times.items()}))
        print('%-12s batch %6d, %d steps: fused (%s) %s ms/step   autograd constraint (%s) %s ms/step' % (
            name, batch, steps, paths['fused'], ' '.join('%.4f' % t for t in times['fused']), paths['autograd'],
            ' '.join('%.4f' % t for t in times['autograd'])))
    os.environ.pop('PYDENS_B200_FUSED_CONSTRAINTS', None)
    print('card: %s' % info)
    if args.out:
        json.dump(dict(card=info, rows=rows), open(args.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
