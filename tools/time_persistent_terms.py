""" Whole `Solver.fit` steps of the fits with a constraint term that the persistent kernels now take — the tutorial's
trainable-variable stage (batch 100, `loss_terms=['equation', 'constraint_0']`) and the README flow with `V('init')` in
the initial condition and a constraint at t = 0.5 (batch 150) — against one launch per step (PYDENS_B200_AUTO_PERSISTENT=0:
equation step, constraint step, `add_`, torch's Adam and the loss record in a captured graph), in one call:

    python tools/time_persistent_terms.py [--steps K] [--runs R] [--out FILE.json]

The two paths alternate, R runs each; every run is warmed up (plans, graph capture, optimizer state) and then timed over
K steps between two device synchronisations.  The card name and its power limit are printed beside the numbers. """
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

from pydens_b200 import Solver, D, V                    # noqa: E402
from time_coupled import card                           # noqa: E402


def tutorial5():
    torch.manual_seed(0)
    return Solver(lambda f, x: D(f, x) - 2 * np.pi * torch.cos(2 * np.pi * x) + V('new_var', data=torch.Tensor([1.0])),
                  ndims=1, initial_condition=1, constraints=lambda f, x: f(torch.tensor([0.5])), device='cuda',
                  backend='fused'), 100, 0.1


def readme():
    torch.manual_seed(0)
    return Solver(lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t), ndims=1,
                  initial_condition=lambda *a: V('init', data=torch.Tensor([3.0])), layout='fafaf', features=[12, 10, 1],
                  activation='Tanh', constraints=lambda u, t: u(torch.tensor([0.5])) - 0.25, device='cuda',
                  backend='fused'), 150, 0.05


def ms_per_step(make, persistent, steps):
    os.environ['PYDENS_B200_AUTO_PERSISTENT'] = '1' if persistent else '0'
    solver, batch, lr = make()
    terms = ['equation', 'constraint_0']
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)
        solver.fit(niters=200, batch_size=batch, lr=lr, loss_terms=terms)             # warm-up
        assert (not solver._engine._graphs) == persistent, 'not on the intended path'
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        solver.fit(niters=steps, batch_size=batch, lr=lr, loss_terms=terms, optimizer=None)
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=1500)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    rows = []
    for name, make in (('tutorial5', tutorial5), ('readme', readme)):
        times = {'persistent': [], 'stepwise': []}
        for _ in range(args.runs):
            for mode in ('persistent', 'stepwise'):
                times[mode].append(ms_per_step(make, mode == 'persistent', args.steps))
        rows.append(dict(name=name, steps=args.steps, **{k + '_ms': v for k, v in times.items()}))
        print('%-10s %d steps: persistent %s ms/step   stepwise %s ms/step' % (
            name, args.steps, ' '.join('%.4f' % t for t in times['persistent']),
            ' '.join('%.4f' % t for t in times['stepwise'])))
    info = card()
    print('card: %s' % info)
    if args.out:
        json.dump(dict(card=info, rows=rows), open(args.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
