""" Whole `fit_ensemble` calls of M members against the same M fits run one after another with `Solver.fit`, for the
tutorial's trainable-variable stage (batch 100, one constraint point) and the README flow with `V('init')` in the initial
condition (batch 150, one constraint point), at M = 1, 8, 16, 32, 64 and 128, in one call:

    python tools/time_ensemble.py [--steps K] [--runs R] [--members 1,8,...] [--out FILE.json]

Every member has its own initialisation and seed.  Both paths are warmed up (plans, optimizer state, one launch) on their
own solvers, then timed over K optimizer steps per member between two device synchronisations; the two paths alternate,
R runs each.  Reported: aggregate optimizer steps per second (M * K / time) and, at M = 1, the ensemble's time over the
solo fit's.  The card name and its power limit are read in the same run. """
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

from pydens_b200 import Solver, D, V, fit_ensemble      # noqa: E402
from time_coupled import card                           # noqa: E402


def tutorial5(j):
    torch.manual_seed(j)
    return Solver(lambda f, x: D(f, x) - 2 * np.pi * torch.cos(2 * np.pi * x) + V('new_var', data=torch.Tensor([1.0])),
                  ndims=1, initial_condition=1, constraints=lambda f, x: f(torch.tensor([0.5])), device='cuda',
                  backend='fused', seed=j), 100, 0.1


def readme(j):
    torch.manual_seed(j)
    return Solver(lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t), ndims=1,
                  initial_condition=lambda *a: V('init', data=torch.Tensor([3.0])), layout='fafaf', features=[12, 10, 1],
                  activation='Tanh', constraints=lambda u, t: u(torch.tensor([0.5])) - 0.25, device='cuda',
                  backend='fused', seed=j), 150, 0.05


TERMS = ['equation', 'constraint_0']


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=1500)
    ap.add_argument('--runs', type=int, default=2)
    ap.add_argument('--members', default='1,8,16,32,64,128')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_ensemble.py needs a CUDA device')
    info = card()
    rows = []
    for name, make in (('tutorial5', tutorial5), ('readme', readme)):
        for M in map(int, args.members.split(',')):
            ens = [make(j) for j in range(M)]
            solo = [make(j) for j in range(M)]
            batch, lr = ens[0][1], ens[0][2]
            ens, solo = [s for s, _, _ in ens], [s for s, _, _ in solo]
            with warnings.catch_warnings():
                warnings.simplefilter('error', UserWarning)          # both on the persistent path, no fallback
                fit_ensemble(ens, niters=50, batch_size=batch, lr=lr, loss_terms=TERMS)
                for s in solo:
                    s.fit(niters=50, batch_size=batch, lr=lr, loss_terms=TERMS)
                t_ens, t_solo = [], []
                for _ in range(args.runs):
                    t_ens.append(timed(lambda: fit_ensemble(ens, niters=args.steps, batch_size=batch, loss_terms=TERMS,
                                                            optimizer=None)))
                    t_solo.append(timed(lambda: [s.fit(niters=args.steps, batch_size=batch, loss_terms=TERMS,
                                                       optimizer=None) for s in solo]))
            row = dict(problem=name, members=M, steps=args.steps, batch=batch, ensemble_s=t_ens, solo_s=t_solo,
                       ensemble_steps_per_s=[M * args.steps / t for t in t_ens],
                       solo_steps_per_s=[M * args.steps / t for t in t_solo])
            rows.append(row)
            print('%-9s M=%3d  ensemble %s s (%s steps/s)   solo one after another %s s (%s steps/s)' % (
                name, M, ' '.join('%.4f' % t for t in t_ens), ' '.join('%.3g' % r for r in row['ensemble_steps_per_s']),
                ' '.join('%.4f' % t for t in t_solo), ' '.join('%.3g' % r for r in row['solo_steps_per_s'])), flush=True)
            del ens, solo
            torch.cuda.empty_cache()
        one = next(r for r in rows if r['problem'] == name and r['members'] == 1) if any(
            r['problem'] == name and r['members'] == 1 for r in rows) else None
        if one:
            print('%-9s M=1 overhead: ensemble / solo = %.3f' % (name, np.median(one['ensemble_s']) / np.median(one['solo_s'])))
    print('card: %s' % info)
    if args.out:
        json.dump(dict(card=info, rows=rows), open(args.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
