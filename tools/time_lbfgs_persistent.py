""" L-BFGS in the persistent cluster kernel (pinn_lbfgs_multi) against the stepwise device L-BFGS (one step launch, one
pinn_lbfgs_advance and a 4-byte status read per evaluation), and fit_ensemble(optimizer='LBFGS') against the same fits
run solo one after another:

    python tools/time_lbfgs_persistent.py [--steps K] [--repeats R] [--out FILE.json]

Fits: poisson2d (cfg2's network) and ode_tanh (the tutorial's first ODE), batches 100 / 400 / 1 000, history 10 and
100, fixed step (lr 0.05) and strong Wolfe (lr 1), max_iter 20; K steps from the same start on both paths, the two
paths alternating R times after one warm-up fit each.  Ensembles: poisson2d, batch 100, strong Wolfe, M = 1, 8, 32,
128 members in one fit_ensemble call against M solo persistent fits.  Host clock around fit() calls, which end in a
device synchronise; reported per step and per evaluation (median, min and max over the repeats).  The card name and
power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
os.environ.setdefault('PYDENS_B200_PROGRESS', '0')

import numpy as np                                      # noqa: E402
import torch                                            # noqa: E402

from gpu_helpers import make_solver                     # noqa: E402
from pydens_b200 import fit_ensemble                    # noqa: E402
from time_coupled import card                           # noqa: E402


def settings(ls, history):
    return (dict(lr=1.0, max_iter=20, history_size=history, line_search_fn='strong_wolfe') if ls
            else dict(lr=0.05, max_iter=20, history_size=history))


def timed_fit(name, params, steps, batch, persistent, kw):
    """ one fit of `steps` L-BFGS steps from `params` -> (seconds, evaluations, final loss) """
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        s = make_solver(name, params=params)
    if persistent:
        os.environ.pop('PYDENS_B200_AUTO_PERSISTENT', None)
    else:
        os.environ['PYDENS_B200_AUTO_PERSISTENT'] = '0'
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s.fit(steps, batch, optimizer='LBFGS', **({'steps_per_launch': steps} if persistent else {}), **kw)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    finally:
        os.environ.pop('PYDENS_B200_AUTO_PERSISTENT', None)
    st = s.optimizer.state[s.optimizer.param_groups[0]['params'][0]]
    return dt, int(st['func_evals']), float(s.losses[-1])


def spread(xs):
    return dict(median=float(np.median(xs)), min=float(np.min(xs)), max=float(np.max(xs)))


def path_rows(steps, repeats):
    rows = []
    for name in ('poisson2d', 'ode_tanh'):
        params = make_solver(name).flat_params().cpu()
        for batch in (100, 400, 1000):
            for history in (10, 100):
                for ls in (False, True):
                    kw = settings(ls, history)
                    for persistent in (True, False):             # warm-up: modules, captures, allocations
                        timed_fit(name, params, 2, batch, persistent, kw)
                    per = {True: [], False: []}
                    for _ in range(repeats):
                        for persistent in (True, False):
                            per[persistent].append(timed_fit(name, params, steps, batch, persistent, kw))
                    row = dict(problem=name, batch=batch, history=history, line_search=ls, steps=steps)
                    for persistent, tag in ((True, 'persistent'), (False, 'stepwise')):
                        runs = per[persistent]
                        row[tag] = dict(ms_per_step=spread([1e3 * r[0] / steps for r in runs]),
                                        ms_per_eval=spread([1e3 * r[0] / max(r[1], 1) for r in runs]),
                                        evals=runs[0][1], final_loss=runs[0][2])
                    row['speedup_per_step'] = row['stepwise']['ms_per_step']['median'] / row['persistent']['ms_per_step']['median']
                    print(json.dumps(row), flush=True)
                    rows.append(row)
    return rows


def ensemble_rows(steps, repeats):
    rows = []
    kw = settings(True, 10)
    for M in (1, 8, 32, 128):
        t_ens, t_solo = [], []
        for r in range(repeats + 1):                            # r = 0: warm-up
            with warnings.catch_warnings():
                warnings.simplefilter('ignore', UserWarning)
                members = [make_solver('poisson2d', seed=j) for j in range(M)]
                solos = [make_solver('poisson2d', seed=j) for j in range(M)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fit_ensemble(members, steps, 100, optimizer='LBFGS', **kw)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            for s in solos:
                s.fit(steps, 100, optimizer='LBFGS', **kw)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if r:
                t_ens.append(1e3 * (t1 - t0))
                t_solo.append(1e3 * (t2 - t1))
        row = dict(members=M, steps=steps, batch=100, ensemble_ms=spread(t_ens), solo_ms=spread(t_solo),
                   speedup=float(np.median(t_solo) / np.median(t_ens)))
        print(json.dumps(row), flush=True)
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--only', choices=('paths', 'ensembles'), default=None)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    res = dict(card=card())
    if args.only != 'ensembles':
        res['paths'] = path_rows(args.steps, args.repeats)
    if args.only != 'paths':
        res['ensembles'] = ensemble_rows(args.steps, args.repeats)
    print(json.dumps(res['card']))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
