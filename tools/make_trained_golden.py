""" Record tests/golden/trained/<name>.npz: each problem of tests/trained_state.FIXTURES trained with the fp64 oracle.

    python tools/make_trained_golden.py [problem names ...] [-j JOBS]

CPU only.  Each problem starts from its golden initial parameters (tests/golden/<name>.npz) and takes `steps` steps of
fp64 Adam (oracle/autograd_port.fit) on batches of tests/problems.make_points-style uniform points at fixed seeds.  The
fp64 oracle is then evaluated at the fixture's points (trained_state.fixture_points) for every variant.  torch runs on
one thread per problem, so that the same torch build on the same machine gives the same bits; problems run in parallel
processes (-j, default: the CPU count).
"""
import argparse
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import trained_state as TS                                 # noqa: E402


def batches(name, batch, seed):
    ranges = TS.cfg_of(name)['ranges']

    def stream(i):
        rng = np.random.RandomState(seed * 100003 + i)
        cols = [rng.uniform(lo, hi, size=(batch, 1)) for lo, hi in ranges]
        return torch.from_numpy(np.concatenate(cols, axis=1).astype(np.float32)).to(torch.float64)
    return stream


def make(name):
    from oracle import autograd_port as ap
    torch.set_num_threads(1)
    t0 = time.time()
    family, steps, batch, lr, seed = TS.FIXTURES[name]
    init = TS.initial_params(name)
    pts = TS.fixture_points(name)
    loss0 = TS.evaluate(name, init, pts, chunks=1)['loss']
    prob = TS.oracle(name, torch.float64, init)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        losses = ap.fit(prob, steps, batch, lr=lr, point_stream=batches(name, batch, seed), criterion=TS.criterion_of(name))
    flat = prob.flat_params().numpy()
    trained = np.zeros(len(init), dtype=np.float32)
    trained[:TS.n_params(name)] = flat[:TS.n_params(name)].astype(np.float32)
    out = dict(trained=trained, points=pts)
    for v in TS.variant_names(name):
        X = TS.evaluate(name, TS.variant_params(name, trained, v), pts)
        for k, val in X.items():
            out['%s_%s' % (v, k)] = np.asarray(val, dtype=np.float64)
    loss1 = float(out['trained_loss'])
    out['meta'] = np.array([steps, lr, seed, batch, loss0, loss1], dtype=np.float64)
    out['train_losses'] = losses.astype(np.float64)
    os.makedirs(TS.TRAINED, exist_ok=True)
    np.savez_compressed(os.path.join(TS.TRAINED, name + '.npz'), **out)
    return '%-22s %-16s %5d steps  loss %.3e -> %.3e (x%.0f)  %.0f s' % (
        name, family, steps, loss0, loss1, loss0 / max(loss1, 1e-300), time.time() - t0)


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument('names', nargs='*')
    ap_.add_argument('-j', '--jobs', type=int, default=os.cpu_count())
    args = ap_.parse_args()
    names = args.names or list(TS.FIXTURES)
    with ProcessPoolExecutor(max_workers=max(1, min(args.jobs, len(names)))) as ex:
        for line in ex.map(make, names):
            print(line, flush=True)


if __name__ == '__main__':
    main()
