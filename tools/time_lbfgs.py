""" L-BFGS on the fused path: the kernel time of one pinn_lbfgs_advance, and whole fit iterations of the device update
against torch.optim.LBFGS driven by the same fused evaluation and against the autograd path:

    python tools/time_lbfgs.py [--iters K] [--out FILE.json]

advance: cfg2 (poisson2d, ~400 parameters) and cfg5 (wave3d, ~13 k), history 10 and 100, a state filled with a full
history; CUDA events around 200 launches after 20 warm-up launches.  Iterations: poisson2d, batches of 10 k and 100 k,
strong-Wolfe line search, max_iter 20, K iterations after one warm-up iteration, host clock around work that ends in a
device synchronise; reported per iteration and per evaluation.  The card name and power limit are read in the same run.
"""
import argparse
import ctypes as C
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
from pydens_b200 import _native as N                    # noqa: E402
from time_coupled import card                           # noqa: E402

LS = dict(lr=1.0, max_iter=20, line_search_fn='strong_wolfe')


def advance_ms(name, history):
    s = make_solver(name)
    s.fit(history + 2, 2000, optimizer='LBFGS', lr=1.0, max_iter=1, history_size=history, tolerance_change=0.0,
          tolerance_grad=0.0)
    eng = s._get_engine()
    cfg, cur, mask = eng._lbfgs_bind(s.optimizer)
    status = torch.zeros(1, dtype=torch.int32, device=eng.device)
    flat, out = eng.flat.clone(), eng.out.clone()
    state = cur['state'].clone()

    def launch():
        N.check(eng.lib.pinn_lbfgs_advance(C.byref(cfg), C.c_int64(eng.n_params), C.c_void_p(flat.data_ptr()),
                                   C.c_void_p(out.data_ptr()), C.c_void_p(state.data_ptr()),
                                   C.c_void_p(status.data_ptr()), eng._stream()))
    for _ in range(20):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(200):
        launch()
    b.record()
    torch.cuda.synchronize()
    return dict(problem=name, n_params=eng.n_params, history=history, ring=int(N.PinnLbfgsState.from_buffer_copy(
        bytes(cur['state'][:C.sizeof(N.PinnLbfgsState)].cpu().numpy())).ring_count), ms=a.elapsed_time(b) / 200)


def fused_closure_fit(s, iters, batch):
    """ torch.optim.LBFGS over the fused evaluation (the batch the in-kernel sampler draws for the step) """
    eng = s._get_engine()
    opt = torch.optim.LBFGS([p for p in s.model.parameters() if p.requires_grad], **LS)
    n = [0]
    for i in range(iters):
        pts = eng.sample(batch, step=i)

        def closure():
            n[0] += 1
            loss, _, _ = eng.loss_and_grads(pts)
            return torch.tensor(loss)
        opt.step(closure)
    return n[0]


def iteration_rows(iters):
    rows = []
    for batch in (10_000, 100_000):
        for path in ('device', 'torch_over_fused', 'autograd'):
            with warnings.catch_warnings():
                warnings.simplefilter('ignore', UserWarning)
                s = make_solver('poisson2d', backend='torch' if path == 'autograd' else 'fused')
                if path == 'torch_over_fused':
                    fused_closure_fit(s, 1, batch)
                else:
                    s.fit(1, batch, optimizer='LBFGS', **LS)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if path == 'torch_over_fused':
                    evals = fused_closure_fit(s, iters, batch)
                else:
                    s.fit(iters, batch, optimizer='LBFGS', **LS)
                    st = s.optimizer.state[s.optimizer.param_groups[0]['params'][0]]
                    evals = int(st['func_evals'])
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
            rows.append(dict(path=path, batch=batch, iters=iters, evals=evals, ms_per_iter=1e3 * dt / iters,
                             ms_per_eval=1e3 * dt / max(evals, 1)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    res = dict(card=card(), advance=[advance_ms(n, m) for n in ('poisson2d', 'wave3d') for m in (10, 100)],
               iterations=iteration_rows(args.iters))
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
