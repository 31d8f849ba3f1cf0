""" Learning-rate sweeps in one `fit_ensemble` call against the same M fits run one after another with `Solver.fit`, for
the two problems of tools/time_ensemble.py (tutorial stage 5, batch 100; README `V('init')` flow, batch 150; one
constraint point each), at M = 8, 32 and 128; and the per-member hyper-parameter load against the build before it:

    python tools/time_ensemble_sweep.py [--steps K] [--runs R] [--members 8,32,128] [--parent-lib SO] [--out FILE.json]

Sweep: member j trains with lr_j spaced geometrically from a tenth of the problem's lr to the lr itself.  Both paths are
warmed up (plans, optimizer state, one launch) on their own solvers, then timed over K optimizer steps per member between
two device synchronisations, alternating, R runs each.  Reported: aggregate optimizer steps per second (M * K / time).

--parent-lib: a libpinn_b200.so built from the parent commit (same ABI version).  Equal-hyper ensembles of M = 8 and 128
members then run through the bare C calls of both libraries on the same problem and member state, 50 steps per launch,
K / 50 launches timed with CUDA events: the parent's pinn_multi_step_ensemble, this build's pinn_multi_step_ensemble
and this build's pinn_multi_step_ensemble_adam with equal rows, alternated R times.  The card name and its power limit
are read in the same run. """
import argparse
import ctypes as C
import json
import os
import sys
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
os.environ.setdefault('PYDENS_B200_PROGRESS', '0')

import numpy as np                                      # noqa: E402
import torch                                            # noqa: E402

from pydens_b200 import fit_ensemble, _native as N      # noqa: E402
from time_coupled import card                           # noqa: E402
from time_ensemble import TERMS, readme, timed, tutorial5   # noqa: E402

PROBLEMS = (('tutorial5', tutorial5), ('readme', readme))


def sweep_rows(args):
    rows = []
    for name, make in PROBLEMS:
        for M in map(int, args.members.split(',')):
            ens = [make(j) for j in range(M)]
            solo = [make(j) for j in range(M)]
            batch, lr = ens[0][1], ens[0][2]
            ens, solo = [s for s, _, _ in ens], [s for s, _, _ in solo]
            lrs = [float(x) for x in np.geomspace(lr / 10, lr, M)]
            with warnings.catch_warnings():
                warnings.simplefilter('error', UserWarning)          # both on the persistent path, no fallback
                fit_ensemble(ens, niters=50, batch_size=batch, lr=lrs, loss_terms=TERMS)
                for s, lr_j in zip(solo, lrs):
                    s.fit(niters=50, batch_size=batch, lr=lr_j, loss_terms=TERMS)
                t_ens, t_solo = [], []
                for _ in range(args.runs):
                    t_ens.append(timed(lambda: fit_ensemble(ens, niters=args.steps, batch_size=batch, loss_terms=TERMS,
                                                            optimizer=None)))
                    t_solo.append(timed(lambda: [s.fit(niters=args.steps, batch_size=batch, loss_terms=TERMS,
                                                       optimizer=None) for s in solo]))
            row = dict(problem=name, members=M, steps=args.steps, batch=batch, lr=[lrs[0], lrs[-1]], ensemble_s=t_ens,
                       solo_s=t_solo, ensemble_steps_per_s=[M * args.steps / t for t in t_ens],
                       solo_steps_per_s=[M * args.steps / t for t in t_solo])
            rows.append(row)
            print('sweep %-9s M=%3d  lr %.3g..%.3g  ensemble %s steps/s   solo one after another %s steps/s' % (
                name, M, lrs[0], lrs[-1], ' '.join('%.3g' % r for r in row['ensemble_steps_per_s']),
                ' '.join('%.3g' % r for r in row['solo_steps_per_s'])), flush=True)
            del ens, solo
            torch.cuda.empty_cache()
    return rows


class _Lib:
    """ one libpinn_b200.so with a plan of the engine's problem and of its constraint """

    def __init__(self, lib, eng, own):
        self.lib = lib
        if own:
            self.plan, self.term = eng.plan, eng._constraint_plan(0)['plan']
        else:
            lib.pinn_plan_create.argtypes = [C.POINTER(N.PinnSpec), C.c_int, C.POINTER(C.c_void_p)]
            lib.pinn_multi_step_ensemble.argtypes = N.load().pinn_multi_step_ensemble.argtypes
            lib.pinn_last_error.restype = C.c_char_p
            self.plan, self.term = C.c_void_p(), C.c_void_p()
            for spec, out in ((eng.spec, self.plan), (eng._constraint_plan(0)['spec'], self.term)):
                if lib.pinn_plan_create(C.byref(spec), 0, C.byref(out)) != 0:
                    raise RuntimeError(lib.pinn_last_error().decode())


def parent_rows(args):
    """ equal-hyper ensembles through the bare C calls: the parent library against this one, alternated """
    parent = C.CDLL(os.path.abspath(args.parent_lib))
    if parent.pinn_abi_version() != N.ABI_VERSION:
        raise SystemExit('%s: ABI %d, this build %d' % (args.parent_lib, parent.pinn_abi_version(), N.ABI_VERSION))
    k, launches = 50, max(1, args.steps // 50)
    rows = []
    for name, make in PROBLEMS:
        s, batch, lr = make(0)
        eng = s._get_engine()
        entry = eng._constraint_plan(0)
        libs = dict(parent=_Lib(parent, eng, False), this=_Lib(eng.lib, eng, True))
        for M in (8, 128):
            n = eng.n_params
            bufs = [dict(p=eng.flat.clone(), m=torch.zeros(n, device='cuda'), v=torch.zeros(n, device='cuda'),
                         mask=torch.ones(n, device='cuda'), steps=torch.zeros(4, device='cuda'),
                         counter=torch.zeros(1, dtype=torch.int64, device='cuda'), ring=torch.zeros(k, device='cuda'))
                    for _ in range(M)]
            table = (N.PinnMember * M)()
            for j, (t, b) in enumerate(zip(table, bufs)):
                t.params, t.exp_avg, t.exp_avg_sq, t.mask = (b['p'].data_ptr(), b['m'].data_ptr(), b['v'].data_ptr(),
                                                             b['mask'].data_ptr())
                t.step_tensors, t.n_step_tensors, t.points = b['steps'].data_ptr(), 4, None
                t.seed, t.step_counter, t.losses_ring = 1000 + j, b['counter'].data_ptr(), b['ring'].data_ptr()
            hyper = (N.PinnAdamHyper * M)()
            for h in hyper:
                h.lr, h.beta1, h.beta2, h.eps, h.weight_decay = lr, 0.9, 0.999, 1e-8, 0.0
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

            def launch(which):
                L = libs['parent' if which == 'parent' else 'this']
                terms = (N.PinnTerm * 1)()
                terms[0].plan, terms[0].n_points, terms[0].point_weight = L.term.value, entry['n'], 1.0 / entry['n']
                terms[0].points = entry['host_points'].data_ptr()
                for _ in range(launches):
                    if which == 'this_adam':
                        rc = L.lib.pinn_multi_step_ensemble_adam(L.plan, M, table, hyper, C.c_int64(batch), C.c_int(k),
                                                                 C.c_int64(k), C.c_float(1.0 / batch), C.c_int(1), terms,
                                                                 None, stream)
                    else:
                        rc = L.lib.pinn_multi_step_ensemble(L.plan, M, table, C.c_int64(batch), C.c_int(k),
                                                            C.c_float(lr), C.c_float(0.9), C.c_float(0.999),
                                                            C.c_float(1e-8), C.c_float(0.0), C.c_int64(k),
                                                            C.c_float(1.0 / batch), C.c_int(1), terms, None, stream)
                    if rc != 0:
                        raise RuntimeError('%s: %s' % (which, L.lib.pinn_last_error().decode()))

            def event_time(which):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                launch(which)
                b.record()
                torch.cuda.synchronize()
                return a.elapsed_time(b) * 1e-3

            whiches = ('parent', 'this', 'this_adam')
            for w in whiches:
                launch(w)                                            # warm-up: module load, first launch
            times = {w: [] for w in whiches}
            for _ in range(args.runs):
                for w in whiches:
                    times[w].append(event_time(w))
            us = {w: [1e6 * t / (launches * k) for t in ts] for w, ts in times.items()}
            rows.append(dict(problem=name, members=M, steps=launches * k, us_per_step=us,
                             steps_per_s={w: [M * launches * k / t for t in ts] for w, ts in times.items()}))
            print('equal rows %-9s M=%3d  us per launch-step: %s' % (name, M, '   '.join(
                '%s %s' % (w, ' '.join('%.2f' % x for x in xs)) for w, xs in us.items())), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=1500)
    ap.add_argument('--runs', type=int, default=2)
    ap.add_argument('--members', default='8,32,128')
    ap.add_argument('--parent-lib', default=None)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_ensemble_sweep.py needs a CUDA device')
    info = card()
    out = dict(card=info, sweep=sweep_rows(args))
    if args.parent_lib:
        out['parent'] = parent_rows(args)
    print('card: %s' % info)
    if args.out:
        json.dump(out, open(args.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
