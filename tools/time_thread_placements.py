""" Step time of the thread kernel on the problems whose placement puts the per-warp gradient accumulators out of shared
memory (DESIGN §4a), and cfg2 as a control.  One JSON line per problem: the placement pinn_plan_info reports and the
median ms per step (CUDA events around `--steps` back-to-back steps on one fixed batch, `--reps` repetitions), with the
card's name and power limit.

    python tools/time_thread_placements.py [--steps 50] [--reps 5] [--out FILE]

To compare two builds, run it from each tree in turn, alternating, in one session on the same GPU. """
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import problems as P  # noqa: E402
from pydens_b200 import Solver, D, V  # noqa: E402

GELU64 = dict(equation=P._poisson2d, ndims=2, nparams=0, ic=None, bc=1, domain=(0, 1), features=[64, 64, 64, 1],
              activation='GELU', layout='fafafaf', ranges=[(0, 1), (0, 1)])
# (label, problem, batch, environment)
CASES = [('cfg3 ode_param', 'ode_param', 1000000, {}),
         ('ode_var', 'ode_var', 1000000, {}),
         ('wave3d thread kernel', 'wave3d', 500000, {'PINN_FORCE_KERNEL': 'thread'}),
         ('gelu64 [2, 64, 64, 64, 1] GELU', 'gelu64', 500000, {}),
         ('cfg2 poisson2d', 'poisson2d', 100000, {})]


def solver_for(name):
    cfg = GELU64 if name == 'gelu64' else P.PROBLEMS[name]
    torch.manual_seed(0)
    eq = cfg['equation']
    pkg_V = lambda n, init: V(n, data=torch.Tensor([init]))
    ic = cfg['ic_factory'](pkg_V) if 'ic_factory' in cfg else cfg['ic']
    return Solver(lambda u, *xs: eq(u, *xs, D=D, V=pkg_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                  initial_condition=ic, boundary_condition=cfg['bc'], domain=cfg['domain'], layout=cfg['layout'],
                  features=cfg['features'], activation=cfg['activation'], device='cuda', backend='fused', seed=1234)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    lines = []
    for label, name, n, env in CASES:
        saved = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            eng = solver_for(name)._get_engine()
        finally:
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        pts = eng.sample(n, None, step=1)
        for _ in range(5):
            eng._step(pts, None, n, 1.0 / n, 0, use_counter=False)
        times = []
        for _ in range(args.reps):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.steps):
                eng._step(pts, None, n, 1.0 / n, 0, use_counter=False)
            t1.record()
            torch.cuda.synchronize()
            times.append(t0.elapsed_time(t1) / args.steps)
        info = eng.info
        rec = dict(case=label, batch=n, gpu=smi, ms_per_step=float(np.median(times)), ms_min=min(times),
                   ms_max=max(times), state='smem' if info.activations_in_smem else 'gmem',
                   warps=info.threads_per_cta // 32, smem_bytes=info.smem_bytes, regs=info.regs_per_thread,
                   workspace_bytes=int(eng.workspace.numel()))
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
        del eng
    if args.out:
        with open(args.out, 'a') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
