""" Step time of the 128-wide class of the tensor-core tile kernel (DESIGN §4b, §8), with the card's name and power limit.

    python tools/time_wide_tile.py [--steps 20] [--reps 5] [--out FILE]

Two comparisons, one JSON line per measurement:
1. a 4 x 128 tanh network on the README Poisson equation (the thread kernel cannot hold it) at 100 000 and 500 000
   points: whole `Solver.fit` steps (sampling, step, Adam) of the fused path on this kernel against the autograd path
   (backend='torch') on the same device; median of `--reps` windows of `--steps` steps, host clock around a device
   synchronise;
2. networks both kernels hold ([128, 128] and [100, 100] hidden units, five jet channels, 500 000 points): one step on
   a fixed batch, the 128-wide tile kernel (PINN_FORCE_KERNEL=wide128) against the thread kernel
   (PINN_FORCE_KERNEL=thread), alternating, `--reps` windows of `--steps` steps each between CUDA events; the two
   kernels' loss and gradient are compared (relative difference). """
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
os.environ.setdefault('PYDENS_B200_PROGRESS', '0')

import numpy as np  # noqa: E402
import torch  # noqa: E402

import problems as P  # noqa: E402
from pydens_b200 import Solver, D  # noqa: E402


def poisson(features, backend='fused', force=None):
    saved = os.environ.pop('PINN_FORCE_KERNEL', None)
    if force:
        os.environ['PINN_FORCE_KERNEL'] = force
    try:
        torch.manual_seed(0)
        solver = Solver(lambda u, x, y: P._poisson2d(u, x, y, D=D, V=None), ndims=2, boundary_condition=1,
                        layout='fa' * (len(features) - 1) + 'f', features=features, activation='Tanh', device='cuda',
                        backend=backend, seed=1234)
        if backend == 'fused':
            solver._get_engine()                         # the plan is made under this PINN_FORCE_KERNEL
        return solver
    finally:
        os.environ.pop('PINN_FORCE_KERNEL', None)
        if saved is not None:
            os.environ['PINN_FORCE_KERNEL'] = saved


def time_fit(solver, n, steps, reps):
    solver.fit(niters=3, batch_size=n, lr=1e-4)               # warm-up: plan, graphs, optimizer state
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        solver.fit(niters=steps, batch_size=n, lr=1e-4)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3 / steps)
    return times


def time_step(eng, pts, steps):
    n = pts.shape[0]
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        eng._step(pts, None, n, 1.0 / n, 0, use_counter=False)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    print('gpu:', smi, flush=True)
    lines = []

    def emit(rec):
        rec['gpu'] = smi
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    # 1. the 4 x 128 network: this kernel against the autograd path
    features = [128, 128, 128, 128, 1]
    for n in (100000, 500000):
        fused = poisson(features)
        info = fused._get_engine().info
        assert info.tensor_core == 2, 'the 128-wide tile kernel does not run the 4 x 128 network'
        t_fused = time_fit(fused, n, args.steps, args.reps)
        del fused
        torch.cuda.empty_cache()
        auto = poisson(features, backend='torch')
        t_auto = time_fit(auto, n, max(2, args.steps // 4), args.reps)
        del auto
        torch.cuda.empty_cache()
        emit(dict(case='4x128 fit step', batch=n, kernel='wide128', ms_per_step=float(np.median(t_fused)),
                  ms_min=min(t_fused), ms_max=max(t_fused), autograd_ms_per_step=float(np.median(t_auto)),
                  autograd_ms_min=min(t_auto), autograd_ms_max=max(t_auto),
                  speedup=float(np.median(t_auto) / np.median(t_fused)), regs=info.regs_per_thread))

    # 2. networks both kernels hold: the 128-wide tile kernel forced against the thread kernel
    for hidden in ([128, 128], [100, 100]):
        n = 500000
        tile = poisson(hidden + [1], force='wide128')._get_engine()
        thread = poisson(hidden + [1], force='thread')._get_engine()
        assert tile.info.tensor_core == 2 and thread.info.tensor_core == 0
        pts = tile.sample(n, None, step=1)
        outs = []
        for eng in (tile, thread):
            eng.flat.copy_(tile.flat)
            for _ in range(3):
                eng._step(pts, None, n, 1.0 / n, 0, use_counter=False)
            torch.cuda.synchronize()
            outs.append(eng.out.clone())
        t_tile, t_thread = [], []
        for _ in range(args.reps):                              # alternating
            t_tile.append(time_step(tile, pts, args.steps))
            t_thread.append(time_step(thread, pts, args.steps))
        npar = tile.n_params
        g_tile, g_thread = outs[0][:npar].double(), outs[1][:npar].double()
        emit(dict(case='[2, %s, 1] step' % ', '.join(map(str, hidden)), batch=n,
                  wide128_ms=float(np.median(t_tile)), wide128_ms_min=min(t_tile), wide128_ms_max=max(t_tile),
                  thread_ms=float(np.median(t_thread)), thread_ms_min=min(t_thread), thread_ms_max=max(t_thread),
                  thread_over_wide128=float(np.median(t_thread) / np.median(t_tile)),
                  loss_rel_diff=float(abs(outs[0][npar] - outs[1][npar]) / abs(outs[1][npar])),
                  grad_rel_l2_diff=float((g_tile - g_thread).norm() / g_thread.norm()),
                  wide128_regs=tile.info.regs_per_thread, thread_regs=thread.info.regs_per_thread,
                  thread_warps=thread.info.threads_per_cta // 32))
        del tile, thread
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'a') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
