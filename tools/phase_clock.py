""" Where the time of a cfg2 fit step goes inside the thread kernel: builds the step kernel of cfg2 (NF = NS = 2) with
-DPINN_PHASE_CLOCK into a temporary directory, runs cfg2 steps on it and prints the clock64() cycles of each phase
(pinn_device.cuh, PINN_PHASE_*) summed over all warps, with their shares of a warp's time.  The reverse phases are per
linear layer (layer 0: the input layer's weight gradients); the butterflies are part of the reverse phases and are
listed again on their own.  The clock reads cost issue slots of their own, so the kernel runs a little slower than the
one build() makes; use the shares, not the cycle counts, to compare two trees.

    python tools/phase_clock.py [--steps 50] [--pool 128] [--out FILE]

To compare two builds, run it from each tree in turn in one session on the same GPU. """
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'pydens_b200', 'csrc')
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

LOAD, FWD, PROG, BFLY, TAIL, REV = 0, 1, 2, 3, 4, 5          # PINN_PHASE_* of pinn_device.cuh
N_SLOTS = REV + 16                                          # PINN_PHASE_SLOTS (PINN_MAX_LAYERS = 16)


def build_lib(tmp):
    """ The cfg2 step unit with the phase clock and the host side, linked into tmp/libpinn_phase.so. """
    import __graft_entry__ as g
    nvcc = g._nvcc()
    # the plan looks kernels up by their general variant too: the nf = 2 step_gen unit, without the clock
    units = [('phase', ['-DPINN_UNIT=PINN_STEP', '-DPINN_NF=2', '-DPINN_LO=2', '-DPINN_HI=2', '-DPINN_PHASE_CLOCK']),
             ('gen', ['-DPINN_UNIT=PINN_STEP_GEN', '-DPINN_NF=2', '-DPINN_LO=2', '-DPINN_HI=2'])]
    jobs = [(os.path.join(tmp, name + '.o'), 'pinn_instances.cu', defines) for name, defines in units]
    jobs.append((os.path.join(tmp, 'kernels.o'), 'pinn_kernels.cu', []))
    procs = [subprocess.Popen([nvcc] + g.NVCC_FLAGS + defines + ['-c', os.path.join(CSRC, src), '-o', obj])
             for obj, src, defines in jobs]
    if any(p.wait() != 0 for p in procs):
        raise RuntimeError('nvcc failed')
    objs = [obj for obj, _, _ in jobs]
    lib = os.path.join(tmp, 'libpinn_phase.so')
    subprocess.check_call([nvcc, '-shared', '-o', lib] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'])
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--pool', type=int, default=128, help='distinct batches cycled through (128 x 800 kB > L2)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix='pinn_phase_')
    lib_path = build_lib(tmp)
    os.environ['PYDENS_B200_LIB'] = lib_path

    import torch
    import problems as P
    from pydens_b200 import Solver, D, V

    cfg = P.PROBLEMS['poisson2d']
    n = 100000
    torch.manual_seed(0)
    solver = Solver(lambda u, *xs: cfg['equation'](u, *xs, D=D, V=V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                    initial_condition=cfg['ic'], boundary_condition=cfg['bc'], domain=cfg['domain'], layout=cfg['layout'],
                    features=cfg['features'], activation=cfg['activation'], device='cuda', backend='fused', seed=1234)
    eng = solver._get_engine()
    pool = [eng.sample(n, None, step=s) for s in range(args.pool)]
    lib = C.CDLL(lib_path)
    lib.pinn_phase_cycles_read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    cyc = (C.c_ulonglong * N_SLOTS)()
    for s in range(10):
        eng._step(pool[s % len(pool)], None, n, 1.0 / n, 0, use_counter=False)
    torch.cuda.synchronize()
    assert lib.pinn_phase_cycles_read(cyc, 1) == 0
    for s in range(args.steps):
        eng._step(pool[s % len(pool)], None, n, 1.0 / n, 0, use_counter=False)
    torch.cuda.synchronize()
    assert lib.pinn_phase_cycles_read(cyc, 0) == 0

    n_layers = len(cfg['features'])
    phases = [('load coordinates', LOAD), ('forward', FWD), ('program and ansatz', PROG)]
    phases += [('reverse, layer %d' % l, REV + l) for l in range(n_layers - 1, -1, -1)]
    phases += [('grid tail', TAIL)]
    total = sum(cyc[s] for _, s in phases)
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    rec = {'tree': ROOT, 'gpu': smi, 'steps': args.steps, 'warp_cycles_per_step': total / args.steps,
           'share': {name: cyc[s] / total for name, s in phases}}
    rec['share']['of which butterflies'] = cyc[BFLY] / total
    print('%-26s %14s %7s' % ('phase (cfg2)', 'cycles/step', 'share'))
    for name, s in phases + [('of which butterflies', BFLY)]:
        print('%-26s %14.4g %6.1f%%' % (name, cyc[s] / args.steps, 100.0 * cyc[s] / total))
    print(json.dumps(rec), flush=True)
    if args.out:
        with open(args.out, 'a') as f:
            f.write(json.dumps(rec) + '\n')


if __name__ == '__main__':
    main()
