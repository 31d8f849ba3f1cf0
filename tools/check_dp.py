""" Data-parallel consistency check, run under torchrun:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tools/check_dp.py OUT.json

Trains the README Poisson problem for a few steps with a fixed GLOBAL batch sampled in-kernel.  Because
the Philox counter is the global point index, every world size sees the same points, so the loss
curves must agree to fp32 reduction noise.  Rank 0 writes the curve to OUT.json. """
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
os.environ.setdefault('PYDENS_B200_PROGRESS', '0')

import numpy as np                # noqa: E402
import torch                      # noqa: E402
import torch.distributed as dist  # noqa: E402


def main():
    out = sys.argv[1]
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    from pydens_b200 import Solver, D, V

    def pde(f, x, y):
        return D(D(f, x), x) + D(D(f, y), y) - 5 * torch.sin(np.pi * (x + y))
    torch.manual_seed(0)
    problem = sys.argv[2] if len(sys.argv) > 2 else 'readme'
    if problem == 'readme':
        solver = Solver(pde, ndims=2, boundary_condition=1, layout='fa fa fa f', activation='Tanh',
                        units=[10, 12, 15, 1], device=torch.device('cuda', local), backend='fused', seed=7)
        solver.fit(niters=30, batch_size=100001, lr=0.005)          # odd size: uneven shards
    else:                                  # a registry problem, e.g. wave3d: the tensor-core tile kernel under data parallelism
        import problems as P
        import problems_wide as PW         # ... or a 128-wide network (poisson_wide128)
        import problems_coupled as PC      # ... or a network of several outputs (navier_stokes2d)
        import problems_wide_coupled as PWC    # ... or both (navier_stokes2d_wide)
        if problem in PW.PROBLEMS:
            P = PW
        elif problem in PC.PROBLEMS:
            P = PC
        elif problem in PWC.PROBLEMS:
            P = PWC
        cfg = P.PROBLEMS[problem]
        solver = Solver(P.bind(problem, D, lambda n, init: V(n, data=torch.Tensor([init]))), ndims=cfg['ndims'],
                        nparams=cfg['nparams'], initial_condition=cfg['ic'], boundary_condition=cfg['bc'],
                        domain=cfg['domain'], layout=cfg['layout'], features=cfg['features'],
                        activation=cfg['activation'], device=torch.device('cuda', local), backend='fused', seed=7)
        solver.fit(niters=30, batch_size=40001, lr=0.001)
    losses = [float(v) for v in solver.losses]
    flat = solver.flat_params()
    if world > 1:
        ref = flat.clone()
        dist.broadcast(ref, 0)
        assert torch.equal(ref, flat), 'replicas diverged'
    if (not dist.is_initialized()) or dist.get_rank() == 0:
        eng = solver._get_engine()
        json.dump({'world': world, 'losses': losses, 'params_norm': float(flat.norm()), 'tensor_core': int(eng.info.tensor_core),
                   'allreduce': 'peer' if eng.comm is not None else ('nccl' if world > 1 else 'none')}, open(out, 'w'))
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
