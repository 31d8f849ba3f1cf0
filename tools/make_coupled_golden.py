""" TEST INFRASTRUCTURE ONLY — generate tests/golden/<name>.npz for the problems of tests/problems_coupled.py (networks
with 2..4 outputs) from the UNMODIFIED reference, the way tools/make_system_golden.py does for tests/problems_systems.py:

    python tools/make_coupled_golden.py [problem names …]

Needs the reference checkout that oracle/make_golden.py imports; nothing at test / bench time runs this.  Recorded per
problem: params, points, residual [N, m], loss, grads (under the problem's criterion), u = Solver.predict [N, k], and
traj_* of the reference's own Solver.fit for the problems of GOLDEN_TRAJ.
"""
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import make_golden as MG                                 # noqa: E402  (puts the reference and tests/ on sys.path)
import problems_coupled as PC                            # noqa: E402


def build(name, seed=0):
    cfg = PC.PROBLEMS[name]
    torch.manual_seed(seed)
    solver = MG.ref.Solver(PC.bind(name, MG.ref.D, MG.ref_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                           initial_condition=PC.make_ic(name, MG.ref_V), boundary_condition=cfg['bc'], domain=cfg['domain'],
                           layout=cfg['layout'], features=cfg['features'], activation=cfg['activation'])
    if 'log_scale' in cfg:
        with torch.no_grad():
            solver.model.log_scale.fill_(cfg['log_scale'])
    return solver


def evaluate(solver, pts, criterion):
    """ MG.evaluate under the problem's criterion (reference :448 `criterion(residual, zeros)`). """
    for p in solver.model.parameters():
        p.grad = None
    xs = [torch.from_numpy(pts[:, i:i + 1].copy()).requires_grad_() for i in range(pts.shape[1])]
    u_hat = solver.ctx.run(solver.model, solver.reshape_and_concat(xs))
    residual = solver.ctx.run(solver.equation, u_hat, *xs)
    loss = criterion(residual, torch.zeros_like(xs[0]))
    loss.backward()
    return residual.detach().numpy(), float(loss.detach())


def main():
    warnings.filterwarnings('ignore', message='Using a target size')      # the [N, m] vs [N, 1] broadcast of :448
    outdir = os.path.join(ROOT, 'tests', 'golden')
    only = set(sys.argv[1:])
    for name, cfg in PC.PROBLEMS.items():
        if only and name not in only:
            continue
        var_names = list(cfg.get('variables', {}))
        crit = PC.torch_criterion(name)
        solver = build(name)
        pts = PC.make_points(name, PC.GOLDEN_BATCH[name], seed=123)
        params = MG.flat_of(solver, var_names)
        residual, loss = evaluate(solver, pts, crit)
        grads = MG.flat_of(solver, var_names, grads=True)
        u = np.asarray(solver.predict(*[pts[:, i] for i in range(pts.shape[1])]))
        assert residual.shape == (pts.shape[0], cfg['m']) and u.shape == (pts.shape[0], cfg['k']), (residual.shape, u.shape)
        out = dict(params=params, points=pts, residual=residual.astype(np.float32), loss=np.float32(loss), grads=grads,
                   u=u.astype(np.float32))
        if name in PC.GOLDEN_TRAJ:
            niters, batch, lr = PC.GOLDEN_TRAJ[name]
            solver = build(name)
            batches = [PC.make_points(name, batch, seed=1000 + i) for i in range(niters)]
            solver.fit(niters=niters, batch_size=batch, sampler=MG.Replay(batches), lr=lr, criterion=crit)
            out.update(traj_losses=np.asarray(solver.losses, dtype=np.float32),
                       traj_params=MG.flat_of(solver, var_names),
                       traj_meta=np.asarray([niters, batch, lr], dtype=np.float64))
        path = os.path.join(outdir, name + '.npz')
        np.savez_compressed(path, **out)
        print('%-20s B=%-4d k=%d m=%d P=%-6d loss=%.6e  |grad|=%.4e  -> %s' % (
            name, pts.shape[0], cfg['k'], cfg['m'], params.size, loss, float(np.linalg.norm(grads)),
            os.path.relpath(path, ROOT)))


if __name__ == '__main__':
    main()
