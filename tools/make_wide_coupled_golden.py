""" TEST INFRASTRUCTURE ONLY — generate tests/golden/<name>.npz for the problems of tests/problems_wide_coupled.py
(coupled systems on hidden layers 65-128 units wide) from the UNMODIFIED reference, the way
tools/make_coupled_golden.py does for tests/problems_coupled.py:

    python tools/make_wide_coupled_golden.py [problem names …]

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
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import make_golden as MG                                 # noqa: E402  (puts the reference and tests/ on sys.path)
from make_coupled_golden import evaluate                 # noqa: E402
import problems_wide_coupled as PWC                      # noqa: E402


def build(name, seed=0):
    cfg = PWC.PROBLEMS[name]
    torch.manual_seed(seed)
    solver = MG.ref.Solver(PWC.bind(name, MG.ref.D, MG.ref_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                           initial_condition=PWC.make_ic(name, MG.ref_V), boundary_condition=cfg['bc'],
                           domain=cfg['domain'], layout=cfg['layout'], features=cfg['features'],
                           activation=cfg['activation'])
    if 'log_scale' in cfg:
        with torch.no_grad():
            solver.model.log_scale.fill_(cfg['log_scale'])
    return solver


def main():
    warnings.filterwarnings('ignore', message='Using a target size')      # the [N, m] vs [N, 1] broadcast of :448
    outdir = os.path.join(ROOT, 'tests', 'golden')
    only = set(sys.argv[1:])
    for name, cfg in PWC.PROBLEMS.items():
        if only and name not in only:
            continue
        var_names = list(cfg.get('variables', {}))
        crit = PWC.torch_criterion(name)
        solver = build(name)
        pts = PWC.make_points(name, PWC.GOLDEN_BATCH[name], seed=123)
        params = MG.flat_of(solver, var_names)
        residual, loss = evaluate(solver, pts, crit)
        grads = MG.flat_of(solver, var_names, grads=True)
        u = np.asarray(solver.predict(*[pts[:, i] for i in range(pts.shape[1])]))
        assert residual.shape == (pts.shape[0], cfg['m']) and u.shape == (pts.shape[0], cfg['k']), (residual.shape, u.shape)
        out = dict(params=params, points=pts, residual=residual.astype(np.float32), loss=np.float32(loss), grads=grads,
                   u=u.astype(np.float32))
        if name in PWC.GOLDEN_TRAJ:
            niters, batch, lr = PWC.GOLDEN_TRAJ[name]
            solver = build(name)
            batches = [PWC.make_points(name, batch, seed=1000 + i) for i in range(niters)]
            solver.fit(niters=niters, batch_size=batch, sampler=MG.Replay(batches), lr=lr, criterion=crit)
            out.update(traj_losses=np.asarray(solver.losses, dtype=np.float32),
                       traj_params=MG.flat_of(solver, var_names),
                       traj_meta=np.asarray([niters, batch, lr], dtype=np.float64))
        path = os.path.join(outdir, name + '.npz')
        np.savez_compressed(path, **out)
        print('%-22s B=%-4d k=%d m=%d P=%-6d loss=%.6e  |grad|=%.4e  -> %s (%d B)' % (
            name, pts.shape[0], cfg['k'], cfg['m'], params.size, loss, float(np.linalg.norm(grads)),
            os.path.relpath(path, ROOT), os.path.getsize(path)))


if __name__ == '__main__':
    main()
