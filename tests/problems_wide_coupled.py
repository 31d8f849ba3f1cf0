""" Coupled systems (networks with k = 2..4 outputs) whose hidden layers are 65-128 units wide and whose weights do not
fit the thread kernel's shared memory: the coupled form of the 128-wide tile kernel (pydens_b200/csrc/pinn_wide_kernel.cuh)
takes them.  Shared by tools/make_wide_coupled_golden.py, which records tests/golden/<name>.npz from the unmodified
reference, and the tests of this feature.  Kept apart from tests/problems_coupled.py and tests/problems_wide.py, whose
registries other tests parametrise over and place on the thread kernel.

Same layout as tests/problems_coupled.py (`k` outputs, `m` residual columns, an optional `criterion`).
"""
import numpy as np
import torch

import problems_coupled as PC


def _react_diff(f, x, t, D, V):                       # 1-D reaction-diffusion pair, a trainable feed rate
    u, v = torch.chunk(f, 2, dim=1)
    b = V('feed', 2.5)
    uuv = u * u * v
    return torch.cat([D(u, t) - 0.05 * D(D(u, x), x) - (1.0 - (b + 1.0) * u + uuv),
                      D(v, t) - 0.05 * D(D(v, x), x) - (b * u - uuv)], dim=1)


def _icf_react_diff(V):
    return lambda x: 1.0 + V('amp', 0.4) * torch.sin(np.pi * x)


PROBLEMS = {
    # 2-D steady incompressible Navier-Stokes in (u, v, p) on the usual flow-PINN size: jet set (2, 2), k = 3
    'navier_stokes2d_wide': dict(equation=PC._navier_stokes, ndims=2, nparams=0, ic=None, bc=0.0,
                                 domain=[(0, 1), (0, 1)], features=[100, 100, 100, 100, 3], activation='Tanh',
                                 layout='fafafafaf', ranges=[(0, 1), (0, 1)], k=3, m=3),
    # k = 2 on mixed widths with an identity layer; V in the equation and in the initial condition
    'react_diff_wide': dict(equation=_react_diff, ndims=2, nparams=0, ic=None, ic_factory=_icf_react_diff, bc=None,
                            domain=[(0, 1), (0, 2)], features=[128, 100, 128, 2], activation=['Tanh', 'Sigmoid'],
                            layout='fa f fa f', variables={'amp': 0.4, 'feed': 2.5}, ranges=[(0, 1), (0, 2)],
                            log_scale=-0.1, k=2, m=2),
    # k = 4 on three 128-unit layers under HuberLoss
    'quad_wide128_huber': dict(equation=PC._quad, ndims=2, nparams=0, ic=None, bc=0.2, domain=[(-1, 1), (0, 2)],
                               features=[128, 128, 128, 4], activation=['Tanh', 'Sigmoid', 'Tanh'], layout='fafafaf',
                               ranges=[(-1, 1), (0, 2)], k=4, m=4, criterion=('huber', 0.5)),
}

GOLDEN_BATCH = {'navier_stokes2d_wide': 80, 'react_diff_wide': 72, 'quad_wide128_huber': 66}
# a short Adam trajectory of the reference's own Solver.fit: name -> (niters, batch, lr)
GOLDEN_TRAJ = {'navier_stokes2d_wide': (12, 48, 0.002), 'react_diff_wide': (12, 48, 0.005)}


def make_points(name, batch, seed):
    rng = np.random.RandomState(seed)
    cols = [rng.uniform(lo, hi, size=(batch, 1)) for lo, hi in PROBLEMS[name]['ranges']]
    return np.concatenate(cols, axis=1).astype(np.float32)


def layer_plan(name):
    """ (per-layer activation names, skip sources) of a dense layout """
    cfg = PROBLEMS[name]
    spec = cfg['activation']
    spec = list(spec) if isinstance(spec, (list, tuple)) else [spec] * cfg['layout'].count('a')
    names = iter(a.lower() for a in spec)
    acts = []
    for letter in cfg['layout'].replace(' ', ''):
        if letter == 'f':
            acts.append('none')
        elif letter == 'a':
            acts[-1] = next(names)
    return acts, [None] * len(acts)


def make_ic(name, V):
    cfg = PROBLEMS[name]
    return cfg['ic_factory'](V) if 'ic_factory' in cfg else cfg['ic']


def has_ic(name):
    cfg = PROBLEMS[name]
    return cfg['ic'] is not None or 'ic_factory' in cfg


def bind(name, D, V):
    eq = PROBLEMS[name]['equation']
    return lambda u, *xs: eq(u, *xs, D=D, V=V)


def torch_criterion(name):
    crit = PROBLEMS[name].get('criterion')
    if crit is None:
        return torch.nn.MSELoss()
    return torch.nn.HuberLoss(delta=crit[1])
