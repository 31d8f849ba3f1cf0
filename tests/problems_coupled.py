""" Coupled systems: networks with k = 2..4 outputs whose equation selects component j of the [N, k] output
(f[:, j:j+1], f[:, [j]], f[..., j:j+1], torch.split, torch.chunk) and returns the residuals of all equations with
torch.cat.  The reference broadcasts its ansatz over the k components (model_torch.py:118-127: the same boundary value,
boundary factor, time gate and initial condition apply to each) and `predict` returns [N, k].

Shared by tools/make_coupled_golden.py, which records tests/golden/<name>.npz from the unmodified reference, and the
tests of this feature.  Same layout as tests/problems_systems.py, plus `k` (outputs) and `m` (residual columns); a
problem may name its `criterion` (('huber', delta) for nn.HuberLoss(delta=delta)).
"""
import numpy as np
import torch


def _lotka_volterra(f, t, D, V):                      # ODE pair, V coefficient, initial condition
    u, v = f[:, 0:1], f[:, 1:2]
    a = V('alpha', 0.8)
    return torch.cat([D(u, t) - (a * u - 0.4 * u * v), D(v, t) - (0.3 * u * v - 0.6 * v)], dim=1)


def _navier_stokes(f, x, y, D, V):                    # 2-D steady incompressible Navier-Stokes in (u, v, p)
    u, v, p = torch.split(f, 1, dim=1)
    nu = 0.05
    ux, uy, vx, vy = D(u, x), D(u, y), D(v, x), D(v, y)
    mom_x = u * ux + v * uy + D(p, x) - nu * (D(ux, x) + D(uy, y))
    mom_y = u * vx + v * vy + D(p, y) - nu * (D(vx, x) + D(vy, y)) + torch.sin(np.pi * x)
    return torch.cat([mom_x, mom_y, ux + vy], dim=1)


def _brusselator(f, x, t, D, V):                      # 1-D reaction-diffusion pair in (x, t)
    u = f[..., 0:1]
    v = f[:, [1]]
    a, b = 1.0, 3.0
    uu = u * u * v
    return torch.cat([D(u, t) - 0.02 * D(D(u, x), x) - (a - (b + 1.0) * u + uu),
                      D(v, t) - 0.02 * D(D(v, x), x) - (b * u - uu)], dim=1)


def _icf_brusselator(V):
    return lambda x: 1.0 + V('amp', 0.5) * torch.sin(np.pi * x)


def _quad(f, x, y, D, V):                             # k = 4 on a residual layout, mixed activations
    a, b, c, d = torch.split(f, 1, dim=1)
    return torch.cat([D(D(a, x), x) + D(D(a, y), y) - b,
                      D(b, x) - c * torch.cos(y),
                      D(c, y) + d * a - 0.5,
                      d - D(a, x) * D(a, y)], dim=1)


PROBLEMS = {
    'lotka_volterra': dict(equation=_lotka_volterra, ndims=1, nparams=0, ic=0.5, bc=None, domain=[(0, 3)],
                           features=[16, 16, 2], activation='Tanh', layout='fafaf', variables={'alpha': 0.8},
                           ranges=[(0, 3)], log_scale=0.2, k=2, m=2),
    'navier_stokes2d': dict(equation=_navier_stokes, ndims=2, nparams=0, ic=None, bc=0.0, domain=[(0, 1), (0, 1)],
                            features=[20, 20, 3], activation='Tanh', layout='fafaf', ranges=[(0, 1), (0, 1)], k=3, m=3),
    'brusselator': dict(equation=_brusselator, ndims=2, nparams=0, ic=None, ic_factory=_icf_brusselator, bc=None,
                        domain=[(0, 1), (0, 2)], features=[12, 12, 2], activation='Sigmoid', layout='fafaf',
                        variables={'amp': 0.5}, ranges=[(0, 1), (0, 2)], log_scale=-0.1, k=2, m=2),
    'quad_resnet_huber': dict(equation=_quad, ndims=2, nparams=0, ic=None, bc=0.2, domain=[(-1, 1), (0, 2)],
                              features=[10, 10, 10, 4], activation=['Tanh', 'SiLU', 'Sigmoid'], layout='faR fa fa+ f',
                              ranges=[(-1, 1), (0, 2)], k=4, m=4, criterion=('huber', 0.5)),
}

GOLDEN_BATCH = {'lotka_volterra': 96, 'navier_stokes2d': 80, 'brusselator': 70, 'quad_resnet_huber': 66}
# a short Adam trajectory of the reference's own Solver.fit: name -> (niters, batch, lr)
GOLDEN_TRAJ = {'lotka_volterra': (20, 48, 0.01), 'navier_stokes2d': (15, 40, 0.005), 'brusselator': (15, 40, 0.01),
               'quad_resnet_huber': (15, 40, 0.01)}


def make_points(name, batch, seed):
    rng = np.random.RandomState(seed)
    cols = [rng.uniform(lo, hi, size=(batch, 1)) for lo, hi in PROBLEMS[name]['ranges']]
    return np.concatenate(cols, axis=1).astype(np.float32)


def layer_plan(name):
    cfg = PROBLEMS[name]
    acts, skips, stack = [], [], []
    spec = cfg['activation']
    spec = list(spec) if isinstance(spec, (list, tuple)) else [spec] * cfg['layout'].count('a')
    names = [(a if isinstance(a, str) else a.__name__).lower() for a in spec]
    i_a = 0
    for letter in cfg['layout'].replace(' ', ''):
        if letter == 'f':
            acts.append('none'); skips.append(None)
        elif letter == 'a':
            acts[-1] = names[i_a]
            i_a += 1
        elif letter == 'R':
            stack.append(len(acts) - 1)
        elif letter == '+':
            skips[-1] = stack.pop()
    return acts, skips


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
