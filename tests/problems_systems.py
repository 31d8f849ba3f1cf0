""" Equations with a residual of several columns, `torch.cat([r_1, …, r_m], dim=1)` (reference model_torch.py:448:
`criterion(residual[N, m], zeros[N, 1])` broadcasts, so the loss is the criterion over all N m entries), on a network
with one output.  Shared by tools/make_system_golden.py, which records tests/golden/<name>.npz from the unmodified
reference, and the tests of this feature.

Same layout as tests/problems.py (`eq(f, *xs, D=..., V=...)`, one dict per problem); a golden's `residual` is the
reference's [N, m] matrix.  The equations pick their column with the forms users write for systems: f[:, 0:1],
torch.split, f[..., 0:1], and concatenate with torch.cat / hstack / column_stack.
"""
import numpy as np
import torch

import problems as P


def _burgers_penalty(f, x, t, D, V):                 # Burgers plus two penalty columns (thread kernel, two directions)
    u = f[:, 0:1]
    ux = D(u, x)
    return torch.cat([D(u, t) + u * ux - 0.01 * D(ux, x), 0.3 * (ux + torch.sin(x)), u * u - 0.25], dim=1)


def _heat_pair(f, x, t, D, V):                       # variables in both columns and in the initial condition, skip layout
    (u,) = torch.split(f, 1, dim=1)
    return torch.hstack([0.3 * D(D(u, x), x) - D(u, t) + V('src', 0.1) * torch.sin(x), V('src', 0.1) * u - 0.2 * x])


def _kdv_pair(f, x, t, D, V):                        # order 3: the whole-jet kernel
    u = f[..., 0:1]
    return torch.column_stack([D(u, t) + 6.0 * u * D(u, x) + D(D(D(u, x), x), x), D(u, x) - torch.cos(x)])


def _wave3d_pair(f, x, y, z, t, D, V):               # the 64-wide network of BASELINE.json cfg5: the tensor-core tile kernel
    u = f[:, [0]]
    return torch.cat([D(D(u, t), t) - (D(D(u, x), x) + D(D(u, y), y) + D(D(u, z), z)), 0.5 * (D(u, t) - u)], dim=-1)


PROBLEMS = {
    'burgers_penalty': dict(equation=_burgers_penalty, ndims=2, nparams=0, ic=P._ic_burgers, bc=0.5,
                            domain=[(-1, 2), (0, 3)], features=[8, 9, 1], activation='Tanh', layout='fafaf',
                            ranges=[(-1, 2), (0, 3)], log_scale=0.3, m=3),
    'heat_pair_skip': dict(equation=_heat_pair, ndims=2, nparams=0, ic=None, ic_factory=P._icf_heat1d, bc=0.0,
                           domain=(0, 1), features=[8, 8, 1], activation=['SiLU', 'Tanh'], layout='fa R fa+ f',
                           variables={'amp': 0.7, 'shift': 0.2, 'src': 0.1}, ranges=[(0, 1), (0, 1)], log_scale=-0.2, m=2),
    'kdv_two_residuals': dict(equation=_kdv_pair, ndims=2, nparams=0, ic=P._ic_kdv, bc=0.1, domain=[(-1, 2), (0, 1.5)],
                              features=[9, 7, 1], activation='Tanh', layout='fafaf', ranges=[(-1, 2), (0, 1.5)],
                              log_scale=0.2, m=2),
    'wave3d_two_residuals': dict(equation=_wave3d_pair, ndims=4, nparams=0, ic=P._ic_wave, bc=0, domain=(0, 1),
                                 features=[64, 64, 64, 64, 1], activation='Tanh', layout='fafafafaf',
                                 ranges=[(0, 1)] * 4, m=2),
}

GOLDEN_BATCH = {'burgers_penalty': 130, 'heat_pair_skip': 90, 'kdv_two_residuals': 72, 'wave3d_two_residuals': 64}
# a short Adam trajectory of the reference's own Solver.fit: name -> (niters, batch, lr)
GOLDEN_TRAJ = {'burgers_penalty': (20, 64, 0.01), 'heat_pair_skip': (20, 48, 0.02), 'kdv_two_residuals': (15, 48, 0.005)}


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


def folded_residual(residual, m, reduction='mean'):
    """ The per-point residual the kernels train on for an MSE fit: sqrt(mean_j r_j^2) (sum_j for reduction='sum'),
    from the reference's [N, m] residual. """
    r2 = np.square(np.asarray(residual, dtype=np.float64).reshape(-1, m))
    return np.sqrt(r2.sum(axis=1) if reduction == 'sum' else r2.mean(axis=1))
