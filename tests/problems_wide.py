""" Problems on networks with hidden layers 65-128 units wide whose weights do not fit the thread kernel's shared memory:
the 128-wide class of the tensor-core tile kernel (pydens_b200/csrc/pinn_wide_kernel.cuh) takes them.  Shared by
tools/make_wide_golden.py, which records tests/golden/<name>.npz from the unmodified reference, and the tests of this
feature.  Kept apart from tests/problems.py so that the parametrisation of the tests over that registry stays as it is.

Same layout as tests/problems.py (`eq(f, *xs, D=..., V=...)`, one dict per problem).
"""
import problems as P

PROBLEMS = {
    # the README Poisson equation on a 3 x 128 tanh network: five jet channels
    'poisson_wide128': dict(equation=P._poisson2d, ndims=2, nparams=0, ic=None, bc=1, domain=(0, 1),
                            features=[128, 128, 128, 1], activation='Tanh', layout='fa fa fa f',
                            ranges=[(0, 1), (0, 1)]),
    # the tutorial heat problem with an initial condition on a 4 x 100 sigmoid network
    'heat_wide100': dict(equation=P._heat2d, ndims=3, nparams=0, ic=P._ic_heat, bc=0, domain=(0, 1),
                         features=[100, 100, 100, 100, 1], activation='Sigmoid', layout='fafafafaf',
                         ranges=[(0, 1), (0, 1), (0, .5)], log_scale=0.1),
    # variables in the equation and in the initial condition; mixed widths and an identity layer
    'heat1d_icvar_wide': dict(equation=P._heat1d_icvar, ndims=2, nparams=0, ic=None, ic_factory=P._icf_heat1d, bc=0.0,
                              domain=(0, 1), features=[128, 100, 128, 1], activation=['Tanh', 'Sigmoid'],
                              layout='fa f fa f', variables={'amp': 0.7, 'shift': 0.2, 'src': 0.1},
                              ranges=[(0, 1), (0, 1)], log_scale=-0.2),
}

GOLDEN_BATCH = {'poisson_wide128': 100, 'heat_wide100': 96, 'heat1d_icvar_wide': 90}
# a short Adam trajectory of the reference's own Solver.fit: name -> (niters, batch, lr)
GOLDEN_TRAJ = {'heat_wide100': (12, 64, 0.001), 'heat1d_icvar_wide': (12, 48, 0.005)}


def make_points(name, batch, seed):
    import numpy as np
    rng = np.random.RandomState(seed)
    cols = [rng.uniform(lo, hi, size=(batch, 1)) for lo, hi in PROBLEMS[name]['ranges']]
    return np.concatenate(cols, axis=1).astype(np.float32)


def make_ic(name, V):
    cfg = PROBLEMS[name]
    return cfg['ic_factory'](V) if 'ic_factory' in cfg else cfg['ic']


def bind(name, D, V):
    eq = PROBLEMS[name]['equation']
    return lambda u, *xs: eq(u, *xs, D=D, V=V)
