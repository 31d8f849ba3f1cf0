""" Constraints that differentiate the solution at their own points (`D(u(t0), t0)`) on the fused kernels: in the
persistent multi-step kernels as terms in the equation's jet set, and as fused stepwise launches otherwise.

As in test_gpu_persistent_terms.py, a kernel's reduced gradient is read back from one step from a zero Adam state
(exp_avg = (1 - beta1) g).  The oracle is the fp64 autograd port: the equation's loss on the batch plus, for every
constraint, the criterion of its value — `prob.ansatz(prob.net(x), x)` at `x.requires_grad_()`, differentiated by
autograd — in one backward pass. """
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

from helpers import rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    from gpu_helpers import Replay
    from oracle import autograd_port as ap
    from pydens_b200 import Solver, D, V, fit_ensemble
    from pydens_b200 import _native as N

LR = 0.01
BETA1, BETA2 = 0.9, 0.999
FEATURES, LAYOUT, ACT = [12, 10, 1], 'fafaf', 'Tanh'
W2 = (2 * np.pi) ** 2


def _osc(u, t, D, V):                             # u'' + (2 pi)^2 u = 0
    return D(D(u, t), t) + W2 * u


def _osc_var(u, t, D, V):
    return D(D(u, t), t) + W2 * u * V('new_var', 1.0)


# name -> equation, initial condition ('const' = 1, or 'init' = V('init', 3.0)), the variables (sorted: the flat layout),
# constraints as (points, value(u at the points, the points, D, V)), criterion
SETUPS = {
    'velocity': dict(eq=_osc, ic='const', variables={}, cons=[([0.0], lambda u, t, D, V_: D(u, t))]),
    'two_terms': dict(eq=_osc_var, ic='init', variables={'init': 3.0, 'new_var': 1.0},
                      cons=[([0.2, 0.5, 0.8], lambda u, t, D, V_: D(u, t) * V_('new_var', 1.0) - 0.5),
                            ([0.5], lambda u, t, D, V_: u - 0.25)]),
    'second_order': dict(eq=_osc, ic='init', variables={'init': 3.0},
                         cons=[([0.0, 1.0], lambda u, t, D, V_: D(D(u, t), t) + D(u, t) - 1.0)]),
    'huber': dict(eq=_osc, ic='const', variables={}, cons=[([0.0], lambda u, t, D, V_: D(u, t))],
                  criterion=lambda: torch.nn.HuberLoss(delta=0.05)),
    'mse_sum': dict(eq=_osc_var, ic='init', variables={'init': 3.0, 'new_var': 1.0},
                    cons=[([0.3, 0.6], lambda u, t, D, V_: D(u, t) - 0.25)],
                    criterion=lambda: torch.nn.MSELoss(reduction='sum')),
}
BATCHES = [1, 16, 17, 127, 128, 129, 256, 1000, 1023, 1024]
MODES = {'c1': {'PINN_SMALL_CLUSTER': '1'}, 'c2': {'PINN_SMALL_CLUSTER': '2'}, 'c4': {'PINN_SMALL_CLUSTER': '4'},
         'c8': {'PINN_SMALL_CLUSTER': '8'}, 'tile': {'PINN_MULTI_KERNEL': 'tile'}}


def _loss_terms(name):
    return ['equation'] + ['constraint_%d' % i for i in range(len(SETUPS[name]['cons']))]


def _criterion(name):
    c = SETUPS[name].get('criterion')
    return c() if c else torch.nn.MSELoss()


def _pkg_V(n, init):
    return V(n, data=torch.Tensor([init]))


def _constraint(p, fn):
    def c(u, t):
        t0 = torch.tensor(p, requires_grad=True, device='cuda')     # where the autograd path can differentiate it too
        return fn(u(t0), t0, D, _pkg_V)
    return c


def _solver(name, backend='fused', seed=1234, torch_seed=0):
    cfg = SETUPS[name]
    torch.manual_seed(torch_seed)
    cons = [_constraint(p, fn) for p, fn in cfg['cons']]
    ic = 1.0 if cfg['ic'] == 'const' else (lambda *a: V('init', data=torch.Tensor([3.0])))
    solver = Solver(lambda u, t: cfg['eq'](u, t, D=D, V=_pkg_V), ndims=1, initial_condition=ic, layout=LAYOUT,
                    features=FEATURES, activation=ACT, constraints=cons, device='cuda', backend=backend, seed=seed)
    if backend == 'fused':
        solver._get_engine()
    return solver


def _oracle_loss_and_grads(name, params, pts):
    """ fp64: equation term on `pts` + every constraint term -> (loss, equation residual, flat grads) """
    cfg = SETUPS[name]
    holder = {}
    ic = 1.0 if cfg['ic'] == 'const' else (lambda *cols: holder['prob'].V('init'))
    prob = ap.Problem(lambda u, t, D, V: cfg['eq'](u, t, D=D, V=V), ndims=1, initial_condition=ic, features=FEATURES,
                      activation=ACT, layout=LAYOUT, dtype=torch.float64, variables=cfg['variables'])
    holder['prob'] = prob
    prob.load_flat(torch.as_tensor(np.asarray(params, dtype=np.float64)))
    crit = _criterion(name)
    prob.zero_grad()
    r, xs = prob.residual(np.asarray(pts, dtype=np.float64))
    loss = crit(r, torch.zeros_like(xs[0]))
    for p, fn in cfg['cons']:
        x = torch.tensor(p, dtype=torch.float64).reshape(-1, 1).requires_grad_()
        val = fn(prob.ansatz(prob.net(x), x), x, D, lambda n, init: prob.V(n)).reshape(-1, 1)
        loss = loss + crit(val, torch.zeros_like(val))
    loss.backward()
    return float(loss.detach()), r.detach().reshape(-1).numpy(), prob.flat_grads().numpy()


def _points(n, seed):
    return np.random.RandomState(seed).uniform(0, 1, size=(n, 1)).astype(np.float32)


def _tensors(name, eng):
    s = eng.spec
    out = []
    for l in range(s.n_layers):
        out.append(('W%d' % l, slice(s.w_off[l], s.w_off[l] + s.widths[l] * s.widths[l + 1])))
        out.append(('b%d' % l, slice(s.b_off[l], s.b_off[l] + s.widths[l + 1])))
    end = s.b_off[s.n_layers - 1] + s.widths[s.n_layers]
    return out + [('log_scale' if i == 0 else 'V%d' % i, slice(end + i, end + i + 1))
                  for i in range(1 + len(SETUPS[name]['variables']))]


def _check_against_oracle(name, eng, loss, grads, ref, tag):
    ref_loss, ref_res, ref_g = ref
    assert np.isfinite(grads).all() and np.isfinite(loss), tag
    assert abs(loss - ref_loss) <= 5e-5 * max(abs(ref_loss), 1e-6), '%s: loss %.9g, oracle %.9g' % (tag, loss, ref_loss)
    assert rel_l2(grads[:ref_g.size], ref_g) <= 2e-4, tag
    scale = 1e-3 * np.linalg.norm(ref_g)
    for tname, sl in _tensors(name, eng):
        err = np.linalg.norm(grads[sl] - ref_g[sl]) / max(np.linalg.norm(ref_g[sl]), scale, 1e-30)
        assert err <= 5e-4, '%s: %s rel err %.2e' % (tag, tname, err)


def _fit_one_step(solver, name, params, pts):
    solver.load_flat_params(params)
    with warnings.catch_warnings():
        warnings.filterwarnings('error', message='.*steps_per_launch')          # the persistent path must take it
        solver.fit(niters=1, batch_size=pts.shape[0], sampler=Replay([pts]), lr=LR, steps_per_launch=1,
                   loss_terms=_loss_terms(name), criterion=_criterion(name))
    eng = solver._engine
    assert not eng._graphs
    m, v = eng._adam_flat[0].cpu().numpy(), eng._adam_flat[1].cpu().numpy()
    return eng, float(solver.losses[-1]), m / (np.float32(1.0) - np.float32(BETA1)), v


_REFS = {}


def _ref(name, params, n):
    if (name, n) not in _REFS:
        pts = _points(n, seed=100 + n)
        _REFS[(name, n)] = (pts, _oracle_loss_and_grads(name, params, pts))
    return _REFS[(name, n)]


def test_constraints_lower_in_the_equation_jet_set():
    for name in SETUPS:
        s = _solver(name)
        for i in range(len(SETUPS[name]['cons'])):
            tr = s._lower_constraint(i)[0]
            assert tr.nf == 0 or (tr.dirs, tr.dir_vecs, tr.ns) == (s._traced.dirs, s._traced.dir_vecs, s._traced.ns)
        assert s._engine._persistent_terms(_loss_terms(name), 100) is not None


@pytest.mark.parametrize('name,mode', [(n, m) for n in SETUPS for m in MODES])
def test_persistent_gradient_matches_fp64_oracle(name, mode, monkeypatch):
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    solver = _solver(name)
    params = solver.flat_params().cpu().numpy()
    for n in BATCHES:
        pts, ref = _ref(name, params, n)
        tag = '%s %s batch %d' % (name, mode, n)
        eng, loss, g, v = _fit_one_step(solver, name, params, pts)
        _check_against_oracle(name, eng, loss, g, ref, tag)
        want = (np.float32(1.0) - np.float32(BETA2)) * g * g
        assert (np.abs(v - want) <= 1e-5 * want + 1e-38).all(), tag


@pytest.mark.parametrize('name', list(SETUPS))
def test_stepwise_fused_gradient_matches_fp64_oracle(name):
    """ The same gradient through the stepwise launches: the equation's step, then every constraint plan's. """
    solver = _solver(name)
    solver._fused_possible(_criterion(name), _loss_terms(name))      # trace the programs for the setup's criterion
    eng = solver._get_engine()
    params = solver.flat_params().cpu().numpy()
    sum_red = eng._sum_reduction()
    for n in BATCHES:
        pts, ref = _ref(name, params, n)
        solver.load_flat_params(params)
        dpts = torch.as_tensor(pts).cuda().contiguous()
        eng._step(dpts, None, n, 1.0 if sum_red else 1.0 / n, 0, use_counter=False)
        for i in range(len(SETUPS[name]['cons'])):
            eng._constraint_step(eng._constraint_plan(i))
        torch.cuda.synchronize()
        out = eng.out.cpu().numpy()
        _check_against_oracle(name, eng, float(out[eng.n_params]), out[:eng.n_params], ref, '%s stepwise %d' % (name, n))


def _curve(name, n, persistent, monkeypatch, niters=100, env=None):
    monkeypatch.setenv('PYDENS_B200_AUTO_PERSISTENT', '1' if persistent else '0')
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    solver = _solver(name)
    batches = [_points(n, seed=5000 + i) for i in range(niters)]
    kw = {'steps_per_launch': 50} if persistent else {}
    with warnings.catch_warnings():
        warnings.filterwarnings('error', message='.*steps_per_launch')
        solver.fit(niters=niters, batch_size=n, sampler=Replay(batches), lr=0.005, loss_terms=_loss_terms(name),
                   criterion=_criterion(name), **kw)
    return solver, np.asarray(solver.losses, dtype=np.float64), solver.flat_params().cpu().numpy()


@pytest.mark.parametrize('name', ['two_terms', 'mse_sum'])
def test_persistent_follows_the_stepwise_fused_path(name, monkeypatch):
    for n in (16, 100, 1000):
        sa, a, pa = _curve(name, n, True, monkeypatch)
        sb, b, pb = _curve(name, n, False, monkeypatch)
        assert not sa._engine._graphs and sb._engine._graphs
        err = np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-6))
        assert err <= 2e-3, '%s batch %d: loss curves %.2e apart' % (name, n, err)
        assert np.linalg.norm(pa - pb) / np.linalg.norm(pb) <= 1e-3, '%s batch %d' % (name, n)


@pytest.mark.parametrize('name', ['two_terms', 'second_order'])
def test_fused_constraints_match_the_autograd_constraints(name, monkeypatch):
    """ The fused constraint launches against PYDENS_B200_FUSED_CONSTRAINTS=0 (autograd adds them), identical batches. """
    _, a, pa = _curve(name, 2000, False, monkeypatch, niters=20)
    _, b, pb = _curve(name, 2000, False, monkeypatch, niters=20, env={'PYDENS_B200_FUSED_CONSTRAINTS': '0'})
    assert np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-6)) <= 1e-4
    assert np.linalg.norm(pa - pb) / np.linalg.norm(pb) <= 1e-4


def test_tiny_batch_oscillator_goes_persistent_by_itself():
    solver = _solver('velocity')
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        solver.fit(niters=200, batch_size=100, lr=0.005, loss_terms=_loss_terms('velocity'))
    assert not solver._engine._graphs and len(solver.losses) == 200 and np.isfinite(solver.losses).all()


def test_ensemble_members_equal_their_solo_fits():
    name = 'two_terms'
    solos = []
    for j in range(8):
        s = _solver(name, seed=900 + j, torch_seed=j)
        s.fit(niters=60, batch_size=100, lr=0.005, loss_terms=_loss_terms(name), steps_per_launch=20)
        solos.append((s.flat_params().cpu(), np.asarray(s.losses)))
    members = [_solver(name, seed=900 + j, torch_seed=j) for j in range(8)]
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        fit_ensemble(members, niters=60, batch_size=100, lr=0.005, loss_terms=_loss_terms(name), steps_per_launch=20)
    for (p, l), s in zip(solos, members):
        assert torch.equal(p, s.flat_params().cpu()) and np.array_equal(l, np.asarray(s.losses))


def _bits(n, k, sampler=True):
    name = 'two_terms'
    solver = _solver(name)
    kw = dict(sampler=Replay([_points(n, seed=700 + i) for i in range(50)])) if sampler else {}
    with warnings.catch_warnings():
        warnings.filterwarnings('error', message='.*steps_per_launch')
        solver.fit(niters=50, batch_size=n, lr=LR, steps_per_launch=k, loss_terms=_loss_terms(name), **kw)
    eng = solver._engine
    return (solver.flat_params().cpu(), eng._adam_flat[0].cpu(), eng._adam_flat[1].cpu(), np.asarray(solver.losses))


@pytest.mark.parametrize('n', [100, 1000])
def test_same_bits_across_steps_per_launch_and_runs(n):
    runs = [_bits(n, k) for k in (1, 7, 50)] + [_bits(n, 7)]
    for run in runs[1:]:
        for a, b in zip(runs[0][:3], run[:3]):
            assert torch.equal(a, b)
        assert np.array_equal(runs[0][3], run[3])
    a, b = _bits(n, 25, sampler=False), _bits(n, 25, sampler=False)       # in-kernel sampling, run to run
    assert all(torch.equal(x, y) for x, y in zip(a[:3], b[:3])) and np.array_equal(a[3], b[3])


def test_in_kernel_sampling_equals_explicit_points():
    """ The in-kernel batch is pinn_sample's: a fit on it equals a fit on those points given explicitly. """
    name, n, k = 'two_terms', 200, 10
    a = _solver(name)
    eng = a._engine
    batches = [eng.sample(n, step=s).cpu().numpy() for s in range(k)]
    with warnings.catch_warnings():
        warnings.filterwarnings('error', message='.*steps_per_launch')
        a.fit(niters=k, batch_size=n, lr=LR, steps_per_launch=k, loss_terms=_loss_terms(name))
        b = _solver(name)
        b.fit(niters=k, batch_size=n, lr=LR, steps_per_launch=k, loss_terms=_loss_terms(name), sampler=Replay(batches))
    assert torch.equal(a.flat_params(), b.flat_params()) and np.array_equal(np.asarray(a.losses), np.asarray(b.losses))


def _param_solver():
    """ u(t; p): the equation differentiates t only, the constraint along the parameter column p. """
    torch.manual_seed(0)

    def flux(u, t, p):
        p0 = torch.tensor([0.5, 0.5], requires_grad=True)
        return D(u(torch.tensor([0.3, 0.7]), p0), p0) - 0.1
    s = Solver(lambda u, t, p: D(u, t) - p * torch.cos(t), ndims=1, nparams=1, initial_condition=1.0, layout=LAYOUT,
               features=FEATURES, activation=ACT, constraints=[flux], device='cuda', backend='fused', seed=7)
    s._get_engine()
    return s


def test_a_constraint_along_another_column_runs_fused_stepwise():
    s = _param_solver()
    tr = s._lower_constraint(0)[0]
    assert tr.dirs == [1] and s._traced.dirs == [0]
    assert s._engine._constraint_plan(0) is not None
    s.fit(niters=30, batch_size=64, lr=0.005, loss_terms=['equation', 'constraint_0'])            # silently stepwise
    assert s._engine._graphs
    with pytest.warns(UserWarning, match='steps_per_launch ignored'):
        s.fit(niters=30, batch_size=64, lr=0.005, loss_terms=['equation', 'constraint_0'], steps_per_launch=10)
    assert np.isfinite(s.losses).all()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def test_a_term_plan_with_another_jet_set_is_refused_and_runs_nothing():
    s = _param_solver()
    eng = s._engine
    entry = eng._constraint_plan(0)
    dev = eng.device
    p = eng.flat.clone()
    m, v = torch.full_like(p, 0.25), torch.full_like(p, 0.5)
    mask = torch.ones_like(p)
    steps = torch.full((len(eng.entries),), 3.0, device=dev)
    counter = torch.full((1,), 11, dtype=torch.int64, device=dev)
    ring = torch.full((64,), -1.0, device=dev)
    before = [t.clone() for t in (p, m, v, steps, counter, ring)]
    arr = (N.PinnTerm * 1)()
    arr[0].plan, arr[0].n_points, arr[0].point_weight = entry['plan'].value, entry['n'], 1.0 / entry['n']
    arr[0].points = entry['host_points'].data_ptr()
    rc = eng.lib.pinn_multi_step_terms(
        eng.plan, _ptr(p), _ptr(m), _ptr(v), _ptr(mask), _ptr(steps), C.c_int(steps.numel()), None,
        N.make_columns(None, 2), C.c_uint64(eng.seed), _ptr(counter), C.c_int64(64), C.c_int(3), C.c_float(LR),
        C.c_float(BETA1), C.c_float(BETA2), C.c_float(1e-8), C.c_float(0.0), C.c_float(0.0), _ptr(ring),
        C.c_int64(ring.numel()), C.c_float(1.0 / 64), C.c_int(1), arr, eng._stream())
    torch.cuda.synchronize()
    assert rc == N.E_INVALID and b'derivative directions' in eng.lib.pinn_last_error()
    for a, b in zip(before, (p, m, v, steps, counter, ring)):
        assert torch.equal(a, b)
