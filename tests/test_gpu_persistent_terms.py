""" Constraint terms in the persistent multi-step kernels (pinn_multi_step_terms): fits with `loss_terms=['equation',
'constraint_k', ...]` whose constraints lower to fused plans, and fits with reduction='sum', run k whole optimizer steps
per launch of small_step_kernel (the constraint points are more columns of the cluster's slices) or multi_step_kernel
(one more tile, walked after the batch tiles).

As in test_gpu_persistent.py, each kernel's own reduced gradient is read back from one step from a zero Adam state:
exp_avg = fmaf(1 - beta1, g, 0), so g = exp_avg / float32(1 - beta1) to within one rounding.  The oracle is the fp64
autograd port: the equation's loss on the batch plus, for every constraint, the criterion of the constraint's value at
its points (the model evaluated there through the ansatz), in one backward pass. """
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
    from pydens_b200 import Solver, D, V
    from pydens_b200 import _native as N
    from pydens_b200.engine import FusedEngine

LR = 0.01
BETA1, BETA2 = 0.9, 0.999
FEATURES, LAYOUT, ACT = [12, 10, 1], 'fafaf', 'Tanh'


def _eq_var(u, t, D, V):                          # tutorial stage 5: a trainable variable in the equation
    return D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t) + V('new_var', 1.0)


def _eq_plain(u, t, D, V):                        # README.md:112-126
    return D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t)


# name -> equation, initial condition ('const' = 1, or 'init' = V('init', 3.0)), the variables (sorted: the flat layout),
# constraints as (points, value(u at the points, V)), criterion
SETUPS = {
    'tutorial5': dict(eq=_eq_var, ic='const', variables={'new_var': 1.0}, cons=[([0.5], lambda u, V_: u)]),
    'readme': dict(eq=_eq_plain, ic='init', variables={'init': 3.0}, cons=[([0.5], lambda u, V_: u - 0.25)]),
    'three_points': dict(eq=_eq_var, ic='init', variables={'init': 3.0, 'new_var': 1.0},
                         cons=[([0.2, 0.5, 0.8], lambda u, V_: u * V_('new_var', 1.0) - 0.5)]),
    'two_terms': dict(eq=_eq_var, ic='init', variables={'init': 3.0, 'new_var': 1.0},
                      cons=[([0.5], lambda u, V_: u - 0.25), ([0.1, 0.9], lambda u, V_: u - V_('init', 3.0))]),
    'huber': dict(eq=_eq_plain, ic='init', variables={'init': 3.0}, cons=[([0.5], lambda u, V_: u - 0.25)],
                  criterion=lambda: torch.nn.HuberLoss(delta=0.05)),
    'mse_sum': dict(eq=_eq_var, ic='init', variables={'init': 3.0, 'new_var': 1.0},
                    cons=[([0.3, 0.6], lambda u, V_: u - 0.25)], criterion=lambda: torch.nn.MSELoss(reduction='sum')),
}
BATCHES = [1, 16, 17, 127, 128, 129, 256, 1000, 1023, 1024, 2047]
MODES = {'c1': {'PINN_SMALL_CLUSTER': '1'}, 'c2': {'PINN_SMALL_CLUSTER': '2'}, 'c4': {'PINN_SMALL_CLUSTER': '4'},
         'c8': {'PINN_SMALL_CLUSTER': '8'}, 'tile': {'PINN_MULTI_KERNEL': 'tile'}}


def _loss_terms(name):
    return ['equation'] + ['constraint_%d' % i for i in range(len(SETUPS[name]['cons']))]


def _criterion(name):
    c = SETUPS[name].get('criterion')
    return c() if c else torch.nn.MSELoss()


def _pkg_V(n, init):
    return V(n, data=torch.Tensor([init]))


def _solver(name, backend='fused'):
    cfg = SETUPS[name]
    torch.manual_seed(0)
    cons = [lambda u, t, p=p, fn=fn: fn(u(torch.tensor(p)), _pkg_V) for p, fn in cfg['cons']]
    ic = 1.0 if cfg['ic'] == 'const' else (lambda *a: V('init', data=torch.Tensor([3.0])))
    solver = Solver(lambda u, t: cfg['eq'](u, t, D=D, V=_pkg_V), ndims=1, initial_condition=ic, layout=LAYOUT,
                    features=FEATURES, activation=ACT, constraints=cons, device='cuda', backend=backend, seed=1234)
    if backend == 'fused':
        solver._get_engine()
    return solver


def _oracle(name, params):
    cfg = SETUPS[name]
    holder = {}
    ic = 1.0 if cfg['ic'] == 'const' else (lambda *cols: holder['prob'].V('init'))
    prob = ap.Problem(lambda u, t, D, V: cfg['eq'](u, t, D=D, V=V), ndims=1, initial_condition=ic, features=FEATURES,
                      activation=ACT, layout=LAYOUT, dtype=torch.float64, variables=cfg['variables'])
    holder['prob'] = prob
    prob.load_flat(torch.as_tensor(np.asarray(params, dtype=np.float64)))
    return prob


def _oracle_loss_and_grads(name, params, pts):
    """ fp64: equation term on `pts` + every constraint term -> (loss, equation residual, flat grads) """
    cfg = SETUPS[name]
    prob = _oracle(name, params)
    crit = _criterion(name)
    prob.zero_grad()
    r, xs = prob.residual(np.asarray(pts, dtype=np.float64))
    loss = crit(r, torch.zeros_like(xs[0]))
    for p, fn in cfg['cons']:
        x = torch.tensor(p, dtype=torch.float64).reshape(-1, 1)
        val = fn(prob.ansatz(prob.net(x), x), lambda n, init: prob.V(n)).reshape(-1, 1)
        loss = loss + crit(val, torch.zeros_like(val))
    # the magnitudes a scalar's gradient (log_scale, V) sums over: 2 w |r| per point (|dr/dV|, |du/dlog_scale| <= 1 here)
    w = 1.0 if getattr(crit, 'reduction', 'mean') == 'sum' else None
    mags = float(torch.sum(torch.abs(r.detach()))) * 2.0 * (w or 1.0 / r.shape[0])
    loss.backward()
    return float(loss.detach()), r.detach().reshape(-1).numpy(), prob.flat_grads().numpy(), mags


def _points(n, seed):
    return np.random.RandomState(seed).uniform(0, 1, size=(n, 1)).astype(np.float32)


def _n_cons(name):
    return sum(len(p) for p, _ in SETUPS[name]['cons'])


def _tensors(name, eng):
    s = eng.spec
    out = []
    for l in range(s.n_layers):
        out.append(('W%d' % l, slice(s.w_off[l], s.w_off[l] + s.widths[l] * s.widths[l + 1])))
        out.append(('b%d' % l, slice(s.b_off[l], s.b_off[l] + s.widths[l + 1])))
    end = s.b_off[s.n_layers - 1] + s.widths[s.n_layers]
    out += [('log_scale' if i == 0 else 'V%d' % i, slice(end + i, end + i + 1))
            for i in range(1 + len(SETUPS[name]['variables']))]
    return out


def _check_against_oracle(name, eng, loss, grads, ref, tag):
    ref_loss, ref_res, ref_g, mags = ref
    cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(ref_res)))), 1e-30))
    assert np.isfinite(grads).all() and np.isfinite(loss), tag
    assert abs(loss - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), '%s: loss %.9g, oracle %.9g' % (tag, loss, ref_loss)
    assert rel_l2(grads[:ref_g.size], ref_g) <= 1e-4 * cond, tag
    scale = 1e-3 * np.linalg.norm(ref_g)
    for tname, sl in _tensors(name, eng):
        scalar = tname == 'log_scale' or tname.startswith('V')
        # a scalar's gradient is one sum over the points, whose fp32 rounding follows the magnitudes it adds, not the
        # (possibly cancelled) result: tutorial5 at 16 points lands 3.8e-4 off a d/dV that is a small mean of residuals ~5
        floor = max(scale, 1e-2 * mags) if scalar else scale
        err = np.linalg.norm(grads[sl] - ref_g[sl]) / max(np.linalg.norm(ref_g[sl]), floor, 1e-30)
        tol = (3e-4 if scalar else 1e-4) * cond
        assert err <= tol, '%s: %s rel err %.2e' % (tag, tname, err)


def _fit_one_step(solver, name, params, pts):
    """ one persistent step on `pts` (+ the constraint points) from `params` and a zero Adam state """
    solver.load_flat_params(params)
    with warnings.catch_warnings():
        warnings.filterwarnings('error', message='.*steps_per_launch')          # the persistent path must take it
        solver.fit(niters=1, batch_size=pts.shape[0], sampler=Replay([pts]), lr=LR, steps_per_launch=1,
                   loss_terms=_loss_terms(name), criterion=_criterion(name))
    eng = solver._engine
    assert not eng._graphs
    m, v = eng._adam_flat[0].cpu().numpy(), eng._adam_flat[1].cpu().numpy()
    return eng, float(solver.losses[-1]), m / (np.float32(1.0) - np.float32(BETA1)), v


def _check_second_moment(g, v, tag):
    want = (np.float32(1.0) - np.float32(BETA2)) * g * g
    err = np.abs(v - want)
    assert (err <= 1e-5 * want + 1e-38).all(), tag


_REFS = {}


def _ref(name, params, n):
    key = (name, n)
    if key not in _REFS:
        pts = _points(n, seed=100 + n)
        _REFS[key] = (pts, _oracle_loss_and_grads(name, params, pts))
    return _REFS[key]


@pytest.mark.parametrize('name,mode', [(n, m) for n in SETUPS for m in MODES])
def test_terms_gradient_matches_fp64_oracle(name, mode, monkeypatch):
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    solver = _solver(name)
    params = solver.flat_params().cpu().numpy()
    for n in BATCHES:
        pts, ref = _ref(name, params, n)
        tag = '%s %s batch %d + %d constraint points' % (name, mode, n, _n_cons(name))
        eng, loss, g, v = _fit_one_step(solver, name, params, pts)
        _check_against_oracle(name, eng, loss, g, ref, tag)
        _check_second_moment(g, v, tag)


def _curve(name, n, persistent, monkeypatch, niters=100):
    monkeypatch.setenv('PYDENS_B200_AUTO_PERSISTENT', '1' if persistent else '0')
    solver = _solver(name)
    batches = [_points(n, seed=5000 + i) for i in range(niters)]
    kw = {'steps_per_launch': 50} if persistent else {}
    with warnings.catch_warnings():
        warnings.filterwarnings('error', message='.*steps_per_launch')
        solver.fit(niters=niters, batch_size=n, sampler=Replay(batches), lr=0.005, loss_terms=_loss_terms(name),
                   criterion=_criterion(name), **kw)
    assert (not solver._engine._graphs) == persistent
    return np.asarray(solver.losses, dtype=np.float64), solver.flat_params().cpu().numpy()


@pytest.mark.parametrize('name', ['two_terms', 'mse_sum'])
def test_terms_follow_the_stepwise_fused_path(name, monkeypatch):
    """ 100 steps, 50 per launch, against one launch per step (equation step, constraint steps, torch's Adam) """
    for n in BATCHES:
        a, pa = _curve(name, n, True, monkeypatch)
        b, pb = _curve(name, n, False, monkeypatch)
        assert a.shape == b.shape == (100,)
        err = np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-6))
        assert err <= 2e-3, '%s batch %d: loss curves %.2e apart' % (name, n, err)
        assert np.linalg.norm(pa - pb) / np.linalg.norm(pb) <= 1e-3, '%s batch %d' % (name, n)


@pytest.mark.parametrize('n', [100, 1000])
def test_steps_per_launch_give_the_same_bits(n):
    name = 'two_terms'
    batches = [_points(n, seed=700 + i) for i in range(50)]
    runs = []
    for k in (1, 7, 50):
        solver = _solver(name)
        with warnings.catch_warnings():
            warnings.filterwarnings('error', message='.*steps_per_launch')
            solver.fit(niters=50, batch_size=n, sampler=Replay(list(batches)), lr=LR, steps_per_launch=k,
                       loss_terms=_loss_terms(name))
        eng = solver._engine
        runs.append((solver.flat_params().cpu(), eng._adam_flat[0].cpu(), eng._adam_flat[1].cpu(),
                     np.asarray(solver.losses)))
    for run in runs[1:]:
        for a, b in zip(runs[0][:3], run[:3]):
            assert torch.equal(a, b)
        assert np.array_equal(runs[0][3], run[3])
    assert np.isfinite(runs[0][3]).all()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


class _State:
    def __init__(self, eng, params, step0, ring_len):
        dev = eng.device
        z = torch.zeros(eng.n_params, dtype=torch.float32, device=dev)
        self.p = torch.as_tensor(params, dtype=torch.float32).to(dev).clone()
        self.m, self.v = z.clone(), z.clone()
        self.mask = torch.ones(eng.n_params, dtype=torch.float32, device=dev)
        self.steps = torch.zeros(len(eng.entries), dtype=torch.float32, device=dev)
        self.counter = torch.full((1,), step0, dtype=torch.int64, device=dev)
        self.ring = torch.zeros(ring_len, dtype=torch.float32, device=dev)


def _terms(eng, entries):
    arr = (N.PinnTerm * max(1, len(entries)))()
    for i, e in enumerate(entries):
        arr[i].plan, arr[i].n_points = e['plan'].value, e['n']
        arr[i].point_weight, arr[i].points = 1.0 / e['n'], e['host_points'].data_ptr()
    return arr


def _multi_step_terms(eng, st, points, n, k, entries, cols=None, plan=None):
    return eng.lib.pinn_multi_step_terms(
        plan if plan is not None else eng.plan, _ptr(st.p), _ptr(st.m), _ptr(st.v), _ptr(st.mask), _ptr(st.steps),
        C.c_int(st.steps.numel()), _ptr(points), N.make_columns(cols, eng.solver.model.total), C.c_uint64(eng.seed),
        _ptr(st.counter), C.c_int64(n), C.c_int(k), C.c_float(LR), C.c_float(BETA1), C.c_float(BETA2), C.c_float(1e-8),
        C.c_float(0.0), C.c_float(0.0), _ptr(st.ring), C.c_int64(st.ring.numel()), C.c_float(1.0 / n),
        C.c_int(len(entries)), _terms(eng, entries), eng._stream())


@pytest.mark.parametrize('n', [200, 700])
def test_in_kernel_sampling_equals_explicit_points(n):
    """ constraint points consume no sampler counters: the in-kernel batch is pinn_sample's """
    solver = _solver('two_terms')
    eng = solver._engine
    entries = [eng._constraint_plan(i) for i in range(2)]
    cols = [(N.COL_NORMAL, 0.5, 0.2)]
    s0, k = (3 << 32) | 5, 3
    params = solver.flat_params().cpu().numpy()
    sampled, explicit = _State(eng, params, s0, 4), _State(eng, params, s0, 4)
    N.check(_multi_step_terms(eng, sampled, None, n, k, entries, cols=cols))
    pts = torch.stack([eng.sample(n, cols, step=s0 + s) for s in range(k)]).contiguous()
    N.check(_multi_step_terms(eng, explicit, pts, n, k, entries))
    torch.cuda.synchronize()
    assert not torch.equal(sampled.p, torch.as_tensor(params).cuda())
    for a, b in zip((sampled.p, sampled.m, sampled.v, sampled.ring, sampled.counter),
                    (explicit.p, explicit.m, explicit.v, explicit.ring, explicit.counter)):
        assert torch.equal(a, b)


def test_tutorial_stage5_runs_persistent():
    """ the tutorial's trainable-variable stage: variable frozen, then trained with the constraint term """
    solver = _solver('tutorial5')
    solver.model.freeze_trainable(variables=('new_var',))
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)
        solver.fit(niters=200, batch_size=500, lr=0.1)
        assert float(solver.model.new_var.detach()) == 1.0
        solver.model.unfreeze_trainable(variables=['new_var'])
        solver.fit(niters=100, batch_size=100, lr=0.1, loss_terms=['equation', 'constraint_0'])
    assert not solver._engine._graphs
    assert float(solver.model.new_var.detach()) != 1.0
    assert len(solver.losses) == 300 and np.isfinite(solver.losses).all()


def test_readme_flow_runs_persistent_and_follows_autograd():
    """ README.md:112-126: V in the initial condition and a constraint; then only the variable trains """
    batches = [_points(150, seed=900 + i) for i in range(200)]
    fused, ref = _solver('readme'), _solver('readme', backend='torch')
    assert torch.equal(fused.model.conv_block.linears[0].weight.detach().cpu(),
                       ref.model.conv_block.linears[0].weight.detach().cpu())
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)
        fused.fit(niters=200, batch_size=150, lr=0.05, sampler=Replay(list(batches)),
                  loss_terms=['equation', 'constraint_0'])
    ref.fit(niters=200, batch_size=150, lr=0.05, sampler=Replay(list(batches)), loss_terms=['equation', 'constraint_0'])
    assert not fused._engine._graphs
    a, b = np.asarray(fused.losses, dtype=np.float64), np.asarray(ref.losses, dtype=np.float64)
    assert np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-6)) <= 2e-3
    assert float(fused.model.init.detach()) != 3.0
    # second stage: the network is frozen, `init` keeps training through the initial condition and the constraint
    fused.model.freeze_layers(['fc1', 'fc2', 'fc3'], ['log_scale'])
    w0 = fused.model.conv_block.linears[0].weight.detach().clone()
    init0 = float(fused.model.init.detach())
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)
        fused.fit(niters=100, batch_size=150, lr=0.05, loss_terms=['equation', 'constraint_0'])
    assert not fused._engine._graphs
    assert torch.equal(w0, fused.model.conv_block.linears[0].weight.detach())
    assert float(fused.model.init.detach()) != init0
    assert np.isfinite(fused.losses).all()


def _no_persistent(monkeypatch):
    def boom(*a, **k):
        raise AssertionError('the persistent path was taken')
    monkeypatch.setattr(FusedEngine, '_fit_persistent', boom)


@pytest.mark.parametrize('case', ['two_evaluations', 'five_terms', 'thirty_three_points', 'constraint_only'])
def test_what_stays_stepwise(case, monkeypatch):
    cons = [lambda u, t: u(torch.tensor([0.5])) - 0.25]
    terms = ['equation', 'constraint_0']
    if case == 'two_evaluations':
        cons = [lambda u, t: u(torch.tensor([0.2])) - u(torch.tensor([0.7]))]
    elif case == 'five_terms':
        cons = [lambda u, t, c=c: u(torch.tensor([0.1 * (c + 1)])) for c in range(5)]
        terms = ['equation'] + ['constraint_%d' % c for c in range(5)]
    elif case == 'thirty_three_points':
        cons = [lambda u, t: u(torch.linspace(0.0, 1.0, 33)) - 0.25]
    else:
        terms = ['constraint_0']
    torch.manual_seed(0)
    solver = Solver(lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t), ndims=1, initial_condition=1.0, layout=LAYOUT, features=FEATURES, activation=ACT, constraints=cons,
                    device='cuda', backend='fused', seed=1234)
    _no_persistent(monkeypatch)
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)                  # automatic: silent
        solver.fit(niters=20, batch_size=100, lr=0.01, loss_terms=terms)
    with pytest.warns(UserWarning, match='steps_per_launch ignored'):
        solver.fit(niters=4, batch_size=100, lr=0.01, loss_terms=terms, steps_per_launch=2)
    assert len(solver.losses) == 24 and np.isfinite(solver.losses).all()


def test_term_plan_with_another_network_is_refused():
    solver = _solver('readme')
    eng = solver._engine
    other_spec_args = list(eng._spec_args)
    other_spec_args[0] = [1, 12, 9, 1]                               # another layer table
    lowered = solver._lower_constraint(0)
    spec = N.build_spec(*other_spec_args, lowered[0], **dict(eng._spec_kwargs, var_offsets=None, w_off=None, b_off=None,
                                                              log_scale_off=None, n_params=None))
    plan = C.c_void_p()
    N.check(eng.lib.pinn_plan_create(C.byref(spec), eng.device.index, C.byref(plan)))
    try:
        entry = dict(plan=plan, n=1, host_points=torch.tensor([[0.5]], dtype=torch.float32))
        st = _State(eng, solver.flat_params().cpu().numpy(), 0, 1)
        pts = torch.from_numpy(_points(100, seed=1)).cuda().reshape(1, 100, 1).contiguous()
        assert _multi_step_terms(eng, st, pts, 100, 1, [entry]) == N.E_INVALID
        assert b'layer table' in eng.lib.pinn_last_error()
        # and a plan that matches is taken
        assert _multi_step_terms(eng, st, pts, 100, 1, [eng._constraint_plan(0)]) == 0
        torch.cuda.synchronize()
        assert int(st.counter) == 1
    finally:
        eng.lib.pinn_plan_destroy(plan)
