""" Criteria other than MSELoss on the GPU (reference model_torch.py:365, :448 `criterion(residual, zeros)`): L1Loss,
HuberLoss and SmoothL1Loss train on the same kernels through the residual transform of tracer.apply_criterion —
through the bare C ABI against torch's own criteria on the fp64 oracle (thread kernel, tensor-core tile kernel, whole-jet
kernel), and through Solver.fit against the oracle port of the reference loop on identical batches.  (Sorted last: this
joined after the round's GPU time was spent; its CPU twin is test_emul.py::test_other_criteria_ride_on_the_mse_kernels.) """
import numpy as np
import pytest
import torch

import problems as P
import emul_harness as E
from helpers import load_golden, oracle_problem, rel_l2, criterion_case

# a hang in a kernel that has not met a GPU yet must end as a failure of that test, not stall the whole tier
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

if torch.cuda.is_available():
    from gpu_helpers import make_solver, Replay, abi_step
    from oracle import autograd_port as ap


@pytest.mark.parametrize('kind', ['l1', 'huber', 'smooth_l1'])
@pytest.mark.parametrize('name', ['poisson2d', 'burgers', 'heat1d_icvar', 'mixed_acts_skip', 'wave3d', 'kdv'])
def test_step_with_other_criteria_matches_torch_criteria_on_the_fp64_oracle(name, kind):
    g = load_golden(name)
    key, crit = criterion_case(kind, g['residual'])
    spec = E.spec_for(name, criterion=key)
    loss, _, grads, u = abi_step(spec, g['params'], g['points'])
    prob = oracle_problem(name, torch.float64, g['params'].astype(np.float64))
    l64, _, g64 = prob.loss_and_grads(g['points'].astype(np.float64), criterion=crit)
    assert abs(loss - l64) <= 2e-5 * abs(l64)
    assert rel_l2(grads, g64.numpy()) <= 1e-4
    assert rel_l2(u, g['u']) <= 1e-5


@pytest.mark.parametrize('make', [lambda: torch.nn.HuberLoss(delta=0.05), lambda: torch.nn.L1Loss(),
                                  lambda: torch.nn.SmoothL1Loss(beta=0.1), lambda: torch.nn.MSELoss(reduction='sum'),
                                  lambda: torch.nn.HuberLoss(delta=0.05, reduction='sum')],
                         ids=['huber', 'l1', 'smooth_l1', 'mse_sum', 'huber_sum'])
def test_fit_with_other_criteria_follows_the_reference_loop(make):
    """ Solver.fit(criterion=...) on the fused path against the oracle port of the reference loop (fp64, same criterion,
    identical initial weights and batches); then back to MSELoss on the same Solver: the engine is rebuilt for the
    criterion of the fit and the parameters carry over. """
    name, niters, batch, lr = 'burgers', 20, 64, 0.01
    g = load_golden(name)
    solver = make_solver(name, g['params'])
    batches = [P.make_points(name, batch, seed=1000 + i) for i in range(niters)]
    prob = oracle_problem(name, torch.float64, g['params'].astype(np.float64))
    ref = ap.fit(prob, niters, batch, lr=lr, criterion=make(),
                 point_stream=lambda i: torch.from_numpy(batches[i].astype(np.float64)))
    solver.fit(niters=niters, batch_size=batch, sampler=Replay(batches), lr=lr, criterion=make())
    assert solver._engine is not None and solver._crit_key != ('mse',)
    losses = np.asarray(solver.losses, dtype=np.float64)
    assert losses.shape == ref.shape
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 2e-3
    final, want = solver.flat_params().cpu().numpy(), prob.flat_params().numpy()
    assert np.linalg.norm(final[:want.size] - want) / np.linalg.norm(want) <= 2e-3
    first = solver._engine
    solver.fit(niters=8, batch_size=batch, lr=lr)                       # MSELoss again, in-kernel sampling
    assert solver._crit_key == ('mse',) and solver._engine is not None and solver._engine is not first
    assert len(solver.losses) == niters + 8 and np.isfinite(np.asarray(solver.losses, dtype=np.float64)).all()
    after = solver.flat_params().cpu().numpy()
    assert np.linalg.norm(after - final) / np.linalg.norm(final) < 0.5   # continued from the Huber fit, not from scratch


def test_unsupported_criterion_takes_the_autograd_path_loudly():
    solver = make_solver('poisson2d', backend='auto')
    with pytest.warns(UserWarning):
        solver.fit(niters=2, batch_size=32, criterion=lambda a, b: ((a - b) ** 2).mean())
    assert len(solver.losses) == 2


@pytest.mark.parametrize('fused_constraints', ['1', '0'])
def test_constraint_only_fit_stays_on_the_engine_and_matches_autograd(fused_constraints, monkeypatch):
    """ loss_terms without 'equation' (reference :382-389, :448-457): the step is the constraint terms alone — as fused
    launches of the constraint plans, or as autograd terms inside the engine's loop — against the autograd backend. """
    from pydens_b200 import Solver, D, V
    monkeypatch.setenv('PYDENS_B200_FUSED_CONSTRAINTS', fused_constraints)

    def odevar(u, t):
        return D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t)

    def initial(*args):
        return V('init', data=torch.Tensor([3.0]))

    def make(backend):
        torch.manual_seed(0)
        return Solver(odevar, ndims=1, initial_condition=initial, layout='fafaf', features=[12, 10, 1], activation='Tanh',
                      constraints=lambda u, t: u(torch.tensor([0.5])) - 0.25, device='cuda', backend=backend)
    fused, ref = make('fused'), make('torch')
    ref.model.load_state_dict(fused.model.state_dict())
    for s in (fused, ref):
        s.fit(niters=30, batch_size=64, lr=0.02, loss_terms='constraint_0')
    assert fused._engine is not None and (fused._engine._constraint_plans[0] is not None) == (fused_constraints == '1')
    a, b = np.asarray(fused.losses, dtype=np.float64), np.asarray(ref.losses, dtype=np.float64)
    assert a.shape == b.shape == (30,) and b[-1] < b[0]
    assert np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-6)) <= 2e-3
    assert abs(float(fused.model.init.detach()) - float(ref.model.init.detach())) <= 1e-4
    assert float(fused.model.init.detach()) != 3.0


def test_piecewise_equation_with_where_trains_fused_like_autograd():
    """ torch.where / comparisons in the equation (a diffusivity that jumps at x = 0.5, a source switched on in a band)
    run as indicator arithmetic in the kernel's residual program: the fused fit against the autograd backend executing
    the user's torch.where, identical weights and batches. """
    from pydens_b200 import Solver, D

    def pde(u, x, y):
        a = torch.where(x < 0.5, 1.0, 10.0)
        return a * D(D(u, x), x) + D(D(u, y), y) - torch.where((x > 0.2) & (y <= 0.7), torch.sin(3.0 * x), torch.zeros_like(x))

    def make(backend):
        torch.manual_seed(0)
        return Solver(pde, ndims=2, boundary_condition=0.0, layout='fafaf', features=[10, 8, 1], activation='Tanh',
                      device='cuda', backend=backend)
    fused, ref = make('fused'), make('torch')
    ref.model.load_state_dict(fused.model.state_dict())
    rng = np.random.RandomState(11)
    batches = [rng.uniform(0.01, 0.99, size=(128, 2)).astype(np.float32) for _ in range(20)]
    fused.fit(niters=20, batch_size=128, sampler=Replay(batches), lr=0.01)
    ref.fit(niters=20, batch_size=128, sampler=Replay(batches), lr=0.01)
    assert fused._engine is not None
    a, b = np.asarray(fused.losses, dtype=np.float64), np.asarray(ref.losses, dtype=np.float64)
    assert a.shape == b.shape == (20,)
    assert np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-6)) <= 2e-3
    grid = np.linspace(0.05, 0.95, 9)
    assert np.abs(fused.predict(grid, 0.5) - ref.predict(grid, 0.5)).max() <= 1e-4
