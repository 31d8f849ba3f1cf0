""" Equations with a residual of several columns on the GPU (CPU twin: test_systems.py): every golden of
tests/problems_systems.py through the bare C ABI and through Solver — thread kernel, the GEN wiring of residual layouts,
the whole-jet kernel (order 3) and the tensor-core tile kernel (64-wide) —, Solver.fit against the reference's own fit,
determinism, in-kernel sampling, graph replay, the persistent small-batch kernel, and a criterion with reduction='sum'. """
import os
import warnings

import numpy as np
import pytest
import torch

import problems_systems as PS
from helpers import load_golden, rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

if torch.cuda.is_available():
    from gpu_helpers import Replay, abi_step
    from pydens_b200 import Solver, D, V
    from test_systems import system_spec, system_oracle, oracle_loss_and_grads


def pkg_V(name, init):
    return V(name, data=torch.Tensor([init]))


def make_system_solver(name, params=None, backend='fused', **kw):
    cfg = PS.PROBLEMS[name]
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)           # the [N, m] vs [N, 1] broadcast of the throw-away run
        solver = Solver(PS.bind(name, D, pkg_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                        initial_condition=PS.make_ic(name, pkg_V), boundary_condition=cfg['bc'], domain=cfg['domain'],
                        layout=cfg['layout'], features=cfg['features'], activation=cfg['activation'],
                        device='cuda', backend=backend, seed=1234, **kw)
    if params is not None:
        solver.load_flat_params(params)
    elif 'log_scale' in cfg:
        with torch.no_grad():
            solver.model.log_scale.fill_(cfg['log_scale'])
    return solver


def _slack(name, g):
    """ order 3: the reference's fp32 nested autograd is itself this far from fp64 (test_systems.py) """
    if name != 'kdv_two_residuals':
        return 0.0, 0.0
    m = PS.PROBLEMS[name]['m']
    _, r64, g64 = oracle_loss_and_grads(system_oracle(name, params=g['params'].astype(np.float64)), g['points'].astype(np.float64))
    return rel_l2(PS.folded_residual(g['residual'], m), PS.folded_residual(r64, m)), rel_l2(g['grads'], g64.numpy())


def _check_against_golden(name, g, loss, residual, grads, u, spec):
    m = PS.PROBLEMS[name]['m']
    slack_r, slack_g = _slack(name, g)
    assert np.isfinite(grads).all()
    assert abs(loss - float(g['loss'])) <= (1e-5 + 2.0 * slack_r) * abs(float(g['loss']))
    assert rel_l2(residual, PS.folded_residual(g['residual'], m)) <= 1e-5 + 1.5 * slack_r
    assert rel_l2(grads, g['grads']) <= 1e-4 + 1.5 * slack_g
    for l in range(spec.n_layers):
        w = slice(spec.w_off[l], spec.w_off[l] + spec.widths[l] * spec.widths[l + 1])
        b = slice(spec.b_off[l], spec.b_off[l] + spec.widths[l + 1])
        assert rel_l2(grads[w], g['grads'][w]) <= 1e-4 + 1.5 * slack_g, 'W%d' % l
        assert rel_l2(grads[b], g['grads'][b]) <= 1e-4 + 1.5 * slack_g, 'b%d' % l
    rest = slice(spec.b_off[spec.n_layers - 1] + spec.widths[spec.n_layers], g['grads'].size)   # log_scale, variables
    if np.linalg.norm(g['grads'][rest]) > 0:
        assert rel_l2(grads[rest], g['grads'][rest]) <= 1e-4 + 1.5 * slack_g
    assert rel_l2(u, g['u']) <= 1e-5


@pytest.mark.parametrize('name', list(PS.PROBLEMS))
def test_c_abi_step_matches_reference_golden(name):
    g = load_golden(name)
    spec = system_spec(name)
    loss, residual, grads, u = abi_step(spec, g['params'], g['points'])
    _check_against_golden(name, g, loss, residual, grads, u, spec)


@pytest.mark.parametrize('name', list(PS.PROBLEMS))
def test_solver_matches_reference_golden(name):
    g = load_golden(name)
    solver = make_system_solver(name, g['params'])
    eng = solver._get_engine()
    assert eng is not None
    if name == 'wave3d_two_residuals':
        assert eng.info.tensor_core == 1                       # 64-wide: the tile kernel
    loss, grads, residual = solver.loss_and_grads(g['points'])
    u = solver.predict(*[g['points'][:, i] for i in range(g['points'].shape[1])])
    assert u.shape == (g['points'].shape[0], 1)
    _check_against_golden(name, g, loss, residual.cpu().numpy(), grads.cpu().numpy(), u.reshape(-1), eng.spec)


@pytest.mark.parametrize('name', list(PS.GOLDEN_TRAJ))
def test_fit_trajectory_matches_reference_fit(name):
    """ Same init, same point stream, same Adam: the fused fit follows the reference's own `Solver.fit`. """
    g = load_golden(name)
    niters, batch, lr = int(g['traj_meta'][0]), int(g['traj_meta'][1]), float(g['traj_meta'][2])
    solver = make_system_solver(name, g['params'])
    batches = [PS.make_points(name, batch, seed=1000 + i) for i in range(niters)]
    solver.fit(niters=niters, batch_size=batch, sampler=Replay(batches), lr=lr)
    assert solver._engine is not None
    losses, ref = np.asarray(solver.losses, dtype=np.float64), g['traj_losses'].astype(np.float64)
    assert losses.shape == ref.shape
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 2e-3
    assert abs(losses[-1] - ref[-1]) <= 1e-5 * max(1.0, abs(ref[-1]))
    final = solver.flat_params().cpu().numpy()
    assert np.linalg.norm(final - g['traj_params']) / np.linalg.norm(g['traj_params']) <= 1e-3


@pytest.mark.parametrize('name', ['burgers_penalty', 'wave3d_two_residuals'])
def test_deterministic_run_to_run_and_sampling_equals_explicit_points(name):
    g = load_golden(name)
    solver = make_system_solver(name, g['params'])
    pts = PS.make_points(name, 20000, seed=5)
    a, b = solver.loss_and_grads(pts), solver.loss_and_grads(pts)
    assert a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])
    eng = solver._get_engine()
    n = 50000
    eng._step(None, None, n, 1.0 / n, 0, use_counter=False, step_value=9)
    torch.cuda.synchronize()
    sampled = eng.out.clone()
    pts = eng.sample(n, None, step=9)
    eng._step(pts, None, n, 1.0 / n, 0, use_counter=False, step_value=9)
    torch.cuda.synchronize()
    assert torch.equal(sampled, eng.out)


def test_graph_replay_equals_plain_launches():
    g = load_golden('heat_pair_skip')
    curves = []
    for no_graph in ('0', '1'):
        os.environ['PYDENS_B200_NO_GRAPH'] = no_graph
        try:
            solver = make_system_solver('heat_pair_skip', g['params'])
            solver.fit(niters=40, batch_size=5000, lr=0.005)
        finally:
            os.environ.pop('PYDENS_B200_NO_GRAPH', None)
        curves.append(np.asarray(solver.losses, dtype=np.float64))
    assert len(curves[0]) == 40 and np.isfinite(curves[0]).all()
    np.testing.assert_allclose(curves[0], curves[1], rtol=1e-6)
    assert curves[0][-1] < curves[0][0]


def test_fresh_points_against_the_fp32_oracle_at_50k():
    """ The 64-wide problem (tile kernel) on 50 000 fresh points against the oracle port of the reference in fp32. """
    name = 'wave3d_two_residuals'
    g = load_golden(name)
    solver = make_system_solver(name, g['params'])
    pts = PS.make_points(name, 50000, seed=77)
    loss, grads, residual = solver.loss_and_grads(pts)
    l, r, gr = oracle_loss_and_grads(system_oracle(name, torch.float32, g['params']), pts)
    assert abs(loss - l) <= 1e-5 * abs(l)
    assert rel_l2(residual.cpu().numpy(), PS.folded_residual(r, 2)) <= 1e-5
    assert rel_l2(grads.cpu().numpy(), gr.numpy()) <= 1e-4


@pytest.mark.parametrize('kernel,k', [(None, None), ('small', 10), ('tile', 7)])
def test_small_batch_fit_follows_the_oracle_loop(kernel, k, monkeypatch):
    """ batch 96: the persistent kernels — taken by themselves, and with an explicit steps_per_launch on the
    (point, unit)-parallel one ('small') and the thread-per-point one ('tile') — against the oracle port of the
    reference loop in fp64 on the same batches. """
    from oracle import autograd_port as ap
    if kernel is not None:
        monkeypatch.setenv('PINN_MULTI_KERNEL', kernel)
    name, niters, batch, lr = 'burgers_penalty', 30, 96, 0.01
    g = load_golden(name)
    batches = [PS.make_points(name, batch, seed=2000 + i) for i in range(niters)]
    prob = system_oracle(name, params=g['params'].astype(np.float64))
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        ref = ap.fit(prob, niters, batch, lr=lr, point_stream=lambda i: torch.from_numpy(batches[i].astype(np.float64)))
    solver = make_system_solver(name, g['params'])
    kw = {} if k is None else {'steps_per_launch': k}
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)            # "steps_per_launch ignored" would be a failure
        solver.fit(niters=niters, batch_size=batch, sampler=Replay(batches), lr=lr, **kw)
    assert not solver._engine._graphs                          # the persistent path, not per-step graphs
    losses = np.asarray(solver.losses, dtype=np.float64)
    assert losses.shape == ref.shape
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 2e-3
    want = prob.flat_params().numpy()
    final = solver.flat_params().cpu().numpy()
    assert np.linalg.norm(final[:want.size] - want) / np.linalg.norm(want) <= 2e-3


def test_fit_with_sum_reduction_follows_the_oracle_loop():
    from oracle import autograd_port as ap
    name, niters, batch, lr = 'heat_pair_skip', 20, 64, 0.002
    g = load_golden(name)
    batches = [PS.make_points(name, batch, seed=3000 + i) for i in range(niters)]
    prob = system_oracle(name, params=g['params'].astype(np.float64))
    crit = lambda: torch.nn.HuberLoss(delta=0.1, reduction='sum')
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        ref = ap.fit(prob, niters, batch, lr=lr, criterion=crit(),
                     point_stream=lambda i: torch.from_numpy(batches[i].astype(np.float64)))
    solver = make_system_solver(name, g['params'])
    solver.fit(niters=niters, batch_size=batch, sampler=Replay(batches), lr=lr, criterion=crit())
    assert solver._engine is not None and solver._crit_key[-1] == 'sum'
    losses = np.asarray(solver.losses, dtype=np.float64)
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 2e-3
    want = prob.flat_params().numpy()
    final = solver.flat_params().cpu().numpy()
    assert np.linalg.norm(final[:want.size] - want) / np.linalg.norm(want) <= 2e-3
