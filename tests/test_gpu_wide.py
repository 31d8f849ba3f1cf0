""" The tensor-core tile kernel for wide networks (pydens_b200/csrc/pinn_wide_kernel.cuh) against the reference's
goldens, the oracle port, and the thread-per-point kernel.  `PINN_FORCE_KERNEL=wide` puts the tile kernel on every
problem it covers (plain dense chains, tanh / sigmoid / identity activations, hidden widths <= 64), so that its
3xTF32 arithmetic is held to the same fp32 tolerances as the CUDA-core kernel: loss rel <= 1e-5, residual rel-L2
<= 1e-5, gradients rel-L2 <= 1e-4 whole and per tensor (reference path: pydens/model_torch.py:430-460). """
import os

import numpy as np
import pytest
import torch

import problems as P
from helpers import load_golden, oracle_problem, rel_l2

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from gpu_helpers import make_solver

# golden problems the tile kernel covers (the others carry residual layouts or sin / softplus / SiLU / GELU)
WIDE_OK = ['poisson2d', 'ode_param', 'heat2d', 'heat_param', 'wave3d', 'ode_var', 'ode_tanh', 'burgers',
           'heat1d_icvar', 'mixed2d', 'mixed_ic', 'nonlinear']


class forced:
    """ Context manager: plans created inside pick the named kernel. """

    def __init__(self, kind):
        self.kind = kind

    def __enter__(self):
        self.prev = os.environ.get('PINN_FORCE_KERNEL')
        os.environ['PINN_FORCE_KERNEL'] = self.kind

    def __exit__(self, *exc):
        if self.prev is None:
            os.environ.pop('PINN_FORCE_KERNEL', None)
        else:
            os.environ['PINN_FORCE_KERNEL'] = self.prev


def wide_solver(name, params=None):
    with forced('wide'):
        solver = make_solver(name, params)
        eng = solver._get_engine()
    assert eng.info.tensor_core == 1
    return solver


@pytest.mark.parametrize('name', WIDE_OK)
def test_tile_kernel_matches_reference_golden(name):
    g = load_golden(name)
    solver = wide_solver(name, g['params'])
    loss, grads, residual = solver.loss_and_grads(g['points'])
    grads = grads.cpu().numpy()
    assert np.isfinite(grads).all()
    assert abs(loss - float(g['loss'])) <= 1e-5 * abs(float(g['loss']))
    assert rel_l2(residual.cpu().numpy(), g['residual']) <= 1e-5
    assert rel_l2(grads, g['grads']) <= 1e-4
    spec = solver._get_engine().spec
    for l in range(spec.n_layers):
        w = slice(spec.w_off[l], spec.w_off[l] + spec.widths[l] * spec.widths[l + 1])
        b = slice(spec.b_off[l], spec.b_off[l] + spec.widths[l + 1])
        assert rel_l2(grads[w], g['grads'][w]) <= 1e-4, 'W%d' % l
        assert rel_l2(grads[b], g['grads'][b]) <= 1e-4, 'b%d' % l
    # log_scale and the equation variables ride in the same buffer
    rest = slice(spec.b_off[spec.n_layers - 1] + 1, g['grads'].size)
    if np.linalg.norm(g['grads'][rest]) > 0:
        assert rel_l2(grads[rest], g['grads'][rest]) <= 1e-4


def test_wide_networks_take_the_tile_kernel_by_default():
    assert make_solver('wave3d')._get_engine().info.tensor_core == 1       # 64-wide: BASELINE configs[4]
    assert make_solver('heat2d')._get_engine().info.tensor_core == 0       # 30 / 40 wide: the thread kernel is faster
    assert make_solver('poisson2d')._get_engine().info.tensor_core == 0    # 10 / 12 / 15 wide: thread kernel


@pytest.mark.parametrize('name', ['wave3d', 'heat2d', 'burgers'])
def test_tile_kernel_vs_fp64(name):
    """ 3xTF32 is fp32-grade: the distance to the fp64 oracle stays at the level of the reference's own fp32 run. """
    g = load_golden(name)
    solver = wide_solver(name, g['params'])
    _, grads, _ = solver.loss_and_grads(g['points'])
    prob = oracle_problem(name, torch.float64, g['params'].astype(np.float64))
    _, _, g64 = prob.loss_and_grads(g['points'].astype(np.float64))
    ours, ref = rel_l2(grads.cpu().numpy(), g64.numpy()), rel_l2(g['grads'], g64.numpy())
    assert ours <= max(8 * ref, 1e-5), (ours, ref)


@pytest.mark.parametrize('n', [1, 2, 127, 128, 129, 1000, 4097, 20000])
def test_tile_kernel_ragged_batches_against_oracle(n):
    """ wave3d (64-wide, 9 jet channels) against the fp32 oracle port on fresh points, ragged sizes incl. 20 000. """
    g = load_golden('wave3d')
    solver = wide_solver('wave3d', g['params'])
    prob = oracle_problem('wave3d', torch.float32, g['params'])
    pts = P.make_points('wave3d', n, seed=77)
    loss, grads, residual = solver.loss_and_grads(pts)
    l, r, gr = prob.loss_and_grads(pts)
    assert abs(loss - l) <= 1e-5 * abs(l)
    assert rel_l2(residual.cpu().numpy(), r) <= 1e-5
    assert rel_l2(grads.cpu().numpy(), gr.numpy()) <= 1e-4


@pytest.mark.parametrize('name,n', [('wave3d', 30000), ('heat2d', 50000), ('burgers', 10000)])
def test_tile_kernel_equals_thread_kernel(name, n):
    g = load_golden(name)
    pts = P.make_points(name, n, seed=3)
    a = wide_solver(name, g['params']).loss_and_grads(pts)
    with forced('thread'):
        solver = make_solver(name, g['params'])
        assert solver._get_engine().info.tensor_core == 0
        b = solver.loss_and_grads(pts)
    assert abs(a[0] - b[0]) <= 1e-5 * abs(b[0])
    assert rel_l2(a[2].cpu().numpy(), b[2].cpu().numpy()) <= 1e-5
    assert rel_l2(a[1].cpu().numpy(), b[1].cpu().numpy()) <= 1e-4


def test_tile_kernel_deterministic_run_to_run():
    g = load_golden('wave3d')
    solver = wide_solver('wave3d', g['params'])
    pts = P.make_points('wave3d', 20000, seed=5)
    a = solver.loss_and_grads(pts)
    b = solver.loss_and_grads(pts)
    assert a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_tile_kernel_sampling_equals_explicit_points():
    g = load_golden('wave3d')
    solver = wide_solver('wave3d', g['params'])
    eng = solver._get_engine()
    n = 50000
    eng._step(None, None, n, 1.0 / n, 0, use_counter=False, step_value=9)
    torch.cuda.synchronize()
    sampled = eng.out.clone()
    pts = eng.sample(n, None, step=9)
    eng._step(pts, None, n, 1.0 / n, 0, use_counter=False, step_value=9)
    torch.cuda.synchronize()
    assert torch.equal(sampled, eng.out)


@pytest.mark.parametrize('name,n', [('wave3d', 500000), ('heat2d', 300000)])
def test_tile_kernel_full_size_additivity(name, n):
    """ BASELINE configs[4] at full per-GPU size (and configs[3]'s network): two half batches add up to the whole
    batch (the property the data-parallel path relies on), everything finite. """
    g = load_golden(name)
    solver = wide_solver(name, g['params'])
    eng = solver._get_engine()
    assert eng.info.tensor_core == 1
    pts = torch.from_numpy(P.make_points(name, n, seed=11)).cuda()
    h = n // 2 + 13
    eng._step(pts, None, n, 1.0 / n, 0, use_counter=False)
    whole = eng.out.clone()
    eng._step(pts[:h].contiguous(), None, h, 1.0 / n, 0, use_counter=False)
    a = eng.out.clone()
    eng._step(pts[h:].contiguous(), None, n - h, 1.0 / n, 0, use_counter=False)
    b = eng.out.clone()
    torch.cuda.synchronize()
    assert torch.isfinite(whole).all()
    np_ = eng.n_params
    assert abs(float(whole[np_] - (a + b)[np_])) <= 1e-5 * abs(float(whole[np_]))
    assert rel_l2((a + b)[:np_].cpu().numpy(), whole[:np_].cpu().numpy()) <= 1e-4


@pytest.mark.parametrize('name,batch,lr', [('wave3d', 2000, 0.001), ('heat2d', 64, 0.001), ('burgers', 200, 0.01)])
def test_tile_kernel_fit_trajectory(name, batch, lr):
    """ 20 Adam steps on replayed batches (host-batch pipeline, captured step graphs): the tile kernel and the thread
    kernel walk the same loss curve — also for batches smaller than one 128-point tile. """
    import warnings
    from gpu_helpers import Replay
    g = load_golden(name)
    batches = [P.make_points(name, batch, seed=100 + i) for i in range(20)]
    curves = []
    for kind in ('wide', 'thread'):
        with forced(kind), warnings.catch_warnings():
            warnings.simplefilter('error')                   # a failed graph capture must not pass silently
            solver = make_solver(name, g['params'])
            solver.fit(niters=20, batch_size=batch, sampler=Replay(batches), lr=lr)
        curves.append(np.array(solver.losses, dtype=np.float64))
    assert np.all(np.abs(curves[0] - curves[1]) <= 1e-4 * np.maximum(1.0, np.abs(curves[1])))
