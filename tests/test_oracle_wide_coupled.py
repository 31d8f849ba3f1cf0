""" The oracle (oracle/autograd_port.py) pinned against outputs of the UNMODIFIED reference on coupled systems whose
hidden layers are 65-128 units wide (tests/problems_wide_coupled.py, goldens by tools/make_wide_coupled_golden.py):
fp32 reproduces the reference's residual [N, m], loss, gradients, predict [N, k] and fit trajectory; fp64 brackets
them.  CPU only. """
import warnings

import numpy as np
import pytest
import torch

import problems_wide_coupled as PWC
from helpers import load_golden, rel_l2
from oracle import autograd_port as ap


def wide_coupled_oracle(name, dtype=torch.float64, params=None):
    cfg = PWC.PROBLEMS[name]
    holder = {}
    ic = PWC.make_ic(name, lambda n, init: holder['prob'].V(n, init))
    prob = ap.Problem(lambda u, *xs, D, V: cfg['equation'](u, *xs, D=D, V=V), ndims=cfg['ndims'],
                      nparams=cfg['nparams'], initial_condition=ic, boundary_condition=cfg['bc'],
                      domain=cfg['domain'], features=cfg['features'], activation=cfg['activation'], dtype=dtype,
                      variables=cfg.get('variables'), layout=cfg['layout'])
    holder['prob'] = prob
    if params is not None:
        prob.load_flat(torch.as_tensor(params))
    return prob


def loss_and_grads(prob, pts, criterion):
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)          # torch's [N, m] vs [N, 1] broadcast, as in the reference
        return prob.loss_and_grads(pts, criterion=criterion)


def test_goldens_are_complete_and_outside_the_thread_kernel_sizes():
    for name, cfg in PWC.PROBLEMS.items():
        g = load_golden(name)
        assert g['points'].shape == (PWC.GOLDEN_BATCH[name], len(cfg['ranges']))
        assert g['residual'].shape == (g['points'].shape[0], cfg['m'])
        assert g['u'].shape == (g['points'].shape[0], cfg['k']) and 2 <= cfg['k'] <= 4
        assert ('traj_losses' in g) == (name in PWC.GOLDEN_TRAJ)
        assert max(cfg['features'][:-1]) > 64 and max(cfg['features'][:-1]) <= 128
        assert cfg['features'][-1] == cfg['k']


@pytest.mark.parametrize('name', list(PWC.PROBLEMS))
def test_port_matches_reference_fp32(name):
    g = load_golden(name)
    cfg = PWC.PROBLEMS[name]
    prob = wide_coupled_oracle(name, torch.float32, g['params'])
    loss, residual, grads = loss_and_grads(prob, g['points'], PWC.torch_criterion(name))
    assert abs(loss - float(g['loss'])) <= 2e-6 * abs(float(g['loss']))
    assert rel_l2(residual, g['residual']) <= 2e-6
    assert rel_l2(grads.numpy(), g['grads']) <= 2e-5
    u = prob.predict(g['points']).reshape(-1, cfg['k'])
    assert u.shape == g['u'].shape and rel_l2(u, g['u']) <= 2e-6


@pytest.mark.parametrize('name', list(PWC.PROBLEMS))
def test_fp64_port_brackets_reference(name):
    g = load_golden(name)
    prob = wide_coupled_oracle(name, torch.float64, g['params'].astype(np.float64))
    loss, _, grads = loss_and_grads(prob, g['points'].astype(np.float64), PWC.torch_criterion(name))
    assert abs(loss - float(g['loss'])) <= 1e-4 * abs(float(g['loss']))
    assert rel_l2(g['grads'], grads.numpy()) <= 2e-3


@pytest.mark.parametrize('name', list(PWC.GOLDEN_TRAJ))
def test_port_trajectory_matches_reference_fit(name):
    g = load_golden(name)
    niters, batch, lr = int(g['traj_meta'][0]), int(g['traj_meta'][1]), float(g['traj_meta'][2])
    prob = wide_coupled_oracle(name, torch.float32, g['params'])
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        losses = ap.fit(prob, niters, batch, lr=lr, criterion=PWC.torch_criterion(name),
                        point_stream=lambda i: torch.from_numpy(PWC.make_points(name, batch, seed=1000 + i)))
    ref = g['traj_losses']
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 1e-3
    assert abs(losses[-1] - ref[-1]) <= 1e-5 * max(1.0, abs(ref[-1]))
    assert rel_l2(prob.flat_params().numpy(), g['traj_params']) <= 1e-4
