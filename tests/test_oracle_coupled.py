""" The fp64 yardstick of the coupled-system tests, oracle/autograd_port.py, against the goldens the unmodified reference
recorded for networks with 2..4 outputs (tools/make_coupled_golden.py): its ansatz broadcasts over the k components as the
reference's does, and in fp32 it reproduces the reference's residual [N, m], loss, gradients and predict [N, k]. """
import warnings

import numpy as np
import pytest
import torch

import problems_coupled as PC
from helpers import load_golden, rel_l2
from test_coupled import coupled_oracle, oracle_loss_and_grads


@pytest.mark.parametrize('name', list(PC.PROBLEMS))
def test_port_reproduces_reference_goldens(name):
    g = load_golden(name)
    cfg = PC.PROBLEMS[name]
    prob = coupled_oracle(name, dtype=torch.float32, params=g['params'])
    loss, residual, grads = oracle_loss_and_grads(prob, g['points'], criterion=PC.torch_criterion(name))
    assert abs(loss - float(g['loss'])) <= 1e-6 * abs(float(g['loss']))
    assert rel_l2(residual, g['residual']) <= 1e-6
    assert rel_l2(grads.numpy(), g['grads']) <= 1e-5
    u = prob.predict(g['points']).reshape(-1, cfg['k'])
    assert u.shape == g['u'].shape and rel_l2(u, g['u']) <= 1e-6


@pytest.mark.parametrize('name', list(PC.GOLDEN_TRAJ))
def test_port_fit_follows_the_reference_fit(name):
    from oracle import autograd_port as ap
    g = load_golden(name)
    niters, batch, lr = int(g['traj_meta'][0]), int(g['traj_meta'][1]), float(g['traj_meta'][2])
    prob = coupled_oracle(name, dtype=torch.float32, params=g['params'])
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)          # the [N, m] vs [N, 1] broadcast, as in the reference
        losses = ap.fit(prob, niters, batch, lr=lr, criterion=PC.torch_criterion(name),
                        point_stream=lambda i: torch.from_numpy(PC.make_points(name, batch, seed=1000 + i)))
    assert np.max(np.abs(losses - g['traj_losses']) / np.abs(g['traj_losses'])) <= 1e-4
    assert rel_l2(prob.flat_params().numpy(), g['traj_params']) <= 1e-4
