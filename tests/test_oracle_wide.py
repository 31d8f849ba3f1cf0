""" The oracle (oracle/autograd_port.py) pinned against outputs of the UNMODIFIED reference on the networks with hidden
layers 65-128 units wide (tests/problems_wide.py, goldens by tools/make_wide_golden.py). CPU only. """
import numpy as np
import pytest
import torch

import problems_wide as PW
from helpers import load_golden, rel_l2
from oracle import autograd_port as ap


def wide_oracle_problem(name, dtype=torch.float32, params=None):
    cfg = PW.PROBLEMS[name]
    holder = {}
    ic = PW.make_ic(name, lambda n, init: holder['prob'].V(n, init))
    prob = ap.Problem(lambda u, *xs, D, V: cfg['equation'](u, *xs, D=D, V=V),
                      ndims=cfg['ndims'], nparams=cfg['nparams'], initial_condition=ic,
                      boundary_condition=cfg['bc'], domain=cfg['domain'], features=cfg['features'],
                      activation=cfg['activation'], dtype=dtype, variables=cfg.get('variables'), layout=cfg['layout'])
    holder['prob'] = prob
    if params is not None:
        prob.load_flat(torch.as_tensor(params))
    return prob


def test_goldens_are_small_and_complete():
    for name in PW.PROBLEMS:
        g = load_golden(name)
        assert g['points'].shape == (PW.GOLDEN_BATCH[name], len(PW.PROBLEMS[name]['ranges']))
        assert ('traj_losses' in g) == (name in PW.GOLDEN_TRAJ)
        assert max(PW.PROBLEMS[name]['features'][:-1]) > 64


@pytest.mark.parametrize('name', list(PW.PROBLEMS))
def test_port_matches_reference_fp32(name):
    g = load_golden(name)
    prob = wide_oracle_problem(name, torch.float32, g['params'])
    loss, residual, grads = prob.loss_and_grads(g['points'])
    assert abs(loss - float(g['loss'])) <= 2e-6 * abs(float(g['loss']))
    assert rel_l2(residual, g['residual']) <= 2e-6
    assert rel_l2(grads.numpy(), g['grads']) <= 2e-5
    assert rel_l2(prob.predict(g['points']), g['u']) <= 2e-6


@pytest.mark.parametrize('name', list(PW.PROBLEMS))
def test_fp64_port_brackets_reference(name):
    g = load_golden(name)
    prob = wide_oracle_problem(name, torch.float64, g['params'].astype(np.float64))
    loss, residual, grads = prob.loss_and_grads(g['points'].astype(np.float64))
    assert abs(loss - float(g['loss'])) <= 1e-4 * abs(float(g['loss']))
    assert rel_l2(g['grads'], grads.numpy()) <= 2e-3


@pytest.mark.parametrize('name', list(PW.GOLDEN_TRAJ))
def test_port_trajectory_matches_reference_fit(name):
    g = load_golden(name)
    niters, batch, lr = g['traj_meta']
    niters, batch = int(niters), int(batch)
    prob = wide_oracle_problem(name, torch.float32, g['params'])
    losses = ap.fit(prob, niters, batch, lr=float(lr),
                    point_stream=lambda i: torch.from_numpy(PW.make_points(name, batch, seed=1000 + i)))
    ref = g['traj_losses']
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 1e-3
    assert abs(losses[-1] - ref[-1]) <= 1e-5 * max(1.0, abs(ref[-1]))
