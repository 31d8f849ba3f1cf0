""" Which optimizers the fused kernels take over, without a GPU.

The step kernel's tail (pinn_step_adam) and the persistent kernels apply torch.optim.Adam's update themselves: L2
weight decay added to the gradient, one bias-correction step t for every parameter.  `engine.plain_adam` decides which
optimizers that is, `engine.adam_hyper` hands their hyper-parameters to the kernels (and keys the captured graphs), and
`engine.adam_steps_equal` checks that one t serves every parameter.  Anything else must stay on torch's own optimizer:
`Adam(decoupled_weight_decay=True)` with weight decay is AdamW, which the kernels do not implement. """
import types
import warnings

import numpy as np
import pytest
import torch

from pydens_b200 import D, V, Solver, ensemble, fit_ensemble
from pydens_b200.engine import adam_hyper, adam_steps_equal, plain_adam


def _params():
    torch.manual_seed(0)
    return [torch.nn.Parameter(torch.randn(3, 2)), torch.nn.Parameter(torch.randn(3))]


# (optimizer factory, plain Adam the kernels implement)
CASES = {
    'adam': (lambda ps: torch.optim.Adam(ps, lr=1e-3), True),
    'adam_fused_capturable': (lambda ps: torch.optim.Adam(ps, lr=1e-3, fused=True, capturable=True), True),
    'adam_l2_decay': (lambda ps: torch.optim.Adam(ps, lr=1e-3, weight_decay=0.1), True),
    'adam_decoupled_no_decay': (lambda ps: torch.optim.Adam(ps, lr=1e-3, decoupled_weight_decay=True), True),
    'adam_decoupled_decay': (lambda ps: torch.optim.Adam(ps, lr=1e-3, weight_decay=0.1, decoupled_weight_decay=True),
                             False),
    'adamw': (lambda ps: torch.optim.AdamW(ps, lr=1e-3), False),
    'amsgrad': (lambda ps: torch.optim.Adam(ps, lr=1e-3, amsgrad=True), False),
    'maximize': (lambda ps: torch.optim.Adam(ps, lr=1e-3, maximize=True), False),
    'tensor_lr': (lambda ps: torch.optim.Adam(ps, lr=torch.tensor(1e-3)), False),
    'two_groups': (lambda ps: torch.optim.Adam([{'params': ps[:1]}, {'params': ps[1:], 'lr': 1e-2}], lr=1e-3), False),
    'sgd': (lambda ps: torch.optim.SGD(ps, lr=1e-3), False),
}


@pytest.mark.parametrize('name', list(CASES))
def test_plain_adam_table(name):
    make, plain = CASES[name]
    opt = make(_params())
    assert plain_adam(opt) is plain, name
    if plain:
        wd = 0.1 if name == 'adam_l2_decay' else 0.0
        assert adam_hyper(opt) == (pytest.approx(1e-3), (0.9, 0.999), 1e-8, pytest.approx(wd))
        assert all(isinstance(x, float) for x in (adam_hyper(opt)[0], adam_hyper(opt)[2], adam_hyper(opt)[3]))


def test_decoupled_decay_is_not_the_update_the_kernels_apply():
    """ what plain_adam guards: with weight decay, Adam(decoupled_weight_decay=True) takes AdamW's steps, not L2
    Adam's; adam_hyper cannot tell the two apart, so the predicate has to """
    runs = {}
    for name, make in (('decoupled', lambda ps: torch.optim.Adam(ps, lr=1e-2, weight_decay=0.1,
                                                                    decoupled_weight_decay=True)),
                       ('adamw', lambda ps: torch.optim.AdamW(ps, lr=1e-2, weight_decay=0.1)),
                       ('l2', lambda ps: torch.optim.Adam(ps, lr=1e-2, weight_decay=0.1))):
        ps = _params()
        opt = make(ps)
        for s in range(50):
            opt.zero_grad()
            sum(((p - 0.3 * s / 50) ** 2).sum() for p in ps).backward()
            opt.step()
        runs[name] = torch.cat([p.detach().reshape(-1) for p in ps])
    assert torch.equal(runs['decoupled'], runs['adamw'])
    assert (runs['decoupled'] - runs['l2']).abs().max() > 1e-3
    opts = [torch.optim.Adam(_params(), lr=1e-2, weight_decay=0.1, decoupled_weight_decay=d) for d in (False, True)]
    assert adam_hyper(opts[0]) == adam_hyper(opts[1])


def test_step_counts_must_be_equal():
    ps = _params()
    opt = torch.optim.Adam(ps, lr=1e-3)
    assert adam_steps_equal(opt)                          # no state yet: every parameter at 0
    for _ in range(3):
        opt.zero_grad()
        sum((p ** 2).sum() for p in ps).backward()
        opt.step()
    assert adam_steps_equal(opt)
    state = opt.state_dict()
    state['state'][1]['step'] = torch.tensor(1.0)
    opt.load_state_dict(state)
    assert not adam_steps_equal(opt)
    part = torch.optim.Adam(ps, lr=1e-3)                  # state for the first tensor only: the second is at 0
    state['state'] = {0: state['state'][0]}
    part.load_state_dict(state)
    assert not adam_steps_equal(part)


def _solver(seed):
    torch.manual_seed(seed)
    return Solver(lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t) + V('c', data=torch.Tensor([1.0])),
                  ndims=1, initial_condition=1.0, layout='fafaf', features=[12, 10, 1], activation='Tanh',
                  device='cpu', seed=seed)


def test_ensemble_with_decoupled_decay_warns_and_names_it(monkeypatch):
    """ fit_ensemble's optimizer check, reached on a CPU device by engines that stand in for the fused ones (every
    check before it passes): decoupled weight decay sends the solvers to their own fits, with a warning that names
    it, and each fit is then torch's Adam(decoupled_weight_decay=True) """
    from pydens_b200 import _native
    spec = _native.PinnSpec()
    ens = [_solver(j) for j in range(3)]
    for s in ens:
        def optimizer_for(optimizer, lr, kwargs, s=s):
            s._make_optimizer(optimizer, lr, **kwargs)
            return s.optimizer, False
        eng = types.SimpleNamespace(spec=spec, _persistent_terms=lambda loss_terms, batch_size: [],
                                    _optimizer_for=optimizer_for)
        monkeypatch.setattr(s, '_get_engine', lambda eng=eng: eng)
    monkeypatch.setattr(Solver, '_fused_possible', lambda self, criterion, loss_terms: (True, ''))
    why = ensemble._fit_together(ens, 3, 16, [None] * 3, ('equation',), 'Adam', torch.nn.MSELoss(), 0.01, 5,
                                 dict(weight_decay=0.1, decoupled_weight_decay=True))
    assert why is not None and 'decoupled weight decay' in why, why
    monkeypatch.undo()
    torch.manual_seed(7)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        fit_ensemble(ens, niters=3, batch_size=16, optimizer='Adam', weight_decay=0.1, decoupled_weight_decay=True)
    assert len([w for w in caught if 'fit_ensemble' in str(w.message)]) == 1
    for s in ens:
        assert len(s.losses) == 3
        assert type(s.optimizer) is torch.optim.Adam and s.optimizer.param_groups[0]['decoupled_weight_decay']
