""" The device loss ring at engine level.  Every fit writes its step losses into a ring on the device and reads them back
before the ring would wrap: the persistent kernels between two launches, the in-kernel-sampler loop between two graph
replays or eager steps, the host-batch pipeline through its pinned buffer.  With the default 32 768-entry ring no fit
of the suite ever wraps it, so each fit here also runs with a ring of 7 entries, which every one of them wraps several
times; losses and parameters must be the bits of the same fit with the default ring. """
import warnings

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

if torch.cuda.is_available():
    from pydens_b200 import Solver, D, V, NumpySampler, fit_ensemble
    from pydens_b200 import engine
    from pydens_b200.engine import FusedEngine

SHORT_RING = 7


def _solver(j=0, cons=False):
    """ tutorial stage 5 (a trainable variable in the equation), optionally with a constraint at t = 0.5 """
    torch.manual_seed(100 + j)
    kw = dict(constraints=[lambda u, t: u(torch.tensor([0.5])) - 0.25]) if cons else {}
    return Solver(lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t) + V('new_var', data=torch.Tensor([1.0])),
                  ndims=1, initial_condition=1.0, layout='fafaf', features=[12, 10, 1], activation='Tanh',
                  device='cuda', backend='fused', seed=1000 + 7 * j, **kw)


def _host_sampler(j=0):
    return NumpySampler('beta', seed=50 + j, a=2.0, b=2.0)          # no in-kernel form: sampled on the host


def _stepwise(monkeypatch):
    def boom(*a, **k):
        raise AssertionError('the persistent path was taken')
    monkeypatch.setattr(FusedEngine, '_fit_persistent', boom)
    monkeypatch.setenv('PYDENS_B200_AUTO_PERSISTENT', '0')


def _persistent_in_kernel(monkeypatch):
    s = _solver()
    s.fit(niters=23, batch_size=100, steps_per_launch=5)
    s.fit(niters=60, batch_size=100, optimizer=None)                  # 50 steps per launch, from step 23 of the ring
    assert not s._engine._graphs
    return [s]


def _persistent_host_constraint(monkeypatch):
    s = _solver(cons=True)
    s.fit(niters=30, batch_size=64, sampler=_host_sampler(), loss_terms=['equation', 'constraint_0'], steps_per_launch=4)
    assert not s._engine._graphs
    return [s]


def _stepwise_graphs(monkeypatch):
    _stepwise(monkeypatch)
    s = _solver()
    s.fit(niters=70, batch_size=100)                                  # graphs of 4 steps, more than the ring has left
    s.fit(niters=66, batch_size=100, optimizer=None)
    assert s._engine._graphs
    return [s]


def _stepwise_no_graph(monkeypatch):
    _stepwise(monkeypatch)
    monkeypatch.setenv('PYDENS_B200_NO_GRAPH', '1')
    s = _solver()
    s.fit(niters=20, batch_size=100)
    assert not s._engine._graphs
    return [s]


def _stepwise_host(monkeypatch):
    _stepwise(monkeypatch)
    s = _solver()
    s.fit(niters=20, batch_size=100, sampler=_host_sampler())
    assert s._engine._graphs
    return [s]


def _ensemble(monkeypatch):
    members = [_solver(j) for j in range(3)]
    fit_ensemble(members, niters=23, batch_size=64, steps_per_launch=5)
    return members


FITS = {'persistent_in_kernel': _persistent_in_kernel, 'persistent_host_constraint': _persistent_host_constraint,
        'stepwise_graphs': _stepwise_graphs, 'stepwise_no_graph': _stepwise_no_graph, 'stepwise_host': _stepwise_host,
        'ensemble': _ensemble}


def _bits(solvers):
    return [(s._engine.flat.view(torch.int32).cpu().numpy(),
             np.array([float(x) for x in s.losses], dtype=np.float32).view(np.int32)) for s in solvers]


@pytest.mark.parametrize('case', list(FITS))
def test_short_ring_gives_the_same_bits(case, monkeypatch):
    runs = {}
    for ring_len in (engine._RING_LEN, SHORT_RING):
        with monkeypatch.context() as mp:
            mp.setattr(engine, '_RING_LEN', ring_len)
            with warnings.catch_warnings():
                warnings.simplefilter('error', UserWarning)           # each fit takes the path it is meant to
                solvers = FITS[case](mp)
            assert all(s._engine.ring.numel() == ring_len for s in solvers)
            runs[ring_len] = _bits(solvers)
    for j, ((pa, la), (pb, lb)) in enumerate(zip(runs[engine._RING_LEN], runs[SHORT_RING])):
        assert la.size > SHORT_RING and np.isfinite(la.view(np.float32)).all(), case
        assert np.array_equal(la, lb), '%s, solver %d: losses differ' % (case, j)
        assert np.array_equal(pa, pb), '%s, solver %d: parameters differ' % (case, j)
