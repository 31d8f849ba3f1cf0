""" Ensembles of tiny-batch fits in one persistent launch (fit_ensemble, pinn_multi_step_ensemble).

Every member of an ensemble must end where its solo `Solver.fit` ends, bit for bit: parameters, both Adam moments, the
optimizer's step tensors, the device step counter and the loss list.  Each test builds every member twice from the same
seeds — once for the ensemble, once for solo fits — and compares the raw bits.  The batch sizes pick the kernel and the
cluster size by the rule of pinn_multi_step_terms: 16 points -> 1 CTA, 32 -> 2, 64 -> 4, 100 -> 8, and batches above 256
(or PINN_MULTI_KERNEL=tile) -> the multi-step kernel, one CTA per member. """
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    from pydens_b200 import Solver, D, V, NumpySampler, fit_ensemble
    from pydens_b200 import _native as N

FEATURES, LAYOUT, ACT = [12, 10, 1], 'fafaf', 'Tanh'


def _make(j, kind='tutorial', init=None, cons=False):
    """ Member j: its own network initialisation, seed and (for the V problems) initial value of the variable. """
    torch.manual_seed(100 + j)
    v0 = 1.0 + 0.25 * j if init is None else init
    kw = dict(ndims=1, layout=LAYOUT, features=FEATURES, activation=ACT, device='cuda', backend='fused', seed=1000 + 7 * j)
    if kind == 'tutorial':          # tutorial stage 5: a trainable variable in the equation
        eq = lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t) + V('new_var', data=torch.Tensor([v0]))
        kw['initial_condition'] = 1.0
    elif kind == 'readme':          # README: V('init') in the initial condition
        eq = lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t)
        kw['initial_condition'] = lambda *a: V('init', data=torch.Tensor([v0]))
    elif kind == 'coef':            # a coefficient held as a frozen V
        eq = lambda u, t: D(u, t) - V('k', data=torch.Tensor([v0])) * torch.cos(2 * np.pi * t)
        kw['initial_condition'] = 1.0
    if cons:
        kw['constraints'] = [lambda u, t: u(torch.tensor([0.5])) - 0.25]
    s = Solver(eq, **kw)
    if kind == 'coef':
        s.model.freeze_trainable(variables=['k'])
    return s


def _state(s):
    eng = s._engine
    m, v, steps, _ = eng._adam_flat
    return dict(flat=eng.flat.view(torch.int32).clone(), m=m.view(torch.int32).clone(), v=v.view(torch.int32).clone(),
                steps=steps.view(torch.int32).clone(), counter=eng.step_counter.clone(), done=eng.steps_done,
                losses=np.array([float(x) for x in s.losses], dtype=np.float32).view(np.int32))


def _same(a, b, tag):
    for k in ('flat', 'm', 'v', 'steps', 'counter'):
        assert torch.equal(a[k], b[k]), '%s: %s differs' % (tag, k)
    assert a['done'] == b['done'], tag
    assert np.array_equal(a['losses'], b['losses']), '%s: losses differ' % tag


def _compare(M, fit, kind='tutorial', cons=False, sampler=None, prepare=None, inits=None, **kw):
    """ fit_ensemble of M members vs M solo fits; sampler(j) -> member j's sampler (a fresh object for each side). """
    members, solos = [], []
    for j in range(M):
        init = None if inits is None else inits[j]
        members.append(_make(j, kind, init, cons))
        solos.append(_make(j, kind, init, cons))
    if prepare:
        for j in range(M):
            prepare(j, members[j])
            prepare(j, solos[j])
    smp = None if sampler is None else [sampler(j) for j in range(M)]
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)            # the ensemble path itself, no fallback
        fit_ensemble(members, sampler=smp, **fit, **kw)
    for j in range(M):
        solos[j].fit(sampler=None if sampler is None else sampler(j), **fit, **kw)
    for j in range(M):
        _same(_state(members[j]), _state(solos[j]), 'member %d' % j)
    return members, solos


@pytest.mark.parametrize('batch', [16, 32, 64, 100])
def test_cluster_sizes_in_kernel_sampler(batch):
    _compare(3, dict(niters=23, batch_size=batch, steps_per_launch=8))


def test_auto_persistent_default_launches():
    _compare(2, dict(niters=60, batch_size=100))


@pytest.mark.parametrize('batch', [1000, 4096])
def test_multi_step_kernel(batch):
    _compare(3, dict(niters=6, batch_size=batch, steps_per_launch=4))


def test_multi_step_kernel_forced(monkeypatch):
    monkeypatch.setenv('PINN_MULTI_KERNEL', 'tile')
    _compare(3, dict(niters=20, batch_size=100, steps_per_launch=8))


@pytest.mark.parametrize('batch', [64, 1000])
def test_host_samplers(batch):
    _compare(3, dict(niters=20, batch_size=batch, steps_per_launch=8),
             sampler=lambda j: NumpySampler('beta', seed=50 + j, a=2.0, b=2.0))


@pytest.mark.parametrize('batch', [48, 600])
def test_constraint_terms(batch):
    _compare(3, dict(niters=20, batch_size=batch, steps_per_launch=8, loss_terms=['equation', 'constraint_0']),
             cons=True)


def test_V_in_initial_condition():
    _compare(4, dict(niters=20, batch_size=100, steps_per_launch=8), kind='readme')


@pytest.mark.parametrize('crit', ['huber', 'sum'])
def test_criteria(crit):
    criterion = torch.nn.HuberLoss(delta=0.05) if crit == 'huber' else torch.nn.MSELoss(reduction='sum')
    _compare(3, dict(niters=20, batch_size=64, steps_per_launch=8, criterion=criterion), kind='readme', cons=True,
             loss_terms=['equation', 'constraint_0'])


def test_frozen_masks_and_prior_histories():
    def prepare(j, s):
        if j == 1:
            s.model.freeze_trainable(variables=['new_var'])
        s.fit(niters=17 + 5 * j, batch_size=32, steps_per_launch=6)     # different optimizer states and step counters
    _compare(3, dict(niters=20, batch_size=32, steps_per_launch=8, optimizer=None), prepare=prepare)


def test_one_member():
    _compare(1, dict(niters=20, batch_size=100, steps_per_launch=8))


def test_more_members_than_one_wave():
    _compare(40, dict(niters=20, batch_size=100, steps_per_launch=10))


def test_split_launch():
    _compare(N.MAX_MEMBERS + 3, dict(niters=16, batch_size=16, steps_per_launch=8))


def test_frozen_coefficient_sweep():
    inits = [0.5, 1.0, 2.0, 4.0, 8.0]
    members, _ = _compare(5, dict(niters=30, batch_size=64, steps_per_launch=10), kind='coef', inits=inits)
    for s, k in zip(members, inits):                   # the frozen coefficient stays where it was set
        eng = s._engine
        assert float(eng.flat[eng._spec_kwargs['var_offsets']['k']]) == k


def test_nan_member_leaves_the_others_alone():
    def prepare(j, s):
        if j == 1:
            eng = s._get_engine()
            eng.flat.fill_(float('nan'))
    members, solos = _compare(3, dict(niters=20, batch_size=100, steps_per_launch=8), prepare=prepare)
    assert torch.isnan(members[1]._engine.flat).all()


def test_fit_after_the_ensemble_continues_like_solo_history():
    members, solos = _compare(3, dict(niters=20, batch_size=64, steps_per_launch=8))
    for s in members + solos:
        s.fit(niters=20, batch_size=64, steps_per_launch=8)
    fit_ensemble(members, niters=20, batch_size=64, steps_per_launch=8)
    for s in solos:
        s.fit(niters=20, batch_size=64, steps_per_launch=8)
    pts = torch.linspace(0, 1, 50)
    for j, (a, b) in enumerate(zip(members, solos)):
        _same(_state(a), _state(b), 'member %d' % j)
        assert np.array_equal(a.predict(pts), b.predict(pts))


def _raw_members(eng, M, points=None):
    """ M copies of one engine's state as raw buffers: params, moments, mask, steps, counter, ring per member. """
    n, bufs = eng.n_params, []
    for j in range(M):
        b = dict(params=eng.flat.clone(), m=torch.zeros(n, device='cuda'), v=torch.zeros(n, device='cuda'),
                 mask=torch.ones(n, device='cuda'), steps=torch.zeros(4, device='cuda'),
                 counter=torch.zeros(1, dtype=torch.int64, device='cuda'), ring=torch.zeros(64, device='cuda'))
        bufs.append(b)
    table = (N.PinnMember * M)()
    for j, b in enumerate(bufs):
        t = table[j]
        t.params, t.exp_avg, t.exp_avg_sq, t.mask = (b['params'].data_ptr(), b['m'].data_ptr(), b['v'].data_ptr(),
                                                     b['mask'].data_ptr())
        t.step_tensors, t.n_step_tensors, t.opt_step0 = b['steps'].data_ptr(), 4, 0.0
        t.points = points.data_ptr() if points is not None else None
        t.seed, t.step_counter, t.losses_ring = 77 + j, b['counter'].data_ptr(), b['ring'].data_ptr()
    return bufs, table


def _call(eng, M, table, n_points=64, k=5, n_terms=0, terms=None, stream=None):
    return eng.lib.pinn_multi_step_ensemble(eng.plan, M, table, C.c_int64(n_points), C.c_int(k), C.c_float(0.01),
                                            C.c_float(0.9), C.c_float(0.999), C.c_float(1e-8), C.c_float(0.0),
                                            C.c_int64(64), C.c_float(1.0 / n_points), C.c_int(n_terms), terms, None,
                                            stream if stream is not None else eng._stream())


@pytest.mark.parametrize('batch', [64, 1000])
def test_graph_capture_replays_the_direct_call(batch):
    eng = _make(0)._get_engine()
    direct, t_direct = _raw_members(eng, 4)
    assert _call(eng, 4, t_direct, n_points=batch) == 0
    graphed, t_graph = _raw_members(eng, 4)
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        g.capture_begin()
        rc = _call(eng, 4, t_graph, n_points=batch, stream=C.c_void_p(side.cuda_stream))
        g.capture_end()
    torch.cuda.current_stream().wait_stream(side)
    assert rc == 0
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(direct, graphed):
        for key in a:
            assert torch.equal(a[key].view(torch.int32) if a[key].dtype == torch.float32 else a[key],
                               b[key].view(torch.int32) if b[key].dtype == torch.float32 else b[key]), key


def test_c_call_refusals():
    eng = _make(0)._get_engine()
    bufs, table = _raw_members(eng, 2)
    assert _call(eng, 0, table) == N.E_INVALID
    big = (N.PinnMember * (N.MAX_MEMBERS + 1))()
    for j in range(N.MAX_MEMBERS + 1):
        C.memmove(C.addressof(big[j]), C.addressof(table[0]), C.sizeof(N.PinnMember))
    assert _call(eng, N.MAX_MEMBERS + 1, big) == N.E_INVALID
    saved = table[1].mask
    table[1].mask = None
    assert _call(eng, 2, table) == N.E_INVALID
    table[1].mask = saved
    table[1].params = bufs[1]['params'].data_ptr() + 4
    assert _call(eng, 2, table) == N.E_INVALID
    table[1].params = bufs[1]['params'].data_ptr()
    assert _call(eng, 2, table, n_points=eng.lib.pinn_multi_step_max_points(eng.plan) + 1) == N.E_INVALID
    # a constraint plan of another network
    torch.manual_seed(0)
    wider = Solver(lambda u, t: D(u, t) - 1.0, ndims=1, layout=LAYOUT, features=[16, 10, 1], activation=ACT,
                   initial_condition=1.0, constraints=[lambda u, t: u(torch.tensor([0.5])) - 0.25], device='cuda',
                   backend='fused')
    entry = wider._get_engine()._constraint_plan(0)
    assert entry is not None
    terms = (N.PinnTerm * 1)()
    terms[0].plan, terms[0].n_points, terms[0].point_weight = entry['plan'].value, entry['n'], 1.0
    terms[0].points = entry['host_points'].data_ptr()
    assert _call(eng, 2, table, n_terms=1, terms=terms) == N.E_INVALID
    # a plan without a persistent kernel: derivatives of order 3
    torch.manual_seed(0)
    hi = Solver(lambda u, t: D(D(D(u, t), t), t) - 1.0, ndims=1, layout=LAYOUT, features=FEATURES, activation=ACT,
                initial_condition=1.0, device='cuda', backend='fused')
    heng = hi._get_engine()
    hb, ht = _raw_members(heng, 1)
    assert _call(heng, 1, ht) == N.E_UNSUPPORTED
    torch.cuda.synchronize()
    # nothing ran: every buffer still holds its initial values
    for b in bufs:
        assert torch.equal(b['params'], eng.flat) and int(b['counter'].item()) == 0


def test_fit_ensemble_refuses_mismatched_and_duplicate_solvers():
    a, b = _make(0), _make(1)
    with pytest.raises(ValueError, match='same Solver'):
        fit_ensemble([a, b, a], niters=20, batch_size=64)
    torch.manual_seed(0)
    wider = Solver(lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t) + V('new_var', data=torch.Tensor([1.0])),
                   ndims=1, layout=LAYOUT, features=[16, 10, 1], activation=ACT, initial_condition=1.0, device='cuda',
                   backend='fused')
    with pytest.raises(ValueError, match='network'):
        fit_ensemble([a, wider], niters=20, batch_size=64)
    other_eq = _make(2, kind='coef')
    with pytest.raises(ValueError, match='equation program'):
        fit_ensemble([a, other_eq], niters=20, batch_size=64)
    assert a.losses == [] and b.losses == []


@pytest.mark.parametrize('case', ['sgd', 'large_batch'])
def test_fallback_warns_once_and_equals_sequential_fits(case):
    fit = dict(niters=20, batch_size=64, optimizer='SGD') if case == 'sgd' else dict(niters=20, batch_size=2000)
    members = [_make(j) for j in range(3)]
    solos = [_make(j) for j in range(3)]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        fit_ensemble(members, **fit)
    ours = [w for w in caught if 'fit_ensemble' in str(w.message)]
    assert len(ours) == 1 and issubclass(ours[0].category, UserWarning)
    for s in solos:
        s.fit(**fit)
    for j in range(3):
        assert torch.equal(members[j]._engine.flat, solos[j]._engine.flat), j
        assert np.array_equal(np.array(members[j].losses, dtype=np.float32), np.array(solos[j].losses, dtype=np.float32))
