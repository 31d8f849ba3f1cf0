""" Hyper-parameter sweeps in one persistent launch: fit_ensemble with Adam hyper-parameters of each member's own, and
pinn_multi_step_ensemble_adam under it.

1. Every member ends where its solo `Solver.fit` with the same lr, betas, eps and weight decay ends, bit for bit
   (parameters, both moments, step tensors, device step counter, loss list), on the cluster kernel at 1, 2, 4 and 8 CTAs
   per member, on the multi-step kernel, with a fused constraint, with host batches, with a frozen layer and resumed
   optimizer states, and over two launches of MAX_MEMBERS + 3 members.  The rows differ in every field; one has no weight
   decay and one has beta1 = 0.
2. pinn_multi_step_ensemble equals pinn_multi_step_ensemble_adam with equal rows, bit for bit, on both kernels.
3. Each member steps with its own row: one step from a zero Adam state with a beta1 per member gives
   exp_avg / (1 - beta1_j) = the fp64 oracle gradient, tensor by tensor; five steps from a used state follow
   oracle/adam.py with each member's row at the per-element bars of test_gpu_step_adam.py; lr = 0 keeps the parameters.
4. The C call refuses rows torch.optim.Adam refuses (and non-finite ones) and writes nothing.
5. Through fit_ensemble: optimizer=None with different optimizers, the SGD fallback, and a later `fit(optimizer=None)`.
"""
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

import test_gpu_ensemble as TE
import test_gpu_persistent as TPer

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    from test_gpu_step_adam import check_adam_elements
    from pydens_b200 import NumpySampler, fit_ensemble
    from pydens_b200 import _native as N

# four rows that differ in every field: one without weight decay, one with beta1 = 0
ROWS = [dict(lr=0.005, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0),
        dict(lr=0.02, betas=(0.0, 0.99), eps=1e-6, weight_decay=1e-3),
        dict(lr=0.001, betas=(0.8, 0.9999), eps=1e-7, weight_decay=0.01),
        dict(lr=0.01, betas=(0.95, 0.995), eps=1e-5, weight_decay=2e-4)]


def _row(j):
    """ member j's hyper-parameters: ROWS cycled, the lr moved by 10 % per cycle so that no two members share one """
    h = dict(ROWS[j % len(ROWS)])
    h['lr'] *= 1.0 + 0.1 * (j // len(ROWS))
    return h


def _sweep(M):
    """ fit_ensemble's per-member keyword arguments for members 0 .. M-1 """
    rows = [_row(j) for j in range(M)]
    return {key: [h[key] for h in rows] for key in ('lr', 'betas', 'eps', 'weight_decay')}


def _compare(M, fit, kind='tutorial', cons=False, sampler=None, prepare=None, optimizer='Adam'):
    """ fit_ensemble of M members with rows _row(j) against M solo fits with the same rows """
    members, solos = [], []
    for j in range(M):
        members.append(TE._make(j, kind, None, cons))
        solos.append(TE._make(j, kind, None, cons))
    if prepare:
        for j in range(M):
            prepare(j, members[j])
            prepare(j, solos[j])
    smp = None if sampler is None else [sampler(j) for j in range(M)]
    sweep = _sweep(M) if optimizer is not None else {}
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)            # the ensemble path itself, no fallback
        fit_ensemble(members, sampler=smp, optimizer=optimizer, **fit, **sweep)
    for j in range(M):
        solo_kw = {key: v[j] for key, v in sweep.items()}
        solos[j].fit(sampler=None if sampler is None else sampler(j), optimizer=optimizer, **fit, **solo_kw)
    for j in range(M):
        TE._same(TE._state(members[j]), TE._state(solos[j]), 'member %d' % j)
    return members, solos


# ---- 1. bit-identity with solo fits -----------------------------------------------------------------------------------
@pytest.mark.parametrize('batch', [16, 32, 64, 100])
def test_cluster_sizes(batch):
    _compare(5, dict(niters=23, batch_size=batch, steps_per_launch=8))


def test_multi_step_kernel():
    _compare(5, dict(niters=6, batch_size=1000, steps_per_launch=4))


def test_multi_step_kernel_forced(monkeypatch):
    monkeypatch.setenv('PINN_MULTI_KERNEL', 'tile')
    _compare(5, dict(niters=20, batch_size=100, steps_per_launch=8))


@pytest.mark.parametrize('batch', [48, 600])
def test_constraint_term(batch):
    _compare(4, dict(niters=20, batch_size=batch, steps_per_launch=8, loss_terms=['equation', 'constraint_0']),
             cons=True)


@pytest.mark.parametrize('batch', [64, 1000])
def test_host_samplers(batch):
    _compare(4, dict(niters=20, batch_size=batch, steps_per_launch=8),
             sampler=lambda j: NumpySampler('beta', seed=50 + j, a=2.0, b=2.0))


def test_frozen_layer_and_resumed_states_keep_their_own_optimizers():
    """ each member first fits alone with its own row for 17 + 5 j steps (member 1 with its first layer frozen), then
    the ensemble continues every member's own optimizer (optimizer=None): different settings and step counts """
    def prepare(j, s):
        if j == 1:
            for p in s.model.conv_block.ops[0].parameters():
                p.requires_grad_(False)
        h = _row(j)
        s.fit(niters=17 + 5 * j, batch_size=32, steps_per_launch=6, **h)
    members, _ = _compare(4, dict(niters=20, batch_size=32, steps_per_launch=8), prepare=prepare, optimizer=None)
    for j, s in enumerate(members):
        g = s.optimizer.param_groups[0]
        assert (g['lr'], tuple(g['betas']), g['eps'], g['weight_decay']) == tuple(_row(j).values()), j


def test_split_launch():
    _compare(N.MAX_MEMBERS + 3, dict(niters=16, batch_size=16, steps_per_launch=8))


# ---- 2. the two C entry points ----------------------------------------------------------------------------------------
def _hyper(rows):
    arr = (N.PinnAdamHyper * len(rows))()
    for a, h in zip(arr, rows):
        a.lr, (a.beta1, a.beta2), a.eps, a.weight_decay = h['lr'], h['betas'], h['eps'], h['weight_decay']
    return arr


def _call_adam(eng, M, table, hyper, n_points=64, k=5, ring_len=64):
    """ pinn_multi_step_ensemble_adam without constraint terms; ring_len 64 is the rings of TE._raw_members """
    return eng.lib.pinn_multi_step_ensemble_adam(eng.plan, M, table, hyper, C.c_int64(n_points), C.c_int(k),
                                                 C.c_int64(ring_len), C.c_float(1.0 / n_points), C.c_int(0), None, None,
                                                 eng._stream())


def _bits(bufs):
    return [{key: (b[key].view(torch.int32) if b[key].dtype == torch.float32 else b[key]).clone() for key in b}
            for b in bufs]


@pytest.mark.parametrize('batch', [64, 1000])
def test_old_entry_point_equals_equal_rows(batch):
    eng = TE._make(0)._get_engine()
    old, t_old = TE._raw_members(eng, 4)
    assert TE._call(eng, 4, t_old, n_points=batch) == 0                 # lr 0.01, betas (0.9, 0.999), eps 1e-8, wd 0
    new, t_new = TE._raw_members(eng, 4)
    rows = [dict(lr=0.01, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)] * 4
    assert _call_adam(eng, 4, t_new, _hyper(rows), n_points=batch) == 0
    torch.cuda.synchronize()
    for j, (a, b) in enumerate(zip(_bits(old), _bits(new))):
        for key in a:
            assert torch.equal(a[key], b[key]), 'member %d: %s' % (j, key)
    assert int(old[0]['counter']) == 5


# ---- 3. each member steps with its own row ----------------------------------------------------------------------------
NAME = 'heat1d_icvar'              # variables in the equation and in the initial condition, log_scale


def _members(eng, states, points):
    """ a member table over TPer._State objects (rings of one loss), all on the device batch `points` """
    table = (N.PinnMember * len(states))()
    for t, st in zip(table, states):
        t.params, t.exp_avg, t.exp_avg_sq, t.mask = (st.p.data_ptr(), st.m.data_ptr(), st.v.data_ptr(),
                                                     st.mask.data_ptr())
        t.step_tensors, t.n_step_tensors = st.steps.data_ptr(), st.steps.numel()
        t.opt_step0 = float(st.steps[0])
        t.points, t.seed, t.step_counter, t.losses_ring = points.data_ptr(), 5, st.counter.data_ptr(), st.ring.data_ptr()
    return table


@pytest.mark.parametrize('kernel,n', [('small', 100), ('multi', 700)])
def test_first_step_moment_is_each_members_gradient(kernel, n):
    """ from a zero Adam state, one step leaves exp_avg = fmaf(1 - beta1_j, g, 0): dividing by member j's own
    (1 - beta1) gives the fp64 oracle gradient; a kernel that used member 0's beta1 everywhere misses it by up to 20x """
    solver = TPer._solver(NAME)
    eng = solver._get_engine()
    TPer._preconditions(NAME, eng, kernel)
    assert TPer._kernel_for(eng, n, {})[0] == kernel
    params = solver.flat_params().cpu().numpy()
    pts, ref = TPer._oracle_prefixes(NAME, params, [n])
    beta1 = [0.9, 0.0, 0.5, 0.95]
    rows = [dict(lr=1e-3 * (j + 1), betas=(b, 0.999 - 0.001 * j), eps=1e-8, weight_decay=0.0) for j, b in enumerate(beta1)]
    states = [TPer._State.fresh(eng, params) for _ in rows]
    dev_pts = torch.from_numpy(pts[:n]).cuda().reshape(1, n, -1).contiguous()
    N.check(_call_adam(eng, len(rows), _members(eng, states, dev_pts), _hyper(rows), n_points=n, k=1, ring_len=1))
    torch.cuda.synchronize()
    for j, (st, h) in enumerate(zip(states, rows)):
        m = st.m.cpu().numpy()
        g = m / (np.float32(1.0) - np.float32(h['betas'][0]))
        tag = '%s n=%d member %d (beta1 %g)' % (kernel, n, j, h['betas'][0])
        TPer._check_against_oracle(NAME, eng, float(st.ring[0]), g, ref[n], tag)
        b2 = np.float32(h['betas'][1])
        want = (np.float32(1.0) - b2) * g * g
        assert (np.abs(st.v.cpu().numpy() - want) <= 1e-5 * want + 1e-38).all(), tag


OPT_STEP0 = 37


@pytest.mark.parametrize('kernel,n', [('small', 100), ('multi', 700)])
def test_five_steps_follow_oracle_adam_per_member(kernel, n):
    """ five steps from a used state (random moments, 37 steps taken, about 1/7 of the entries frozen, log_scale and
    the first bias among them) with four different rows, each step against oracle/adam.py with the member's row at the
    per-element bars of test_gpu_step_adam.check_adam_elements.  The gradient each member's update was made from is the
    kernel's own: a probe member on the same parameters and batch, with a zero state and beta1 = 0, holds it bit for bit
    in its exp_avg after the step (fmaf(1, g, 0) = g). """
    solver = TPer._solver(NAME)
    eng = solver._get_engine()
    TPer._preconditions(NAME, eng, kernel)
    assert TPer._kernel_for(eng, n, {})[0] == kernel
    params = solver.flat_params().cpu().numpy()
    rng = np.random.RandomState(21)
    g_scale = np.abs(rng.randn(eng.n_params)).astype(np.float32) * 1e-2
    mask = np.ones(eng.n_params, dtype=np.float32)
    mask[rng.choice(eng.n_params, eng.n_params // 7, replace=False)] = 0.0
    names = dict(TPer._tensors(NAME, eng))
    mask[names['log_scale']] = 0.0
    mask[names['b0']] = 0.0
    M = len(ROWS)
    states = []
    for j in range(M):
        st = TPer._State.fresh(eng, params)
        st.m.copy_(torch.from_numpy((g_scale * rng.randn(eng.n_params)).astype(np.float32)))
        st.v.copy_(torch.from_numpy((g_scale * g_scale * rng.uniform(0.5, 2.0, eng.n_params)).astype(np.float32)))
        st.mask.copy_(torch.from_numpy(mask))
        st.steps.fill_(float(OPT_STEP0))
        states.append(st)
    probe_row = dict(lr=0.0, betas=(0.0, 0.5), eps=1.0, weight_decay=0.0)
    hyper = _hyper(ROWS + [probe_row] * M)
    worst = {}
    for s in range(5):
        pts = torch.from_numpy(TPer._points(NAME, n, seed=300 + s)).cuda().reshape(1, n, -1).contiguous()
        probes = [TPer._State.fresh(eng, st.p.cpu().numpy()) for st in states]
        before = [(st.p.cpu().numpy(), st.m.cpu().numpy(), st.v.cpu().numpy()) for st in states]
        N.check(_call_adam(eng, 2 * M, _members(eng, states + probes, pts), hyper, n_points=n, k=1, ring_len=1))
        torch.cuda.synchronize()
        t = OPT_STEP0 + s + 1
        for j, (st, pr) in enumerate(zip(states, probes)):
            h = ROWS[j]
            h32 = dict(lr=h['lr'], beta1=h['betas'][0], beta2=h['betas'][1], eps=h['eps'], weight_decay=h['weight_decay'])
            p0, m0, v0 = before[j]
            g = pr.m.cpu().numpy()
            assert torch.equal(pr.p, torch.from_numpy(p0).cuda())                 # lr = 0: the probe did not move
            w = check_adam_elements('%s n=%d member %d step %d' % (kernel, n, j, s), h32, t, p0, m0, v0, g, mask,
                                    (st.p.cpu().numpy(), st.m.cpu().numpy(), st.v.cpu().numpy()))
            worst = {key: max(val, worst.get(key, 0.0)) for key, val in w.items()}
            assert torch.equal(st.steps, torch.full_like(st.steps, float(t)))
    print('NOISE sweep %s n=%d: %s' % (kernel, n, ' '.join('%s %.3f' % kv for kv in worst.items())))


@pytest.mark.parametrize('batch', [64, 1000])
def test_zero_lr_keeps_the_parameters(batch):
    eng = TE._make(0)._get_engine()
    bufs, table = TE._raw_members(eng, 2)
    rows = [dict(lr=0.0, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01),
            dict(lr=0.01, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)]
    assert _call_adam(eng, 2, table, _hyper(rows), n_points=batch) == 0
    torch.cuda.synchronize()
    assert torch.equal(bufs[0]['params'].view(torch.int32), eng.flat.view(torch.int32))
    assert bool((bufs[0]['m'] != 0).any()) and bool((bufs[0]['v'] != 0).any())
    assert not torch.equal(bufs[1]['params'], eng.flat)
    assert int(bufs[0]['counter']) == 5 and float(bufs[0]['steps'][0]) == 5.0


# ---- 4. refusals ------------------------------------------------------------------------------------------------------
BAD = [('lr', float('nan')), ('lr', -1.0), ('lr', float('inf')), ('beta1', 1.0), ('beta2', 1.0), ('beta1', -0.1),
       ('eps', -1e-8), ('eps', float('inf')), ('weight_decay', -1e-4), ('weight_decay', float('nan'))]


def test_c_call_refusals():
    eng = TE._make(0)._get_engine()
    bufs, table = TE._raw_members(eng, 2)
    good = [dict(lr=0.01, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)] * 2
    assert _call_adam(eng, 2, table, None) == N.E_INVALID
    for field, value in BAD:
        hyper = _hyper(good)
        setattr(hyper[1], field, value)
        assert _call_adam(eng, 2, table, hyper) == N.E_INVALID, (field, value)
        assert 'member 1' in eng.lib.pinn_last_error().decode()
    torch.cuda.synchronize()
    for b in bufs:                                   # nothing ran: every buffer still holds its initial values
        assert torch.equal(b['params'], eng.flat) and int(b['counter'].item()) == 0
        assert not bool(b['m'].any()) and not bool(b['ring'].any()) and not bool(b['steps'].any())


# ---- 5. through fit_ensemble ------------------------------------------------------------------------------------------
def test_optimizer_none_with_different_optimizers_trains_together():
    """ members whose optimizers differ only in lr, as a solo history leaves them, train in one launch """
    def prepare(j, s):
        s.fit(niters=10, batch_size=64, steps_per_launch=5, lr=0.002 * (j + 1))
    _compare(3, dict(niters=20, batch_size=64, steps_per_launch=8), prepare=prepare, optimizer=None)


def test_sgd_with_an_lr_list_falls_back_once():
    lrs = [0.001, 0.003, 0.01]
    members = [TE._make(j) for j in range(3)]
    solos = [TE._make(j) for j in range(3)]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        fit_ensemble(members, niters=20, batch_size=64, optimizer='SGD', lr=lrs)
    ours = [w for w in caught if 'fit_ensemble' in str(w.message)]
    assert len(ours) == 1 and issubclass(ours[0].category, UserWarning)
    for s, lr in zip(solos, lrs):
        s.fit(niters=20, batch_size=64, optimizer='SGD', lr=lr)
    for j in range(3):
        assert members[j].optimizer.param_groups[0]['lr'] == lrs[j]
        assert torch.equal(members[j]._engine.flat, solos[j]._engine.flat), j
        assert np.array_equal(np.array(members[j].losses, dtype=np.float32), np.array(solos[j].losses, dtype=np.float32))


def test_fit_after_the_sweep_continues_like_solo_history():
    M = 4
    members, solos = _compare(M, dict(niters=20, batch_size=64, steps_per_launch=8))
    for j, s in enumerate(members):
        g = s.optimizer.param_groups[0]
        h = _row(j)
        assert (g['lr'], tuple(g['betas']), g['eps'], g['weight_decay']) == (h['lr'], h['betas'], h['eps'],
                                                                           h['weight_decay']), j
    for s in members + solos:
        s.fit(niters=20, batch_size=64, steps_per_launch=8, optimizer=None)
    pts = torch.linspace(0, 1, 50)
    for j, (a, b) in enumerate(zip(members, solos)):
        TE._same(TE._state(a), TE._state(b), 'member %d' % j)
        assert np.array_equal(a.predict(pts), b.predict(pts))
