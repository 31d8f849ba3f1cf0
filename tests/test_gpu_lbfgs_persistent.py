""" L-BFGS in the persistent cluster kernel (pinn_lbfgs_multi, pinn_lbfgs_multi_ensemble): the gradient it steps on
against the fp64 oracle, its steps against the stepwise device L-BFGS (one pinn_lbfgs_advance per evaluation), launch
boundaries, the hand-over to and from torch's LBFGS, ensembles against solo fits, and the refusals. """
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

import gpu_helpers
import problems as P
from helpers import rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    from oracle import autograd_port as ap
    from pydens_b200 import Solver, D, V, fit_ensemble
    from pydens_b200 import _native as N


def make_solver(name, seed=0, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        s = gpu_helpers.make_solver(name, seed=seed, **kw)
        s._get_engine()
    return s


def readme_solver(seed=0):
    """ README.md:112-126: V('init') in the initial condition and the constraint u(0.5) = 0.25 """
    torch.manual_seed(seed)
    return Solver(lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t), ndims=1,
                  initial_condition=lambda *a: V('init', data=torch.Tensor([3.0])), layout='fafaf', features=[12, 10, 1],
                  activation='Tanh', constraints=[lambda u, t: u(torch.tensor([0.5])) - 0.25], device='cuda',
                  backend='fused', seed=1234)


README_TERMS = ['equation', 'constraint_0']


def lbfgs_state(opt):
    return opt.state[opt.param_groups[0]['params'][0]]


def state_bytes(solver):
    return solver._get_engine()._lbfgs['state'].cpu().numpy().tobytes()


# ---- the gradient of an evaluation, against the fp64 oracle ------------------------------------------------------------
def oracle(name, params):
    cfg = P.PROBLEMS[name]
    holder = {}
    ic = cfg['ic_factory'](lambda n, init: holder['prob'].V(n, init)) if 'ic_factory' in cfg else cfg['ic']
    prob = ap.Problem(lambda u, *xs, D, V: cfg['equation'](u, *xs, D=D, V=V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                      initial_condition=ic, boundary_condition=cfg['bc'], domain=cfg['domain'], features=cfg['features'],
                      activation=cfg['activation'], dtype=torch.float64, variables=cfg.get('variables'),
                      layout=cfg['layout'])
    holder['prob'] = prob
    prob.load_flat(torch.as_tensor(np.asarray(params, dtype=np.float64)))
    return prob


def check_against_oracle(eng, loss, grads, ref, tag):
    """ the bars of test_gpu_persistent.py: loss 2e-5, whole gradient 1e-4, each tensor 1e-4 (scalars 3e-4) of the
    oracle, relaxed by the residual's cancellation factor """
    ref_loss, ref_res, ref_g = ref
    cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(ref_res)))), 1e-30))
    assert np.isfinite(grads).all() and np.isfinite(loss), tag
    assert abs(loss - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), (tag, loss, ref_loss)
    assert rel_l2(grads[:ref_g.size], ref_g) <= 1e-4 * cond, tag
    s = eng.spec
    scale = 1e-3 * np.linalg.norm(ref_g)
    tensors = []
    for l in range(s.n_layers):
        tensors.append(('W%d' % l, slice(s.w_off[l], s.w_off[l] + s.widths[l] * s.widths[l + 1])))
        tensors.append(('b%d' % l, slice(s.b_off[l], s.b_off[l] + s.widths[l + 1])))
    tensors.append(('log_scale', slice(s.log_scale_off, s.log_scale_off + 1)))
    tensors += [('V%d' % i, slice(s.var_off[i], s.var_off[i] + 1)) for i in range(s.n_vars)]
    for tname, sl in tensors:
        err = np.linalg.norm(grads[sl] - ref_g[sl]) / max(np.linalg.norm(ref_g[sl]), scale, 1e-30)
        tol = (3e-4 if tname == 'log_scale' or tname.startswith('V') else 1e-4) * cond
        assert err <= tol, '%s: %s rel err %.2e' % (tag, tname, err)


def first_direction(eng, params, n, points=None, terms=None, point_weight=None):
    """ One pinn_lbfgs_multi step of max_iter=1, fixed step, from a fresh state: -> (d = -g from state vector 0, the
    step's loss from the ring, the batch it drew) """
    dev = eng.device
    flat = torch.as_tensor(np.asarray(params, dtype=np.float32)).to(dev).contiguous()
    mask = torch.zeros(eng.n_params, dtype=torch.float32, device=dev)
    nreal = sum(p.numel() for p, _ in eng.entries)
    mask[:nreal] = 1.0
    state = torch.zeros(eng.lib.pinn_lbfgs_state_bytes(eng.n_params, 4), dtype=torch.uint8, device=dev)
    counter = torch.full((1,), 7, dtype=torch.int64, device=dev)
    ring = torch.zeros(16, dtype=torch.float32, device=dev)
    cfg = N.PinnLbfgs(lr=1.0, tolerance_grad=0.0, tolerance_change=0.0, max_iter=1, max_eval=2, history_size=4,
                      line_search=0, mask=mask.data_ptr(), losses_ring=ring.data_ptr(), ring_len=16,
                      step_counter=counter.data_ptr())
    pts = None if points is None else torch.as_tensor(points).to(dev).contiguous()
    term_arr = (N.PinnTerm * 4)()
    for i, e in enumerate(terms or []):
        term_arr[i].plan, term_arr[i].n_points = e['plan'].value, e['n']
        term_arr[i].point_weight, term_arr[i].points = 1.0 / e['n'], e['host_points'].data_ptr()
    N.check(eng.lib.pinn_lbfgs_multi(eng.plan, C.byref(cfg), C.c_void_p(flat.data_ptr()), C.c_void_p(state.data_ptr()),
                                     C.c_void_p(pts.data_ptr()) if pts is not None else None, None, C.c_uint64(eng.seed),
                                     C.c_int64(n), C.c_int(1), C.c_float(point_weight or 1.0 / n),
                                     C.c_int(len(terms or [])), term_arr, eng._stream()))
    torch.cuda.synchronize()
    assert int(counter) == 8
    lay = N.lbfgs_layout(eng.n_params, 4)
    d = state[lay['vectors']:lay['vectors'] + 4 * eng.n_params].view(torch.float32).cpu().numpy()
    drawn = pts if pts is not None else eng.sample(n, step=7)
    return -d, float(ring[7].item()), drawn.cpu().numpy()


BATCHES = [1, 16, 17, 128, 129, 1024]


@pytest.mark.parametrize('cluster', [1, 2, 4, 8])
@pytest.mark.parametrize('name', ['poisson2d', 'ode_tanh', 'heat1d_icvar'])
def test_first_direction_is_the_fp64_gradient(name, cluster, monkeypatch):
    """ from a fresh state the first iteration sets d = -g: the evaluation's gradient, per tensor, at every batch edge,
    from host batches and (for the largest) from the in-kernel sampler; heat1d_icvar has V() in its initial condition """
    monkeypatch.setenv('PINN_SMALL_CLUSTER', str(cluster))
    s = make_solver(name)
    eng = s._get_engine()
    assert int(eng.info.small_batch_points) == 1024
    params = s.flat_params().cpu().numpy()
    prob = oracle(name, params)
    rng = np.random.RandomState(3)
    pts = np.concatenate([rng.uniform(lo, hi, size=(1024, 1)) for lo, hi in P.PROBLEMS[name]['ranges']],
                         axis=1).astype(np.float32)
    for n in BATCHES:
        for host in (True, False) if n in (17, 1024) else (True,):
            g, loss, drawn = first_direction(eng, params, n, pts[:n] if host else None)
            with warnings.catch_warnings():
                warnings.simplefilter('ignore', UserWarning)
                ref_l, ref_r, ref_g = prob.loss_and_grads(drawn.astype(np.float64))
            check_against_oracle(eng, loss, g, (ref_l, ref_r, ref_g.numpy()), '%s n=%d host=%s' % (name, n, host))


@pytest.mark.parametrize('cluster', [1, 2, 4, 8])
def test_first_direction_with_a_constraint_term(cluster, monkeypatch):
    """ the README flow's constraint u(0.5) = 0.25 rides along: -g equals the fused evaluation of the stepwise path (the
    equation launch plus the constraint launch, both held to the fp64 oracle by test_gpu_persistent_terms.py) """
    monkeypatch.setenv('PINN_SMALL_CLUSTER', str(cluster))
    s = readme_solver()
    eng = s._get_engine()
    terms = eng._persistent_terms(README_TERMS, 100)
    assert terms
    params = s.flat_params().cpu().numpy()
    for n in (1, 17, 129):
        pts = np.random.RandomState(n).uniform(0, 1, size=(n, 1)).astype(np.float32)
        g, loss, _ = first_direction(eng, params, n, pts, terms=terms)
        ev = eng._eval_setup(1, n, gpu_helpers.Replay([pts]), README_TERMS, torch.nn.MSELoss())
        eng._evaluate(ev, torch.as_tensor(pts).cuda())
        torch.cuda.synchronize()
        out = eng.out.cpu().numpy()
        assert abs(loss - out[eng.n_params]) <= 1e-5 * abs(out[eng.n_params])
        assert rel_l2(g, out[:eng.n_params]) <= 1e-5, n


# ---- against the stepwise device L-BFGS ---------------------------------------------------------------------------------
def fit_steps(solver, n_steps, batch, persistent, terms=('equation',), **kw):
    """ n_steps fits of one step each (the first builds the optimizer) -> (losses, evaluations per step, n_iter) """
    evals, iters = [], []
    for i in range(n_steps):
        args = dict(optimizer='LBFGS', **kw) if i == 0 else dict(optimizer=None)
        if persistent:
            args['steps_per_launch'] = 1
        with warnings.catch_warnings():
            warnings.filterwarnings('error', message='.*steps_per_launch')
            solver.fit(1, batch, loss_terms=list(terms), **args)
        st = lbfgs_state(solver.optimizer)
        evals.append(int(st['func_evals']) - sum(evals))
        iters.append(int(st['n_iter']))
    return [float(x) for x in solver.losses], evals, iters


CASES = [('poisson2d', None), ('poisson2d', 'strong_wolfe'), ('ode_tanh', None), ('ode_tanh', 'strong_wolfe')]


@pytest.mark.parametrize('name,ls', CASES)
def test_steps_match_the_stepwise_device_lbfgs(name, ls, monkeypatch):
    """ three steps from the same start on the same batches, each path on its own kernels: the cluster kernel sums the
    gradient in another order than the step kernel (~1e-7 apart, test_first_direction_is_the_fp64_gradient), and the
    iterations amplify that: with max_iter=20 and a fixed step, poisson2d's second and third step losses part by 1.3e-4
    and 2e-4 on an H100 (the evaluation counts still equal).  Five iterations per step stay within the bar. """
    kw = dict(lr=1.0, max_iter=5, line_search_fn=ls) if ls else dict(lr=0.05, max_iter=5)
    a, b = make_solver(name), make_solver(name)
    got = fit_steps(a, 3, 400, True, **kw)
    monkeypatch.setenv('PYDENS_B200_AUTO_PERSISTENT', '0')
    ref = fit_steps(b, 3, 400, False, **kw)
    assert got[1] == ref[1] and got[2] == ref[2], (got, ref)
    for x, y in zip(got[0], ref[0]):
        assert abs(x - y) <= 1e-4 * abs(y), (got, ref)


def test_readme_flow_with_its_constraint_trains_like_the_stepwise_path(monkeypatch):
    """ 100 steps of the README flow, each on a fresh batch, against the stepwise path.  Over 100 steps the two
    trajectories part (their gradients are summed in different orders); measured on an H100 with strong Wolfe and
    max_iter=2 they end 0.1 % apart at seed 0 and 13-15 % apart at seeds 1 and 2, and with max_iter=5 27-35 % apart at
    losses near 1e-5.  With a fixed step (lr 0.01-0.05) both paths diverge or reach NaN at some seeds: L-BFGS pairs
    from a new batch every step are not a stable fixed-step method on this problem. """
    kw = dict(lr=1.0, max_iter=2, line_search_fn='strong_wolfe')
    a, b = readme_solver(), readme_solver()
    with warnings.catch_warnings():
        warnings.filterwarnings('error', message='.*steps_per_launch')
        a.fit(100, 100, loss_terms=README_TERMS, optimizer='LBFGS', **kw)      # by itself: tiny batch, >= 16 steps
    monkeypatch.setenv('PYDENS_B200_AUTO_PERSISTENT', '0')
    b.fit(100, 100, loss_terms=README_TERMS, optimizer='LBFGS', **kw)
    la, lb = float(a.losses[-1]), float(b.losses[-1])
    assert len(a.losses) == len(b.losses) == 100 and np.isfinite(a.losses).all() and np.isfinite(b.losses).all()
    assert abs(la - lb) <= 0.1 * abs(lb), (la, lb)
    assert la < 1e-3 * float(a.losses[0])


# ---- launch boundaries and reruns -----------------------------------------------------------------------------------------
@pytest.mark.parametrize('ls', [None, 'strong_wolfe'])
def test_launch_boundaries_are_invisible(ls):
    kw = dict(lr=1.0, max_iter=10, line_search_fn=ls) if ls else dict(lr=0.05, max_iter=10)
    runs = []
    for how in ('k40', 'k7', 'split', 'k40'):
        s = make_solver('poisson2d')
        if how == 'split':
            s.fit(20, 200, optimizer='LBFGS', **kw)
            s.fit(20, 200, optimizer=None)
        else:
            s.fit(40, 200, optimizer='LBFGS', steps_per_launch=int(how[1:]), **kw)
        st = lbfgs_state(s.optimizer)
        runs.append((np.array(s.losses), s.flat_params().cpu().numpy(), state_bytes(s),
                     int(st['n_iter']), int(st['func_evals']),
                     torch.cat([t.cpu() for t in st['old_dirs'] + st['old_stps']]).numpy()))
    for r in runs[1:]:
        assert np.array_equal(r[0], runs[0][0]) and np.array_equal(r[1], runs[0][1]) and r[2] == runs[0][2]
        assert r[3:5] == runs[0][3:5] and np.array_equal(r[5], runs[0][5])


# ---- hand-over with torch's LBFGS -----------------------------------------------------------------------------------------
def torch_step(solver, batch):
    eng = solver._get_engine()
    pts = eng.sample(batch, step=eng.steps_done)

    def closure():
        return torch.tensor(eng.loss_and_grads(pts)[0])
    loss = float(solver.optimizer.step(closure))
    eng.steps_done += 1
    eng.step_counter += 1
    return loss


def test_hand_over_to_and_from_torch(monkeypatch):
    """ from the state a persistent fit exported, torch's opt.step(closure) and the stepwise device step agree (the bars
    of test_continuation_and_alternation_with_torch); from a state torch stepped, the persistent and the stepwise
    device steps agree """
    kw = dict(lr=1.0, max_iter=8, line_search_fn='strong_wolfe')
    a, b = make_solver('poisson2d'), make_solver('poisson2d')
    for s in (a, b):
        s.fit(16, 200, optimizer='LBFGS', **kw)                 # persistent by itself, bit-identical twice
    assert torch.equal(a.flat_params(), b.flat_params()) and state_bytes(a) == state_bytes(b)
    la = torch_step(a, 200)                                      # torch from the exported state
    monkeypatch.setenv('PYDENS_B200_AUTO_PERSISTENT', '0')
    b.fit(1, 200, optimizer=None)                                # the stepwise device step from the device state
    lb = float(b.losses[-1])
    assert abs(la - lb) <= 1e-3 * abs(lb), (la, lb)
    assert rel_l2(a.flat_params().cpu().numpy(), b.flat_params().cpu().numpy()) <= 1e-2
    # and back: both take one torch step, then one device step from torch's state, persistent against stepwise
    b.load_flat_params(a.flat_params())
    b._get_engine()._lbfgs = None
    b.optimizer.load_state_dict(a.optimizer.state_dict())
    for s in (a, b):
        torch_step(s, 200)
    a.fit(1, 200, optimizer=None, steps_per_launch=1)
    b.fit(1, 200, optimizer=None)
    la, lb = float(a.losses[-1]), float(b.losses[-1])
    assert abs(la - lb) <= 1e-3 * abs(lb), (la, lb)
    assert lbfgs_state(a.optimizer)['func_evals'] == lbfgs_state(b.optimizer)['func_evals']
    assert rel_l2(a.flat_params().cpu().numpy(), b.flat_params().cpu().numpy()) <= 1e-2


# ---- ensembles -----------------------------------------------------------------------------------------------------------
def solo_and_members(M, lr, batch=100, niters=20, name='poisson2d', **kw):
    members = [make_solver(name, seed=j) for j in range(M)]
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)            # the ensemble path: no warning
        fit_ensemble(members, niters, batch, optimizer='LBFGS', lr=lr, **kw)
    lrs = lr if isinstance(lr, list) else [lr] * M
    for j, m in enumerate(members):
        s = make_solver(name, seed=j)
        s.fit(niters, batch, optimizer='LBFGS', lr=lrs[j], **kw)
        assert np.array_equal(np.array(m.losses), np.array(s.losses)), j
        assert torch.equal(m.flat_params(), s.flat_params()), j
        assert state_bytes(m) == state_bytes(s), j
    return members


@pytest.mark.parametrize('M', [1, 3, 8, 130])
def test_ensemble_members_are_their_solo_fits(M):
    solo_and_members(M, 1.0, niters=16 if M == 130 else 20, max_iter=5, line_search_fn='strong_wolfe')


def test_ensemble_per_member_lr():
    solo_and_members(3, [0.02, 0.05, 0.1], max_iter=5)


def test_ensemble_nan_member_leaves_the_others_alone():
    members = [make_solver('poisson2d', seed=j) for j in range(3)]
    bad = members[1].flat_params().clone()
    bad[0] = float('nan')
    members[1].load_flat_params(bad)
    fit_ensemble(members, 16, 100, optimizer='LBFGS', lr=1.0, max_iter=5, line_search_fn='strong_wolfe')
    for j in (0, 2):
        s = make_solver('poisson2d', seed=j)
        s.fit(16, 100, optimizer='LBFGS', lr=1.0, max_iter=5, line_search_fn='strong_wolfe')
        assert np.array_equal(np.array(members[j].losses), np.array(s.losses))
        assert torch.equal(members[j].flat_params(), s.flat_params())


def test_ensemble_of_fits_the_kernel_does_not_take_warns_and_runs_them_in_turn():
    members = [make_solver('poisson2d', seed=j) for j in range(2)]
    with pytest.warns(UserWarning, match='one after another'):
        fit_ensemble(members, 4, 100, optimizer='LBFGS', lr=1.0, max_iter=5)      # 4 steps: a solo fit is stepwise
    assert all(len(m.losses) == 4 for m in members)


# ---- refusals ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['poisson_skip', 'kdv', 'wave3d'])
def test_fits_without_the_cluster_kernel_stay_stepwise(name):
    """ a residual layout, order 3 and cfg5's 64-wide network: no cluster kernel; the auto rule passes silently, an
    explicit steps_per_launch warns """
    s = make_solver(name)
    assert int(s._get_engine().info.small_batch_points) == 0
    with warnings.catch_warnings():
        warnings.simplefilter('error', UserWarning)
        s.fit(16, 64, optimizer='LBFGS', lr=0.05, max_iter=3)
    with pytest.warns(UserWarning, match='steps_per_launch ignored'):
        s.fit(2, 64, optimizer=None, steps_per_launch=2)
    assert len(s.losses) == 18 and np.isfinite(s.losses).all()


def test_bad_arguments_are_refused():
    s = make_solver('poisson2d')
    eng = s._get_engine()
    lib, dev = eng.lib, eng.device
    flat = s.flat_params().cuda().contiguous()
    mask = torch.ones(eng.n_params, device=dev)
    state = torch.zeros(lib.pinn_lbfgs_state_bytes(eng.n_params, 4), dtype=torch.uint8, device=dev)
    counter = torch.zeros(1, dtype=torch.int64, device=dev)
    ring = torch.zeros(8, device=dev)

    def cfg(**over):
        c = dict(lr=1.0, tolerance_grad=1e-7, tolerance_change=1e-9, max_iter=5, max_eval=6, history_size=4,
                 line_search=0, mask=mask.data_ptr(), losses_ring=ring.data_ptr(), ring_len=8,
                 step_counter=counter.data_ptr())
        c.update(over)
        return N.PinnLbfgs(**c)

    def solo(c, params=flat.data_ptr(), st=state.data_ptr(), n=100, k=1):
        return lib.pinn_lbfgs_multi(eng.plan, C.byref(c), C.c_void_p(params), C.c_void_p(st), None, None, C.c_uint64(1),
                                    C.c_int64(n), C.c_int(k), C.c_float(0.01), C.c_int(0), None, eng._stream())
    for bad in (dict(lr=-1.0), dict(lr=float('nan')), dict(max_iter=0), dict(max_eval=0), dict(history_size=0),
                dict(line_search=2), dict(ring_len=0), dict(mask=None), dict(losses_ring=None), dict(step_counter=None)):
        assert solo(cfg(**bad)) == N.E_INVALID, bad
    assert solo(cfg(), params=0) == N.E_INVALID
    assert solo(cfg(), st=0) == N.E_INVALID
    assert solo(cfg(), params=flat.data_ptr() + 4) == N.E_INVALID
    assert solo(cfg(), n=0) == N.E_INVALID and solo(cfg(), n=1025) == N.E_INVALID and solo(cfg(), k=0) == N.E_INVALID
    assert lib.pinn_lbfgs_multi(eng.plan, None, C.c_void_p(flat.data_ptr()), C.c_void_p(state.data_ptr()), None, None,
                                C.c_uint64(1), C.c_int64(100), C.c_int(1), C.c_float(0.01), C.c_int(0), None,
                                eng._stream()) == N.E_INVALID
    m = (N.PinnLbfgsMember * 1)()
    m[0].params, m[0].state, m[0].mask = flat.data_ptr(), state.data_ptr(), mask.data_ptr()
    m[0].step_counter, m[0].losses_ring, m[0].lr = counter.data_ptr(), ring.data_ptr(), 1.0

    def ens(n_members, members=m, c=None):
        return lib.pinn_lbfgs_multi_ensemble(eng.plan, C.byref(c or cfg()), n_members, members, None, C.c_int64(100),
                                             C.c_int(1), C.c_float(0.01), C.c_int(0), None, eng._stream())
    assert ens(0) == N.E_INVALID and ens(129) == N.E_INVALID and ens(1, None) == N.E_INVALID
    m[0].lr = -1.0
    assert ens(1) == N.E_INVALID
    torch.cuda.synchronize()
    assert int(counter) == 0 and torch.equal(flat, s.flat_params().cuda())      # nothing ran
    wide = make_solver('wave3d')._get_engine()
    assert lib.pinn_lbfgs_multi(wide.plan, C.byref(cfg()), C.c_void_p(flat.data_ptr()), C.c_void_p(state.data_ptr()),
                                None, None, C.c_uint64(1), C.c_int64(100), C.c_int(1), C.c_float(0.01), C.c_int(0), None,
                                wide._stream()) == N.E_UNSUPPORTED
