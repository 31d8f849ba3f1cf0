""" The persistent multi-step kernels (pinn_multi_step) against the fp64 oracle, at every cluster size and batch edge.

Fits with a batch of at most 1 024 points, plain Adam, one device and no constraint term run in one of two kernels:
small_step_kernel (pinn_small_kernel.cuh: batches of up to 256 points, or up to 1 024 when the other kernel does not fit;
a cluster of 1, 2, 4 or 8 CTAs, each taking a contiguous slice of the batch, the gradient partials summed over
distributed shared memory in rank order) and multi_step_kernel (pinn_step_kernel.cuh: one CTA, any batch up to 4 096).
Loss curves cannot tell a wrong gradient scale from a right one: Adam's update m^/(sqrt(v^)+eps) does not change when a
whole tensor's gradient is scaled.  So the tests here read each kernel's own reduced gradient: from a zero Adam state,
one step leaves exp_avg = fmaf(1 - beta1, g, 0), and g = exp_avg / float32(1 - beta1) to within one rounding.

Which kernel runs is not observable through the ABI; _kernel_for restates the selection rule of pinn_multi_step, and the
tests check its preconditions from the plan (pinn_plan_info.small_batch_points, pinn_multi_step_max_points).  All batch
sizes of a problem are prefixes of one 4 096-point batch: the oracle runs once per problem and is cut at every prefix. """
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

import problems as P
import problems_systems as PS
from helpers import rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    from gpu_helpers import Replay
    from oracle import adam as oracle_adam
    from oracle import autograd_port as ap
    from pydens_b200 import Solver, D, V
    from pydens_b200 import _native as N


def _heat_two_params(f, x, y, t, a, b, D, V):
    return D(D(f, x), x) + D(D(f, y), y) - a * D(f, t) + 0.1 * b * f


# five point columns: the in-kernel sampler draws a second Philox block for columns 4.. (and the oracle checks them)
SYNTHETIC = {
    'heat_two_params': dict(equation=_heat_two_params, ndims=3, nparams=2, ic=P._ic_heat, bc=0, domain=(0, 1),
                            features=[12, 10, 1], activation='Tanh', layout='fafaf',
                            ranges=[(0, 1), (0, 1), (0, .5), (.1, 4), (-1, 1)]),
}
ORDER2 = [n for n in P.PROBLEMS if n not in P.HI_DIRECTION and n not in P.HI_ORDER]
NO_PERSISTENT = list(P.HI_DIRECTION) + list(P.HI_ORDER) + ['kdv_two_residuals']     # five / six directions, orders 3 / 4
NAMES = ORDER2 + [n for n in PS.PROBLEMS if n not in NO_PERSISTENT] + list(SYNTHETIC)


def _cfg(name):
    for reg in (P.PROBLEMS, PS.PROBLEMS, SYNTHETIC):
        if name in reg:
            return reg[name]
    raise KeyError(name)


def _has_skips(name):
    return 'R' in _cfg(name)['layout']


def _wide(name):
    return max(_cfg(name)['features']) >= 64


# the small kernel takes dense chains without residual wiring whose jets of 128 points fit shared memory (not the 30- and
# 40-wide layers of heat2d / heat_param with six jet channels: test_small_kernel_is_placed_where_its_layout_fits); the
# multi kernel every network narrower than 64 (its staged weights and per-warp state of cfg5's network do not fit)
TOO_BIG_FOR_SMALL = ('heat2d', 'heat_param')
SMALL_NAMES = [n for n in NAMES if not _has_skips(n) and not _wide(n) and n not in TOO_BIG_FOR_SMALL]
MULTI_NAMES = [n for n in NAMES if not _wide(n)]

SMALL_SIZES = [1, 2, 15, 16, 17, 32, 33, 48, 49, 64, 65, 100, 127, 128, 129, 255, 256]
FORCED_SIZES = [1, 3, 7, 128, 129, 200, 256]
MULTI_SIZES = [1, 31, 32, 33, 257, 1000, 1024]
ABI_SIZES = [2047, 4096]
ORACLE_N = 4096
MODES = {'small': {}, 'small_c1': {'PINN_SMALL_CLUSTER': '1'}, 'small_c2': {'PINN_SMALL_CLUSTER': '2'},
         'small_c4': {'PINN_SMALL_CLUSTER': '4'}, 'small_c8': {'PINN_SMALL_CLUSTER': '8'},
         'multi': {'PINN_MULTI_KERNEL': 'tile'}}
LR = 0.01
BETA1, BETA2 = 0.9, 0.999


def _ic(name, V_):
    cfg = _cfg(name)
    return cfg['ic_factory'](V_) if 'ic_factory' in cfg else cfg['ic']


def _solver(name):
    cfg = _cfg(name)
    torch.manual_seed(0)
    eq = cfg['equation']
    pkg_V = lambda n, init: V(n, data=torch.Tensor([init]))
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)           # systems: the [N, m] vs [N, 1] broadcast of the trial run
        solver = Solver(lambda u, *xs: eq(u, *xs, D=D, V=pkg_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                        initial_condition=_ic(name, pkg_V), boundary_condition=cfg['bc'], domain=cfg['domain'],
                        layout=cfg['layout'], features=cfg['features'], activation=cfg['activation'],
                        device='cuda', backend='fused', seed=1234)
        solver._get_engine()
    if 'log_scale' in cfg:
        with torch.no_grad():
            solver.model.log_scale.fill_(cfg['log_scale'])
    return solver


def _oracle(name, params):
    cfg = _cfg(name)
    holder = {}
    ic = _ic(name, lambda n, init: holder['prob'].V(n, init))
    prob = ap.Problem(lambda u, *xs, D, V: cfg['equation'](u, *xs, D=D, V=V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                      initial_condition=ic, boundary_condition=cfg['bc'], domain=cfg['domain'], features=cfg['features'],
                      activation=cfg['activation'], dtype=torch.float64, variables=cfg.get('variables'),
                      layout=cfg['layout'])
    holder['prob'] = prob
    prob.load_flat(torch.as_tensor(params, dtype=torch.float64))
    return prob


def _points(name, n, seed):
    rng = np.random.RandomState(seed)
    return np.concatenate([rng.uniform(lo, hi, size=(n, 1)) for lo, hi in _cfg(name)['ranges']], axis=1).astype(np.float32)


def _oracle_loss_and_grads(prob, name, pts, criterion=None):
    """ fp64 oracle on one batch -> (loss, folded residual [n], grads) """
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        l, r, g = prob.loss_and_grads(np.asarray(pts, dtype=np.float64), criterion=criterion)
    cfg = _cfg(name)
    return l, (PS.folded_residual(r, cfg['m']) if 'm' in cfg else r), g.numpy()


_ORACLE = {}


def _oracle_prefixes(name, params, cuts, criterion=None, crit_key=None):
    """ fp64 oracle on prefixes of one batch: {n: (loss, residual [n], grads)}, segment by segment between the cuts (the
    loss and the gradients are means over the points: their sums add over segments).  Kept per problem and parameters. """
    key = (name, crit_key, hash(np.asarray(params, dtype=np.float32).tobytes()), tuple(cuts))
    if key in _ORACLE:
        return _ORACLE[key]
    pts = _points(name, max(cuts), seed=2024)
    prob = _oracle(name, np.asarray(params, dtype=np.float64))
    bounds = sorted(set([0] + list(cuts)))
    sums, res = {}, []
    l_acc, g_acc = 0.0, None
    for a, b in zip(bounds[:-1], bounds[1:]):
        l, r, g = _oracle_loss_and_grads(prob, name, pts[a:b], criterion)
        l_acc += l * (b - a)
        g_acc = g * (b - a) if g_acc is None else g_acc + g * (b - a)
        res.append(r)
        sums[b] = (l_acc / b, np.concatenate(res), g_acc / b)
    _ORACLE[key] = (pts, sums)
    return _ORACLE[key]


def _tensors(name, eng):
    """ (name, slice) of every weight and bias tensor, log_scale and the equation variables in the flat layout """
    s = eng.spec
    out = []
    for l in range(s.n_layers):
        out.append(('W%d' % l, slice(s.w_off[l], s.w_off[l] + s.widths[l] * s.widths[l + 1])))
        out.append(('b%d' % l, slice(s.b_off[l], s.b_off[l] + s.widths[l + 1])))
    end = s.b_off[s.n_layers - 1] + s.widths[s.n_layers]
    n_scalars = 1 + len(_cfg(name).get('variables') or {})
    out += [('log_scale' if i == 0 else 'V%d' % i, slice(end + i, end + i + 1)) for i in range(n_scalars)]
    return out


def _check_against_oracle(name, eng, loss, grads, ref, tag):
    """ the tolerances of test_gpu_placement.py::test_placement_matches_fp64_oracle (cancellation factor of
    test_gpu_fuzz.py) """
    ref_loss, ref_res, ref_g = ref
    cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(ref_res)))), 1e-30))
    assert np.isfinite(grads).all() and np.isfinite(loss), tag
    assert abs(loss - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), '%s: loss %.9g, oracle %.9g' % (tag, loss, ref_loss)
    assert rel_l2(grads[:ref_g.size], ref_g) <= 1e-4 * cond, tag
    scale = 1e-3 * np.linalg.norm(ref_g)           # a tensor whose gradient is 1000x below the whole is held to that
    for tname, sl in _tensors(name, eng):
        err = np.linalg.norm(grads[sl] - ref_g[sl]) / max(np.linalg.norm(ref_g[sl]), scale, 1e-30)
        # log_scale and V_i are single sums over the points, which can cancel at a handful of points: mixed_ic's
        # d/dlog_scale is -8.1e-3 at 3 points and -2.2e-5 at 7, where the kernel lands 1.3e-4 - 1.5e-4 (relative to
        # the 1e-3 * |g| floor) off the oracle on every cluster size.  So the scalars get 3x.
        tol = (3e-4 if tname == 'log_scale' or tname.startswith('V') else 1e-4) * cond
        assert err <= tol, '%s: %s rel err %.2e' % (tag, tname, err)


# ---- which kernel pinn_multi_step launches (pinn_kernels.cu, restated) ---------------------------------------------------
def _has_small(eng):
    return int(eng.info.small_batch_points) > 0


def _has_multi(eng):
    return int(eng.lib.pinn_multi_step_max_points(eng.plan)) == 4096


def _kernel_for(eng, n, env):
    """ -> ('small', cluster size) or ('multi', 1) for a batch of n points under the environment `env` """
    small_ok = (_has_small(eng) and n <= 1024 and (n <= 256 or not _has_multi(eng))
                and not (env.get('PINN_MULTI_KERNEL') == 'tile' and _has_multi(eng)))
    if not small_ok:
        return 'multi', 1
    nc = min(8, (n + 15) // 16)
    forced = int(env.get('PINN_SMALL_CLUSTER', '0'))
    if 1 <= forced <= 8:
        nc = forced
    while (n + nc - 1) // nc > 128:
        nc += 1
    nc = 4 if nc == 3 else (8 if 4 < nc < 8 else nc)
    return 'small', nc


def _preconditions(name, eng, kernel):
    if kernel == 'small':
        assert int(eng.info.small_batch_points) == 1024, '%s: no small_step_kernel' % name
    else:
        assert int(eng.lib.pinn_multi_step_max_points(eng.plan)) == 4096, '%s: no multi_step_kernel' % name


# ---- the public path: Solver.fit, one step from a zero Adam state -------------------------------------------------------
def _fit_one_step(solver, params, pts, criterion=None):
    """ one persistent step on `pts` from `params` and a zero Adam state -> (engine, loss, g, exp_avg, exp_avg_sq) """
    solver.load_flat_params(params)
    kw = {} if criterion is None else dict(criterion=criterion)
    with warnings.catch_warnings():
        warnings.filterwarnings('error', message='.*steps_per_launch')          # the persistent path must take it
        solver.fit(niters=1, batch_size=pts.shape[0], sampler=Replay([pts]), lr=LR, steps_per_launch=1, **kw)
    eng = solver._engine
    m, v = eng._adam_flat[0].cpu().numpy(), eng._adam_flat[1].cpu().numpy()
    g = m / (np.float32(1.0) - np.float32(BETA1))
    return eng, float(solver.losses[-1]), g, m, v


def _check_second_moment(g, v, tag):
    """ exp_avg_sq of the first step is (1 - beta2) g^2, from the gradient that exp_avg holds """
    want = (np.float32(1.0) - np.float32(BETA2)) * g * g
    err = np.abs(v - want)
    assert (err <= 1e-5 * want + 1e-38).all(), '%s: exp_avg_sq off (1 - beta2) g^2 by up to %.2e' % (
        tag, float((err / np.maximum(want, 1e-30)).max()))


def _all_cuts():
    return sorted(set(SMALL_SIZES + FORCED_SIZES + MULTI_SIZES + ABI_SIZES + [ORACLE_N]))


@pytest.mark.parametrize('name,mode', [(n, m) for m in MODES for n in (MULTI_NAMES if m == 'multi' else SMALL_NAMES)])
def test_persistent_gradient_matches_fp64_oracle(name, mode, monkeypatch):
    kernel = 'multi' if mode == 'multi' else 'small'
    env = MODES[mode]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    solver = _solver(name)
    eng = solver._get_engine()
    _preconditions(name, eng, kernel)
    params = solver.flat_params().cpu().numpy()
    pts, ref = _oracle_prefixes(name, params, _all_cuts())
    sizes = {'small': SMALL_SIZES, 'multi': MULTI_SIZES}.get(mode, FORCED_SIZES)
    for n in sizes:
        which, nc = _kernel_for(eng, n, env)
        assert which == kernel, '%s n=%d: would run %s' % (name, n, which)
        tag = '%s %s n=%d (%s kernel, %d CTAs)' % (name, mode, n, which, nc)
        eng, loss, g, m, v = _fit_one_step(solver, params, pts[:n])
        _check_against_oracle(name, eng, loss, g, ref[n], tag)
        _check_second_moment(g, v, tag)
        if kernel == 'multi' and n >= 257:
            # the default selection sends 257..1024 points to the same kernel: the same bits
            monkeypatch.delenv('PINN_MULTI_KERNEL')
            assert _kernel_for(eng, n, {}) == ('multi', 1)
            _, loss_d, _, m_d, v_d = _fit_one_step(solver, params, pts[:n])
            assert loss_d == loss and np.array_equal(m_d, m) and np.array_equal(v_d, v), tag
            monkeypatch.setenv('PINN_MULTI_KERNEL', 'tile')
    if kernel == 'multi':
        # beyond what fit sends here: the C ABI takes up to 4 096 points
        for n in ABI_SIZES:
            st = _State.fresh(eng, params)
            pts_d = torch.from_numpy(pts[:n]).cuda().reshape(1, n, -1).contiguous()
            N.check(_multi_step(eng, st, pts_d, n, 1))
            torch.cuda.synchronize()
            m = st.m.cpu().numpy()
            g = m / (np.float32(1.0) - np.float32(BETA1))
            tag = '%s C ABI n=%d' % (name, n)
            _check_against_oracle(name, eng, float(st.ring[0]), g, ref[n], tag)
            _check_second_moment(g, st.v.cpu().numpy(), tag)


def _small_smem_bytes(eng):
    """ small_step_kernel's dynamic shared memory (pinn_small_kernel.cuh make_layout) """
    s, ch, sr = eng.spec, int(eng.info.channels), 128 + 4
    np4 = (eng.n_params + 3) & ~3
    floats = 3 * np4 + 3 * (np4 + 4) + (N.MAX_DIMS + s.n_slots + 2 + N.MAX_VARS) * sr
    for l in range(s.n_layers):
        floats += s.widths[l + 1] * ch * sr * (2 if l + 1 < s.n_layers else 1)
    return 4 * floats


def test_small_kernel_is_placed_where_its_layout_fits():
    """ the small kernel exists for the dense chains whose layout fits shared memory, and never for residual wiring """
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    for name in NAMES:
        eng = _solver(name)._get_engine()
        has = _has_small(eng)
        if _has_skips(name):
            assert not has and _has_multi(eng), name
            continue
        need = _small_smem_bytes(eng)
        if need <= optin - 2048:                 # the kernel's static shared memory and the 64-byte margin fit in 2 KB
            assert has and name in SMALL_NAMES, '%s: %d bytes' % (name, need)
        elif need > optin:
            assert not has and name not in SMALL_NAMES, '%s: %d bytes' % (name, need)
        assert _has_multi(eng) == (name in MULTI_NAMES), name


# five / six directions and orders 3 / 4 have no persistent kernel; neither has the 64-wide network of cfg5
@pytest.mark.parametrize('name', NO_PERSISTENT + [n for n in NAMES if _wide(n)])
def test_problems_without_a_persistent_kernel_warn(name):
    solver = _solver(name)
    eng = solver._get_engine()
    assert int(eng.lib.pinn_multi_step_max_points(eng.plan)) == 0
    assert int(eng.info.small_batch_points) == 0
    pts = _points(name, 64, seed=3)
    with pytest.warns(UserWarning, match='steps_per_launch ignored'):
        solver.fit(niters=1, batch_size=64, sampler=Replay([pts]), lr=LR, steps_per_launch=1)
    assert len(solver.losses) == 1 and np.isfinite(solver.losses[-1])


@pytest.mark.parametrize('mode', ['small', 'multi'])
def test_huber_criterion_gradient_matches_fp64_oracle(mode, monkeypatch):
    """ HuberLoss (mean) trains on the persistent kernels too (the residual transform of tracer.apply_criterion) """
    name = 'burgers'
    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    solver = _solver(name)
    params = solver.flat_params().cpu().numpy()
    crit = torch.nn.HuberLoss(delta=0.05)
    pts, ref = _oracle_prefixes(name, params, _all_cuts(), criterion=crit, crit_key='huber0.05')
    for n in ([1, 17, 100, 256] if mode == 'small' else [1, 33, 257, 1024]):
        eng, loss, g, m, v = _fit_one_step(solver, params, pts[:n], criterion=torch.nn.HuberLoss(delta=0.05))
        assert solver._crit_key != ('mse',)
        _preconditions(name, eng, mode)
        assert _kernel_for(eng, n, MODES[mode])[0] == mode
        tag = '%s huber %s n=%d' % (name, mode, n)
        _check_against_oracle(name, eng, loss, g, ref[n], tag)
        _check_second_moment(g, v, tag)


# ---- the bare C ABI ---------------------------------------------------------------------------------------------------
class _State:
    """ Everything pinn_multi_step reads and writes, on the device """

    def __init__(self, p, m, v, mask, steps, counter, ring):
        self.p, self.m, self.v, self.mask, self.steps, self.counter, self.ring = p, m, v, mask, steps, counter, ring

    @classmethod
    def fresh(cls, eng, params, ring_len=1, step0=0):
        dev = eng.device
        z = torch.zeros(eng.n_params, dtype=torch.float32, device=dev)
        return cls(torch.as_tensor(params, dtype=torch.float32).to(dev).clone(), z.clone(), z.clone(),
                   torch.ones(eng.n_params, dtype=torch.float32, device=dev),
                   torch.zeros(len(eng.entries), dtype=torch.float32, device=dev),
                   torch.full((1,), step0, dtype=torch.int64, device=dev),
                   torch.zeros(ring_len, dtype=torch.float32, device=dev))

    def clone(self):
        return _State(*(t.clone() for t in (self.p, self.m, self.v, self.mask, self.steps, self.counter, self.ring)))


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _multi_step(eng, st, points, n, k, cols=None, lr=LR, betas=(BETA1, BETA2), eps=1e-8, weight_decay=0.0, opt_step0=0.0):
    """ pinn_multi_step on the engine's plan -> its return code.  `points`: [k, n, total] on the device, or None (the
    in-kernel sampler draws columns `cols`). """
    return eng.lib.pinn_multi_step(
        eng.plan, _ptr(st.p), _ptr(st.m), _ptr(st.v), _ptr(st.mask), _ptr(st.steps), C.c_int(st.steps.numel()),
        _ptr(points), N.make_columns(cols, eng.solver.model.total), C.c_uint64(eng.seed), _ptr(st.counter),
        C.c_int64(n), C.c_int(k), C.c_float(lr), C.c_float(betas[0]), C.c_float(betas[1]), C.c_float(eps),
        C.c_float(weight_decay), C.c_float(opt_step0), _ptr(st.ring), C.c_int64(st.ring.numel()), eng._stream())


ADAM = dict(lr=3e-3, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.01)
STEP0, OPT_STEP0 = 1000, 37


@pytest.mark.parametrize('kernel,n', [('small', 100), ('multi', 700)])
def test_adam_ring_and_counters_follow_the_oracle(kernel, n):
    """ Five steps from a used Adam state (random moments, 37 steps taken, non-default lr / betas / eps, weight decay
    0.01, log_scale and the first bias frozen) on explicit batches, ring of three losses.  Each step, launched alone,
    against oracle/adam.py applied to the fp64 oracle gradient of its batch at the kernel's parameters; the five steps in
    one launch give the same bits.  Tolerances: loss 2e-5 * cond, exp_avg and exp_avg_sq 1e-5 * cond (relative L2), the
    parameter update 1e-4 * cond (relative L2 of new - old against the oracle's).  Measured on an H100 80GB HBM3, over
    the five steps of either kernel: loss <= 2.5e-7, exp_avg <= 9.3e-8, exp_avg_sq <= 6.5e-8, update <= 1.0e-6 (cond 1):
    the tolerances are 100x the fp32 noise floor, and a gradient off by a tensor-wide factor moves exp_avg by that
    factor. """
    name = 'heat1d_icvar'                        # variables in the equation and in the initial condition, log_scale
    solver = _solver(name)
    eng = solver._get_engine()
    _preconditions(name, eng, kernel)
    assert _kernel_for(eng, n, {})[0] == kernel
    params = solver.flat_params().cpu().numpy()
    prob = _oracle(name, params.astype(np.float64))
    k = 5
    batches = [_points(name, n, seed=70 + s) for s in range(k)]
    rng = np.random.RandomState(5)
    _, _, g0 = _oracle_loss_and_grads(prob, name, batches[0])
    g0 = np.concatenate([g0, np.zeros(eng.n_params - g0.size)]).astype(np.float32)
    m0 = (np.abs(g0) * rng.randn(eng.n_params)).astype(np.float32)
    v0 = (g0 * g0 * rng.uniform(0.5, 2.0, eng.n_params) + 1e-12).astype(np.float32)
    mask = np.ones(eng.n_params, dtype=np.float32)
    names = dict(_tensors(name, eng))
    mask[names['log_scale']] = 0.0
    mask[names['b0']] = 0.0
    st0 = _State.fresh(eng, params, ring_len=3, step0=STEP0)
    st0.m.copy_(torch.from_numpy(m0)); st0.v.copy_(torch.from_numpy(v0)); st0.mask.copy_(torch.from_numpy(mask))
    st0.steps.fill_(float(OPT_STEP0))

    # each step alone, against the oracle
    st = st0.clone()
    losses, noise = [], []
    for s in range(k):
        p_prev, m_prev, v_prev = (t.cpu().numpy().copy() for t in (st.p, st.m, st.v))
        pts = torch.from_numpy(batches[s]).cuda().reshape(1, n, -1).contiguous()
        N.check(_multi_step(eng, st, pts, n, 1, opt_step0=float(OPT_STEP0 + s), **ADAM))
        torch.cuda.synchronize()
        loss = float(st.ring[(STEP0 + s) % 3])
        losses.append(loss)
        prob.load_flat(torch.as_tensor(p_prev, dtype=torch.float64))
        l64, r64, g64 = _oracle_loss_and_grads(prob, name, batches[s])
        cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(r64)))), 1e-30))
        g64 = np.concatenate([g64, np.zeros(eng.n_params - g64.size)]).astype(np.float32)
        p_o, m_o, v_o = oracle_adam.adam_step(p_prev.copy(), g64, m_prev.copy(), v_prev.copy(), OPT_STEP0 + s + 1,
                                              lr=ADAM['lr'], beta1=ADAM['betas'][0], beta2=ADAM['betas'][1],
                                              eps=ADAM['eps'], weight_decay=ADAM['weight_decay'], mask=mask)
        p_k, m_k, v_k = (t.cpu().numpy() for t in (st.p, st.m, st.v))
        errs = dict(loss=abs(loss - l64) / abs(l64), m=rel_l2(m_k, m_o), v=rel_l2(v_k, v_o),
                    update=rel_l2(p_k - p_prev, p_o - p_prev))
        noise.append(errs)
        tag = '%s %s step %d (cond %.1f): %s' % (kernel, name, s, cond, errs)
        assert errs['loss'] <= 2e-5 * cond, tag
        assert errs['m'] <= 1e-5 * cond and errs['v'] <= 1e-5 * cond, tag
        assert errs['update'] <= 1e-4 * cond, tag
        frozen = mask == 0
        for a, b in ((p_k, p_prev), (m_k, m_prev), (v_k, v_prev)):
            assert np.array_equal(a[frozen], b[frozen]), tag
        assert np.abs(p_k - p_prev)[~frozen].max() > 0, tag
    print('NOISE %s n=%d: %s' % (kernel, n, ' | '.join(
        ' '.join('%s %.1e' % kv for kv in e.items()) for e in noise)))
    assert torch.equal(st.steps, torch.full_like(st.steps, float(OPT_STEP0 + k)))
    assert int(st.counter) == STEP0 + k

    # all five in one launch: the same bits, the ring holds the last three losses at (step0 + s) % 3
    one = st0.clone()
    pts = torch.from_numpy(np.stack(batches)).cuda().contiguous()
    N.check(_multi_step(eng, one, pts, n, k, opt_step0=float(OPT_STEP0), **ADAM))
    torch.cuda.synchronize()
    assert torch.equal(one.p, st.p) and torch.equal(one.m, st.m) and torch.equal(one.v, st.v)
    ring = one.ring.cpu().numpy()
    for s in range(k - 3, k):
        assert ring[(STEP0 + s) % 3] == np.float32(losses[s]), s
    assert torch.equal(one.steps, torch.full_like(one.steps, float(OPT_STEP0 + k)))
    assert int(one.counter) == STEP0 + k
    frozen = torch.from_numpy(mask == 0).cuda()
    for a, b in ((one.p, st0.p), (one.m, st0.m), (one.v, st0.v)):
        assert torch.equal(a[frozen], b[frozen])

    # rejected arguments, and nothing written
    max_n = int(eng.lib.pinn_multi_step_max_points(eng.plan))
    bad = st0.clone()
    big = torch.zeros((1, max_n + 1, pts.shape[-1]), dtype=torch.float32, device='cuda')
    assert _multi_step(eng, bad, pts, 0, 1, **ADAM) == N.E_INVALID
    assert _multi_step(eng, bad, big, max_n + 1, 1, **ADAM) == N.E_INVALID
    assert _multi_step(eng, bad, pts, n, 0, **ADAM) == N.E_INVALID
    torch.cuda.synchronize()
    assert torch.equal(bad.p, st0.p) and torch.equal(bad.m, st0.m) and int(bad.counter) == STEP0


# ---- bit-level invariants -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kernel,n', [('small', 100), ('multi', 600)])
def test_one_launch_equals_many(kernel, n):
    """ six steps in one launch == six launches of one step == launches of 4 + 2 steps, through Solver.fit """
    name = 'heat1d_icvar'
    batches = [_points(name, n, seed=90 + s) for s in range(6)]
    runs = {}
    for k in (1, 6, 4):
        solver = _solver(name)
        eng = solver._get_engine()
        _preconditions(name, eng, kernel)
        assert _kernel_for(eng, n, {})[0] == kernel
        with warnings.catch_warnings():
            warnings.filterwarnings('error', message='.*steps_per_launch')
            solver.fit(niters=6, batch_size=n, sampler=Replay(list(batches)), lr=LR, steps_per_launch=k)
        runs[k] = (solver.flat_params().cpu(), eng._adam_flat[0].cpu(), eng._adam_flat[1].cpu(), np.asarray(solver.losses))
    for k in (6, 4):
        for a, b in zip(runs[1][:3], runs[k][:3]):
            assert torch.equal(a, b), 'steps_per_launch=%d' % k
        assert np.array_equal(runs[1][3], runs[k][3]), 'steps_per_launch=%d' % k
    assert len(runs[1][3]) == 6 and np.isfinite(runs[1][3]).all()


@pytest.mark.parametrize('kernel,n', [('small', 200), ('multi', 700)])
def test_in_kernel_sampling_equals_explicit_points(kernel, n):
    """ steps sampled in the kernel at step counter s, s+1, s+2 == the same steps on pinn_sample's batches.  Five columns
    (the second Philox block), uniform, normal, truncated-normal and mixture columns; a counter above 2^32 (the high
    counter word). """
    name = 'heat_two_params'
    solver = _solver(name)
    eng = solver._get_engine()
    _preconditions(name, eng, kernel)
    assert _kernel_for(eng, n, {})[0] == kernel
    cols = [(N.COL_UNIFORM, 0.0, 1.0), (N.COL_NORMAL, 0.5, 0.2), (N.COL_TNORMAL, 0.2, 0.3, 0.0, 0.5),
            ('mix', 'a', [(1.0, N.COL_UNIFORM, 0.1, 1.0), (2.0, N.COL_UNIFORM, 2.0, 4.0)]), (N.COL_UNIFORM, -1.0, 1.0)]
    s0, k = (5 << 32) | 77, 3
    st0 = _State.fresh(eng, solver.flat_params().cpu().numpy(), ring_len=4, step0=s0)
    sampled = st0.clone()
    N.check(_multi_step(eng, sampled, None, n, k, cols=cols))
    pts = torch.stack([eng.sample(n, cols, step=s0 + s) for s in range(k)]).contiguous()
    explicit = st0.clone()
    N.check(_multi_step(eng, explicit, pts, n, k))
    torch.cuda.synchronize()
    assert torch.isfinite(sampled.p).all() and not torch.equal(sampled.p, st0.p)
    for a, b in zip((sampled.p, sampled.m, sampled.v, sampled.ring, sampled.counter),
                    (explicit.p, explicit.m, explicit.v, explicit.ring, explicit.counter)):
        assert torch.equal(a, b)
    # and the columns are what was asked for
    p = pts.cpu().numpy().reshape(-1, 5)
    assert p[:, 0].min() >= 0 and p[:, 0].max() < 1 and p[:, 2].min() >= 0 and p[:, 2].max() <= 0.5
    assert ((p[:, 3] < 1) | (p[:, 3] >= 2)).all() and p[:, 4].min() >= -1 and p[:, 4].max() < 1


@pytest.mark.parametrize('kernel,n,env', [('small', 256, {'PINN_SMALL_CLUSTER': '8'}), ('multi', 1024, {})])
def test_run_to_run_bits(kernel, n, env, monkeypatch):
    """ small_step_kernel on eight CTAs (rank-order sum over distributed shared memory) and multi_step_kernel on 1 024
    points: four steps from the same state give the same bits every time """
    for key, val in env.items():
        monkeypatch.setenv(key, val)
    name = 'heat1d_icvar'
    solver = _solver(name)
    eng = solver._get_engine()
    _preconditions(name, eng, kernel)
    assert _kernel_for(eng, n, env) == ((kernel, 8) if kernel == 'small' else (kernel, 1))
    st0 = _State.fresh(eng, solver.flat_params().cpu().numpy(), ring_len=4, step0=11)
    runs = []
    for _ in range(3):
        st = st0.clone()
        N.check(_multi_step(eng, st, None, n, 4))
        torch.cuda.synchronize()
        runs.append(st)
    for st in runs[1:]:
        for a, b in zip((st.p, st.m, st.v, st.ring), (runs[0].p, runs[0].m, runs[0].v, runs[0].ring)):
            assert torch.equal(a, b)
