""" The grid tail every step kernel shares (finish_grid in pydens_b200/csrc/pinn_step_kernel.cuh): the two-level fold of
the CTA partials (groups of FOLD_GROUP = 12 CTAs, then the group results, tickets reset at the end of each launch) and
the in-kernel Adam (adam_hyper / adam_apply), which is optimizer.step() of every stepwise fit.

a. pinn_step_adam = pinn_step + Adam, element by element, on every kernel family: step_kernel at every placement of
   test_gpu_placement.py on two networks (between them, the per-warp gradient accumulators are in shared memory and in
   the workspace), coupled_step_kernel (k = 2, 3, 4), wide_step_kernel, wide128_step_kernel and its coupled form, and
   hi_step_kernel at orders 3 and 4.  Four steps on one Adam state (random moments, about 1/7 of the entries frozen,
   log_scale and the first bias among them, weight decay 0.01, betas (0.85, 0.995), eps 1e-7, a ring of three losses):
   `out` is bit-equal to pinn_step's (the same kernel, the same fixed-order fold), the moments follow oracle/adam.py
   per element, the parameters follow Adam's update of the kernel's own moments per element, frozen entries keep their
   bits, every step tensor and the step counter advance by one, and the ring holds the loss bits.
b. Adam state edges: t = 1 and t = 2 (an off-by-one in t moves the update by tens of percent there), t = 10^6 + 1
   (beta^t underflows), beta1 = 0, beta2 = 0.9999, eps large (1e-3) and eps small (1e-12) from v = 0; and t = 1, 2 on
   the persistent kernels (small and multi), which have their own Adam code.
c. Fold-group edges against the fp64 oracle at the bars of the placement tests: grids of G = 1, 2, 11, 12, 13, 24, 25,
   sm_count - 1 and sm_count CTAs and one point past each, on the thread kernel (one warp per CTA), the 64-wide tile
   kernel (PINN_WIDE_CTAS) and the whole-jet kernel; at G = 13 and 25 (a last group of one CTA) also check (a).
d. One workspace through grids of 13, 5, 25, 1, sm_count and 13 CTAs gives the bits of a fresh workspace every time:
   every ticket is reset at the end of every fold shape.
e. Through Solver.fit: weight decay with the in-kernel Adam against torch's fused Adam on every family;
   Adam(decoupled_weight_decay=True) against AdamW on the stepwise and the persistent route and in fit_ensemble; an
   optimizer state whose step counts differ per tensor against torch's Adam.

Per-element bars, u = 2^-24, g' = g + wd * p0 (the kernel forms it with an fma, numpy with two roundings, so the
bars take |g| + |wd * p0| rather than |g'|):
    m:  |m_k - m_o| <= 8u (|m0| + (1 - b1) (|g| + |wd p0| + |m0|))
    v:  |v_k - v_o| <= 12u (|v0| + (1 - b2) (|g| + |wd p0|)^2)
    p:  |p_k - p_e| <= 2^-23 |p0| + c_t |p_e - p0|,   c_t = 16u (1 + b1^t / (1 - b1^t) + b2^t / (2 (1 - b2^t)))
where m_o, v_o are oracle/adam.py's moments from the kernel's own gradient (out), and p_e is Adam's update of p0
computed in fp32 from the kernel's m_k and v_k: the parameter bar checks the update itself (step size, bias
corrections, eps) without charging it for the moments' last bits, which the m and v bars already hold, and which a
moment that cancels to near zero would otherwise magnify without bound.  The m and v bars are the first-order sums
of both sides' rounding errors (numpy rounds g + wd * p0, g' - m0, the product and the sum one by one, the kernel
fuses two of them), so they hold for every element, not only for typical ones.  The oracle gets the hyper-parameters
rounded to fp32, as the kernels receive them through the C ABI (1 - b2 is then exact). """
import warnings

import numpy as np
import pytest
import torch

import test_gpu_coupled_placement as TCP
import test_gpu_hi as TH
import test_gpu_persistent as TPer
import test_gpu_placement as TP
import test_gpu_tile as TG
import test_gpu_tile128 as TG128
from helpers import rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    from gpu_helpers import make_solver
    from oracle import adam as oracle_adam
    from pydens_b200 import fit_ensemble, _native as N
    import problems_wide_coupled as PWC
    import test_gpu_coupled as TGC
    import test_gpu_tile128_coupled as TG128C
    from helpers import load_golden

U = 2.0 ** -24
HYPER = dict(lr=0.003, beta1=0.85, beta2=0.995, eps=1e-7, weight_decay=0.01)
RING = 3


# ---- launching pinn_step / pinn_step_adam on any plan ---------------------------------------------------------------
def _launcher(lib, plan, spec):
    """ test_gpu_tile._Plan's launches (step) on a plan made elsewhere (an engine's, the coupled tests'); the plan
    stays owned by its maker """
    p = object.__new__(TG._Plan)
    p.lib, p.plan, p.spec, p.dev, p.ws = lib, plan, spec, torch.device('cuda:0'), None
    return p


def _state(spec, params, rng, step0=0.0, n_steps=5, v0=None):
    """ test_gpu_tile128._AdamState with log_scale and the first bias frozen too, `n_steps` step tensors at `step0`
    and a ring of RING losses """
    st = TG128._AdamState(spec.n_params, np.asarray(params, dtype=np.float32), rng)
    st.mask[spec.log_scale_off] = 0.0
    st.mask[spec.b_off[0]:spec.b_off[0] + spec.widths[1]] = 0.0
    st.steps = torch.full((n_steps,), float(step0), dtype=torch.float32, device=st.p.device)
    st.ring = torch.zeros(RING, dtype=torch.float32, device=st.p.device)
    if v0 is not None:
        st.v.fill_(v0)
    return st


def _f32(h):
    return {k: float(np.float32(v)) for k, v in h.items()}


def update_bar(h, t, p0, m_k, v_k):
    """ -> (p_e, the p bar of the module docstring): Adam's update of p0 from the moments m_k, v_k in fp32, as
    oracle/adam.py computes it, and the bar around it; `h` holds fp32-rounded hyper-parameters """
    f = np.float32
    step_size = f(h['lr']) / f(1.0 - np.power(f(h['beta1']), f(t)))
    bc2 = np.sqrt(f(1.0 - np.power(f(h['beta2']), f(t))), dtype=np.float32)
    p_e = p0 - step_size * m_k / (np.sqrt(v_k) / bc2 + f(h['eps']))
    b1t, b2t = h['beta1'] ** float(t), h['beta2'] ** float(t)
    c_t = 16 * U * (1 + b1t / (1 - b1t) + b2t / (2 * (1 - b2t)))
    return p_e, 2.0 ** -23 * np.abs(p0.astype(np.float64)) + c_t * np.abs(p_e.astype(np.float64) - p0)


def check_adam_elements(tag, h, t, p0, m0, v0, g, mask, got):
    """ the per-element bars of the module docstring -> the largest error / bar of p, m and v """
    h = _f32(h)
    b1, b2, wd = h['beta1'], h['beta2'], h['weight_decay']
    p_k, m_k, v_k = got
    on = mask != 0
    assert np.isfinite(p_k).all() and np.isfinite(m_k).all() and np.isfinite(v_k).all(), tag
    for a, b, what in ((p_k, p0, 'p'), (m_k, m0, 'exp_avg'), (v_k, v0, 'exp_avg_sq')):
        assert np.array_equal(a[~on].view(np.int32), b[~on].view(np.int32)), '%s: frozen %s changed' % (tag, what)
    _, m_o, v_o = oracle_adam.adam_step(p0.copy(), g, m0.copy(), v0.copy(), t, lr=h['lr'], beta1=b1, beta2=b2,
                                        eps=h['eps'], weight_decay=wd, mask=mask)
    d = np.float64
    ga = np.abs(g.astype(d)) + np.abs(wd * p0.astype(d))
    bar_m = 8 * U * (np.abs(m0.astype(d)) + (1 - b1) * (ga + np.abs(m0.astype(d))))
    bar_v = 12 * U * (np.abs(v0.astype(d)) + (1 - b2) * ga * ga)
    p_e, bar_p = update_bar(h, t, p0, m_k, v_k)
    worst = {}
    for what, k, o, bar in (('p', p_k, p_e, bar_p), ('m', m_k, m_o, bar_m), ('v', v_k, v_o, bar_v)):
        err = np.abs(k[on].astype(d) - o[on].astype(d))
        ratio = np.where(err == 0, 0.0, err / np.maximum(bar[on], 1e-300))
        i = int(np.argmax(ratio))
        worst[what] = float(ratio[i])
        assert ratio[i] <= 1.0, '%s: %s off by %.3e at entry %d (bar %.3e, error / bar %.2f)' % (
            tag, what, err[i], np.flatnonzero(on)[i], bar[on][i], ratio[i])
    return worst


def adam_steps(tag, p, params, points, rng, h=HYPER, step0=0.0, k=4, v0=None):
    """ k steps of pinn_step_adam on one Adam state, each against pinn_step on the same parameters and points followed
    by the per-element bars; `points(s)` -> the device batch of step s.  -> the worst error / bar per tensor """
    spec = p.spec
    st = _state(spec, params, rng, step0=step0, v0=v0)
    mask = st.mask.cpu().numpy()
    worst = {}
    for s in range(k):
        pts = points(s)
        p0, m0, v0_ = (x.cpu().numpy().copy() for x in (st.p, st.m, st.v))
        loss, _, g, out = p.step(p0, pts)
        TG128._step_adam(p, st, pts, h, st.ring)
        torch.cuda.synchronize()
        t = step0 + s + 1
        stag = '%s step %d (t = %g)' % (tag, s, t)
        assert torch.equal(st.out, out), '%s: out differs from pinn_step in %d of %d' % (
            stag, int((st.out != out).sum()), out.numel())
        w = check_adam_elements(stag, h, t, p0, m0, v0_, g, mask, (st.p.cpu().numpy(), st.m.cpu().numpy(),
                                                                   st.v.cpu().numpy()))
        worst = {key: max(val, worst.get(key, 0.0)) for key, val in w.items()}
        assert torch.equal(st.steps, torch.full_like(st.steps, float(t))), stag
        assert int(st.counter) == s + 1, stag
        assert st.ring[s % RING].cpu().numpy().view(np.int32) == np.float32(loss).view(np.int32), stag
    print('NOISE %s: %s' % (tag, ' '.join('%s %.3f' % kv for kv in worst.items())))
    return worst


def _device_points(pts):
    return torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float32)).cuda()


# ---- the families --------------------------------------------------------------------------------------------------
N_ADAM = 3001
THREAD_NETS = ('ode_param', 'gelu64')       # per-warp accumulators in smem and in the workspace, by placement


def _thread(name, placement, monkeypatch):
    solver, eng, (smem, warps, acc) = TP._placed_engine(name, placement, monkeypatch)
    assert acc.startswith('per-warp'), '%s %s: gradient accumulators %s' % (name, placement, acc)
    p = _launcher(eng.lib, eng.plan, eng.spec)
    p.keep = solver
    tag = 'step_kernel %s %s (%s, %d warps, accumulators %s)' % (name, placement, 'smem' if smem else 'gmem', warps, acc)
    return p, solver.flat_params().cpu().numpy(), lambda n, seed: TP._points(name, n, seed), tag


COUPLED = {'ns_20x2': 'smem', 'gelu_48x64_k2': 'gmem', 'resnet_silu_40_k4': 'gmem_w1'}


def _coupled(net):
    cfg, _, params, _, _, spec = TCP._setup(net)
    plan, (smem, warps, acc, _) = TCP.placed(spec, COUPLED[net])
    assert (spec.widths[spec.n_layers], smem) == (cfg['k'], COUPLED[net] == 'smem')
    p = _launcher(plan.lib, plan.plan, spec)
    p.keep = plan
    tag = 'coupled_step_kernel %s k=%d %s (%d warps, accumulators %s)' % (net, cfg['k'], COUPLED[net], warps, acc)
    return p, params, lambda n, seed: TCP._points(cfg, n, seed), tag


def _wide(name, monkeypatch):
    spec, _ = TG._spec(TG.EDGE[name])
    p = TG._tile_plan(spec, monkeypatch)
    return p, TG._params(TG.EDGE[name], spec), lambda n, seed: TG._points(TG.EDGE[name], n, seed), 'wide_step_kernel ' + name


def _wide128(name, monkeypatch):
    spec, _ = TG._spec(TG128.EDGE[name])
    p = TG128._plan128(spec, monkeypatch)
    cfg = TG128.EDGE[name]
    return p, TG._params(cfg, spec), lambda n, seed: TG._points(cfg, n, seed), 'wide128_step_kernel ' + name


def _wide128_coupled():
    name = 'navier_stokes2d_wide'
    p = TG128C._plan(TG128C.wide_coupled_spec(name))
    return (p, load_golden(name)['params'],
            lambda n, seed: np.clip(PWC.make_points(name, n, seed=seed), 1e-3, 1.0 - 1e-3),
            'wide128_coupled_step_kernel ' + name)


def _hi(jet, monkeypatch, placement='default'):
    cfg = TH.CASES[jet]
    spec = TH._spec(cfg)
    p = TH._hi_plan(spec, placement, monkeypatch, jet=jet)
    return p, TH._params(cfg, spec), lambda n, seed: TH._points(cfg, n, seed), 'hi_step_kernel<%d, %d> %s (%s)' % (
        jet + (placement, TH._where(p)))


def _family(kind, monkeypatch):
    what, _, arg = kind.partition(':')
    if what == 'thread':
        name, placement = arg.split('@')
        return _thread(name, placement, monkeypatch)
    if what == 'coupled':
        return _coupled(arg)
    if what == 'wide':
        return _wide(arg, monkeypatch)
    if what == 'wide128':
        return _wide128(arg, monkeypatch)
    if what == 'wide128_coupled':
        return _wide128_coupled()
    return _hi(tuple(map(int, arg.split(','))), monkeypatch)


FAMILIES = (['thread:%s@%s' % (n, pl) for n in THREAD_NETS for pl in TP.PLACEMENTS] + ['coupled:' + n for n in COUPLED]
            + ['wide:wide64', 'wide128:mixed', 'wide128_coupled', 'hi:1,3', 'hi:2,4'])


def _close(p):
    """ destroy a plan the test made itself (plans of engines and of the coupled tests' Plan are kept by their maker) """
    if not hasattr(p, 'keep'):
        p.__exit__(None, None, None)


# ---- a. pinn_step_adam = pinn_step + Adam on every family ------------------------------------------------------------
@pytest.mark.parametrize('kind', FAMILIES)
def test_step_adam_equals_step_then_oracle_adam_per_element(kind, monkeypatch):
    p, params, points, tag = _family(kind, monkeypatch)
    try:
        rng = np.random.RandomState(FAMILIES.index(kind))
        adam_steps(tag, p, params, lambda s: _device_points(points(N_ADAM, 300 + s)), rng, step0=37.0)
    finally:
        _close(p)


def test_thread_cases_reach_both_accumulator_placements(monkeypatch):
    """ the step_kernel cases above run with the per-warp gradient accumulators in shared memory and in the
    workspace, each with per-point state in global memory, and in the workspace with state in shared memory """
    seen = set()
    for name in THREAD_NETS:
        for placement in TP.PLACEMENTS:
            with monkeypatch.context() as mp:
                try:
                    _, eng, (smem, _, acc) = TP._placed_engine(name, placement, mp)
                except pytest.skip.Exception:
                    continue
            seen.add((smem, acc))
    assert {(False, 'per-warp, smem'), (False, 'per-warp, workspace'), (True, 'per-warp, workspace')} <= seen, seen


# ---- b. Adam state edges ---------------------------------------------------------------------------------------------
EDGES = {
    't1': dict(step0=0.0),
    't2': dict(step0=1.0),
    't_1e6': dict(step0=1e6),
    'beta1_0': dict(step0=5.0, h=dict(HYPER, beta1=0.0)),
    'beta2_0.9999': dict(step0=5.0, h=dict(HYPER, beta2=0.9999)),
    'eps_1e-3': dict(step0=5.0, h=dict(HYPER, eps=1e-3)),
    'eps_1e-12_v0': dict(step0=5.0, h=dict(HYPER, eps=1e-12), v0=0.0),
}


@pytest.mark.parametrize('kind', ['thread:ode_param@default', 'wide:wide64', 'hi:1,3'])
@pytest.mark.parametrize('edge', list(EDGES))
def test_adam_state_edges(edge, kind, monkeypatch):
    e = EDGES[edge]
    p, params, points, tag = _family(kind, monkeypatch)
    try:
        adam_steps('%s %s' % (tag, edge), p, params, lambda s: _device_points(points(N_ADAM, 500 + s)),
                   np.random.RandomState(11), h=e.get('h', HYPER), step0=e['step0'], k=2, v0=e.get('v0'))
    finally:
        _close(p)


@pytest.mark.parametrize('opt_step0', [0, 1])
@pytest.mark.parametrize('kernel,n', [('small', 100), ('multi', 700)])
def test_persistent_kernels_first_steps(kernel, n, opt_step0):
    """ small_step_kernel / multi_step_kernel at t = 1 and t = 2 from random moments, weight decay, log_scale and the
    first bias frozen: the moments against oracle/adam.py on the fp64 oracle gradient at the bars of
    test_gpu_persistent.test_adam_ring_and_counters_follow_the_oracle, the parameters per element against Adam's update
    of the kernel's own moments (the module docstring's p bar), frozen entries bit-unchanged """
    name = 'heat1d_icvar'
    solver = TPer._solver(name)
    eng = solver._get_engine()
    TPer._preconditions(name, eng, kernel)
    assert TPer._kernel_for(eng, n, {})[0] == kernel
    params = solver.flat_params().cpu().numpy()
    prob = TPer._oracle(name, params.astype(np.float64))
    pts = TPer._points(name, n, seed=80 + opt_step0)
    _, r64, g64 = TPer._oracle_loss_and_grads(prob, name, pts)
    cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(r64)))), 1e-30))
    g64 = np.concatenate([g64, np.zeros(eng.n_params - g64.size)]).astype(np.float32)
    rng = np.random.RandomState(6)
    m0 = (np.abs(g64) * rng.randn(eng.n_params)).astype(np.float32)
    v0 = (g64 * g64 * rng.uniform(0.5, 2.0, eng.n_params) + 1e-12).astype(np.float32)
    mask = np.ones(eng.n_params, dtype=np.float32)
    mask[rng.choice(eng.n_params, eng.n_params // 7, replace=False)] = 0.0
    names = dict(TPer._tensors(name, eng))
    mask[names['log_scale']] = 0.0
    mask[names['b0']] = 0.0
    st = TPer._State.fresh(eng, params, ring_len=RING, step0=0)
    st.m.copy_(torch.from_numpy(m0)); st.v.copy_(torch.from_numpy(v0)); st.mask.copy_(torch.from_numpy(mask))
    st.steps.fill_(float(opt_step0))
    h = dict(lr=3e-3, beta1=0.8, beta2=0.99, eps=1e-6, weight_decay=0.01)
    N.check(TPer._multi_step(eng, st, torch.from_numpy(pts).cuda().reshape(1, n, -1).contiguous(), n, 1,
                             lr=h['lr'], betas=(h['beta1'], h['beta2']), eps=h['eps'], weight_decay=h['weight_decay'],
                             opt_step0=float(opt_step0)))
    torch.cuda.synchronize()
    t = opt_step0 + 1
    tag = '%s t=%d' % (kernel, t)
    p_k, m_k, v_k = (x.cpu().numpy() for x in (st.p, st.m, st.v))
    _, m_o, v_o = oracle_adam.adam_step(params.copy(), g64, m0.copy(), v0.copy(), t, mask=mask, **{
        'lr': h['lr'], 'beta1': h['beta1'], 'beta2': h['beta2'], 'eps': h['eps'], 'weight_decay': h['weight_decay']})
    assert rel_l2(m_k, m_o) <= 1e-5 * cond and rel_l2(v_k, v_o) <= 1e-5 * cond, tag
    # the parameters from the kernel's own moments: the gradient's error against the fp64 oracle does not enter
    p_e, bar = update_bar(_f32(h), t, params, m_k, v_k)
    on = mask != 0
    err = np.abs(p_k.astype(np.float64) - p_e)[on]
    bar = bar[on]
    ratio = float(np.max(np.where(err == 0, 0.0, err / np.maximum(bar, 1e-300))))
    print('NOISE persistent %s: p %.3f m %.1e v %.1e' % (tag, ratio, rel_l2(m_k, m_o), rel_l2(v_k, v_o)))
    assert ratio <= 1.0, '%s: parameter update off Adam\'s at t = %d by %.2f of the bar' % (tag, t, ratio)
    for a, b in ((p_k, params), (m_k, m0), (v_k, v0)):
        assert np.array_equal(a[~on], b[~on]), tag
    assert torch.equal(st.steps, torch.full_like(st.steps, float(t)))


# ---- c. fold-group edges ---------------------------------------------------------------------------------------------
def _grids(sm):
    return sorted({1, 2, 11, 12, 13, 24, 25, sm - 1, sm})


def test_thread_kernel_fold_groups_match_fp64_oracle(monkeypatch):
    """ one warp per CTA: n = 32 G points run on G CTAs, 32 G + 1 on G + 1 (on sm_count CTAs at G = sm_count) """
    name = 'poisson2d'
    p, params, points, tag = _thread(name, 'gmem_w1', monkeypatch)
    eng = p.keep._get_engine()
    sm = eng.info.sm_count
    cuts = sorted({32 * g + d for g in _grids(sm) for d in (0, 1)})
    pts, ref = TP._oracle_prefixes(name, params.astype(np.float64), cuts)
    for n in cuts:
        loss, res, grads, _ = p.step(params, _device_points(pts[:n]))
        TG._check('%s n=%d (%d CTAs)' % (tag, n, min(sm, (n + 31) // 32)), eng.spec, (loss, res, grads), ref[n][:3])
    for g in (13, 25):
        adam_steps('%s G=%d' % (tag, g), p, params, lambda s: _device_points(points(32 * g, 700 + s)),
                   np.random.RandomState(g), step0=37.0, k=2)


def test_wide_kernel_fold_groups_match_fp64_oracle(monkeypatch):
    """ PINN_WIDE_CTAS = G on n = 128 G points (one 128-point tile per CTA), and G + 1 CTAs on 128 G + 1 points """
    name = 'narrow9'
    cfg = TG.EDGE[name]
    spec, _ = TG._spec(cfg)
    with TG._tile_plan(spec, monkeypatch) as p:
        sm = p.info.sm_count
        params = TG._params(cfg, spec)
        runs = [(128 * g, g) for g in _grids(sm)] + [(128 * g + 1, min(g + 1, sm)) for g in _grids(sm)]
        cuts = sorted({n for n, _ in runs})
        pts = TG._points(cfg, max(cuts), seed=29)
        ref = TG._oracle_prefixes(('fold', name, tuple(cuts)), cfg, params, pts, cuts)
        for n, ctas in runs:
            monkeypatch.setenv('PINN_WIDE_CTAS', str(ctas))
            loss, res, grads, _ = p.step(params, pts[:n])
            TG._check('wide_step_kernel %s n=%d (%d CTAs)' % (name, n, ctas), spec, (loss, res, grads), ref[n])
        for g in (13, 25):
            monkeypatch.setenv('PINN_WIDE_CTAS', str(g))
            adam_steps('wide_step_kernel %s G=%d' % (name, g), p, params,
                       lambda s: _device_points(TG._points(cfg, 128 * g, 700 + s)), np.random.RandomState(g),
                       step0=37.0, k=2)


def test_hi_kernel_fold_groups_match_fp64_oracle(monkeypatch):
    """ n = 32 warps G points on G CTAs, one point more on G + 1 """
    jet = (1, 3)
    cfg = TH.CASES[jet]
    spec = TH._spec(cfg)
    with TH._hi_plan(spec, 'default', monkeypatch, jet=jet) as p:
        sm, warps = p.info.sm_count, p.where[0]
        params = TH._params(cfg, spec)
        cuts = sorted({32 * warps * g + d for g in _grids(sm) for d in (0, 1)})
        pts = TH._points(cfg, max(cuts), seed=31)
        ref = TH._oracle_prefixes(('fold', jet, tuple(cuts)), cfg, params, pts, cuts)
        for n in cuts:
            loss, res, grads, _ = p.step(params, pts[:n])
            u = p.forward(params, pts[:n])
            TH._check('hi_step_kernel<1, 3> n=%d (%d warps)' % (n, warps), cfg, spec, (loss, res, grads, u), ref[n])
        for g in (13, 25):
            adam_steps('hi_step_kernel<1, 3> G=%d' % g, p, params,
                       lambda s: _device_points(TH._points(cfg, 32 * warps * g, 700 + s)), np.random.RandomState(g),
                       step0=37.0, k=2)


# ---- d. one workspace, changing grids --------------------------------------------------------------------------------
def test_one_workspace_through_changing_fold_shapes(monkeypatch):
    name = 'poisson2d'
    p, params, points, tag = _thread(name, 'gmem_w1', monkeypatch)
    sm = p.keep._get_engine().info.sm_count
    p.ws = torch.zeros(int(p.lib.pinn_workspace_bytes(p.plan, 32 * sm)), dtype=torch.uint8, device=p.dev)
    shared = _state(p.spec, params, np.random.RandomState(4), step0=37.0)
    fresh = _launcher(p.lib, p.plan, p.spec)
    for i, g in enumerate([13, 5, 25, 1, sm, 13]):
        pts = _device_points(points(32 * g, 900 + i))
        alone = TG128._AdamState.clone(shared)
        fresh.ws = None                                  # a zeroed workspace of its own
        TG128._step_adam(fresh, alone, pts, HYPER, alone.ring)
        TG128._step_adam(p, shared, pts, HYPER, shared.ring)
        torch.cuda.synchronize()
        for what in ('out', 'p', 'm', 'v', 'steps', 'counter', 'ring'):
            a, b = getattr(shared, what), getattr(alone, what)
            assert torch.equal(a, b), '%s launch %d (%d CTAs): %s differs in %d entries' % (
                tag, i, g, what, int((a != b).sum()))


# ---- e. through Solver.fit -------------------------------------------------------------------------------------------
FIT_FAMILIES = {'poisson2d': 0, 'wave3d': 1, 'kdv': 0, 'lotka_volterra': 0}       # name -> pinn_plan_info.tensor_core


def _make(name, seed=0):
    return TGC.make_solver(name) if name == 'lotka_volterra' else make_solver(name, seed=seed)


def _flat(solver):
    return solver.flat_params().cpu().numpy().astype(np.float64)


@pytest.mark.parametrize('name', list(FIT_FAMILIES))
def test_weight_decay_in_kernel_adam_equals_torch_adam(name, monkeypatch):
    """ 20 stepwise steps with weight decay and non-default betas: the in-kernel Adam against torch's fused Adam, at
    the bars of test_gpu_fit.test_adam_in_the_step_kernel_equals_torch_adam_and_shares_its_state """
    monkeypatch.setenv('PYDENS_B200_AUTO_PERSISTENT', '0')
    runs = {}
    for mode in ('1', '0'):
        monkeypatch.setenv('PYDENS_B200_FUSED_ADAM', mode)
        s = _make(name)
        s.fit(niters=20, batch_size=3000, lr=0.005, weight_decay=0.01, betas=(0.8, 0.99))
        eng = s._engine
        assert eng is not None and eng.info.tensor_core == FIT_FAMILIES[name]
        assert (eng._adam_flat is not None) == (mode == '1'), 'the in-kernel Adam ran: %s' % (eng._adam_flat is not None)
        runs[mode] = (np.asarray(s.losses, dtype=np.float64), _flat(s))
    la, lb = runs['1'][0], runs['0'][0]
    assert la.shape == lb.shape == (20,)
    assert np.max(np.abs(la - lb) / np.maximum(np.abs(lb), 1e-6)) <= 1e-4
    assert np.linalg.norm(runs['1'][1] - runs['0'][1]) / np.linalg.norm(runs['0'][1]) <= 1e-5


@pytest.mark.parametrize('batch', [3000, 100])
def test_decoupled_weight_decay_is_adamw(batch, monkeypatch):
    """ Adam(decoupled_weight_decay=True) is AdamW: the same parameters from the same start and points, on the
    stepwise route (3000 points) and on a batch that would go to the persistent kernels by itself (100 points; it
    falls back to one step at a time without a warning) """
    runs = {}
    for opt, kw in (('Adam', dict(decoupled_weight_decay=True)), ('AdamW', {})):
        s = make_solver('poisson2d')
        with warnings.catch_warnings():
            warnings.simplefilter('error', UserWarning)
            s.fit(niters=40, batch_size=batch, lr=0.005, optimizer=opt, weight_decay=0.1, **kw)
        runs[opt] = (np.asarray(s.losses, dtype=np.float64), _flat(s))
    assert np.max(np.abs(runs['Adam'][0] - runs['AdamW'][0]) / np.abs(runs['AdamW'][0])) <= 1e-6
    assert np.linalg.norm(runs['Adam'][1] - runs['AdamW'][1]) / np.linalg.norm(runs['AdamW'][1]) <= 1e-6


def test_ensemble_with_decoupled_weight_decay_warns_and_matches_adamw():
    ens = [make_solver('poisson2d', seed=j) for j in range(3)]
    with pytest.warns(UserWarning, match='decoupled weight decay'):
        fit_ensemble(ens, niters=40, batch_size=100, lr=0.005, weight_decay=0.1, decoupled_weight_decay=True)
    for j, a in enumerate(ens):
        b = make_solver('poisson2d', seed=j)
        b.fit(niters=40, batch_size=100, lr=0.005, optimizer='AdamW', weight_decay=0.1)
        assert np.linalg.norm(_flat(a) - _flat(b)) / np.linalg.norm(_flat(b)) <= 1e-6, j
        assert np.max(np.abs(np.asarray(a.losses) - np.asarray(b.losses)) / np.abs(np.asarray(b.losses))) <= 1e-6, j


@pytest.mark.parametrize('counts', ['unequal', 'equal'])
@pytest.mark.parametrize('batch', [3000, 100])
def test_loaded_step_counts_follow_torch_adam(batch, counts, monkeypatch):
    """ an optimizer state loaded with new step counts: 40 on every tensor ('equal'), or 40 on every tensor but 3 on
    the second ('unequal').  torch applies each tensor's own bias correction, and so must fit(optimizer=None), on the
    stepwise route and on the batch that goes persistent by itself: the kernels take one t for all tensors, so unequal
    counts run on torch's Adam, and equal ones on the kernels from the loaded count (load_state_dict keeps the moments
    the engine bound and replaces only the step tensors).  The reference is the same fit with torch's Adam one step at
    a time. """
    runs = {}
    for mode in ('kernels', 'torch'):
        if mode == 'torch':
            monkeypatch.setenv('PYDENS_B200_FUSED_ADAM', '0')
            monkeypatch.setenv('PYDENS_B200_AUTO_PERSISTENT', '0')
        s = make_solver('poisson2d')
        s.fit(niters=5, batch_size=batch, lr=0.005)
        state = s.optimizer.state_dict()
        step0 = [3.0 if i == 1 and counts == 'unequal' else 40.0 for i in range(len(state['state']))]
        for i, st in state['state'].items():
            st['step'] = torch.tensor(step0[i])
        s.optimizer.load_state_dict(state)
        s.fit(niters=20, batch_size=batch, optimizer=None)
        st = [s.optimizer.state[q] for q in s.optimizer.param_groups[0]['params']]
        assert [float(x['step']) for x in st] == [x + 20 for x in step0], mode
        runs[mode] = (np.asarray(s.losses, dtype=np.float64), [q.detach().cpu().numpy().astype(np.float64).ravel()
                                                               for q in s.optimizer.param_groups[0]['params']])
    assert np.max(np.abs(runs['kernels'][0] - runs['torch'][0]) / np.abs(runs['torch'][0])) <= 1e-4
    for i, (a, b) in enumerate(zip(runs['kernels'][1], runs['torch'][1])):
        assert np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30) <= 1e-5, 'parameter tensor %d' % i
