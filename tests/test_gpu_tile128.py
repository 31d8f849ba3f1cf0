""" The 128-wide class of the tensor-core tile kernel, wide_step_kernel<NF, NS, 512, 128> and its forward-only form
(pydens_b200/csrc/pinn_wide_kernel.cuh), against the fp64 oracle and the unmodified reference.

Networks with hidden layers of 65-128 units whose weights do not fit the thread kernel's shared memory (e.g. 3 x 128 or
4 x 100 units) go to this kernel by default; PINN_FORCE_KERNEL=wide128 forces it on any network it covers.  Every
bare-ABI test first asserts from pinn_plan_info that this kernel runs (tensor_core == 2, 512 threads, the intended
jet set).  Checked:
- placement: the example networks of tests/problems_wide.py are refused by the thread kernel and get this kernel by
  default; networks the thread kernel holds keep it; what the kernel does not cover is refused under wide128;
- the fp64 oracle, tensor by tensor, at the tolerances of test_gpu_tile.py: all 15 jet sets on 2-6 linear layers with
  hidden widths at the block edges (65, 72, 96, 100, 127, 128) and mixed, 30 seeded random problems (up to 8 columns
  and 4 variables, V in the initial condition, the L1 / Huber / SmoothL1 criteria), batch and grid edges around the
  64-point tile and about 40 tiles through one CTA;
- bit level: in-kernel sampling equals pinn_sample's points, and steps are identical run to run;
- pinn_step_adam against pinn_step + oracle/adam.py, and CUDA-graph replay against plain launches;
- pinn_forward (the forward-only form) against the fp64 oracle and the reference's `u`;
- Solver: golden parity, a fit trajectory against the reference's own fit, a fused constraint, tiny batches without a
  warning, and (two GPUs) the data-parallel fit against one GPU. """
import ctypes as C
import warnings

import numpy as np
import pytest
import torch

import problems_wide as PW
import test_gpu_tile as TG
from helpers import load_golden, rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    from gpu_helpers import Replay
    from oracle import adam as oracle_adam
    from pydens_b200 import Solver, D, V, _native as N

EDGE_WIDTHS = [65, 72, 96, 100, 127, 128]


def _plan128(spec, monkeypatch, force=True):
    """ A plan on the 128-wide tile kernel (forced, or by default); asserts from pinn_plan_info that it runs. """
    if force:
        monkeypatch.setenv('PINN_FORCE_KERNEL', 'wide128')
    else:
        monkeypatch.delenv('PINN_FORCE_KERNEL', raising=False)
    monkeypatch.delenv('PINN_WIDE_THREADS', raising=False)
    p = TG._Plan(spec)
    try:
        assert p.info.tensor_core == 2, 'the 128-wide tile kernel does not run this plan (%d)' % p.info.tensor_core
        assert (p.info.nf, p.info.ns) == (spec.nf, spec.ns), ((p.info.nf, p.info.ns), (spec.nf, spec.ns))
        assert p.info.threads_per_cta == 512
    except AssertionError:
        p.__exit__(None, None, None)
        raise
    return p


def _create_rc(spec, force):
    """ pinn_plan_create's return code under PINN_FORCE_KERNEL=force (None: default selection) """
    import os
    old = os.environ.pop('PINN_FORCE_KERNEL', None)
    if force:
        os.environ['PINN_FORCE_KERNEL'] = force
    try:
        lib = N.load()
        plan = C.c_void_p()
        rc = lib.pinn_plan_create(C.byref(spec), 0, C.byref(plan))
        info = None
        if rc == 0:
            info = N.PinnPlanInfo()
            N.check(lib.pinn_plan_info(plan, C.byref(info)))
            lib.pinn_plan_destroy(plan)
        return rc, info
    finally:
        os.environ.pop('PINN_FORCE_KERNEL', None)
        if old is not None:
            os.environ['PINN_FORCE_KERNEL'] = old


def _pkg_V(name, init):
    return V(name, data=torch.Tensor([init]))


def _solver(name, params=None, **kw):
    cfg = PW.PROBLEMS[name]
    torch.manual_seed(0)
    solver = Solver(PW.bind(name, D, _pkg_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                    initial_condition=PW.make_ic(name, _pkg_V), boundary_condition=cfg['bc'], domain=cfg['domain'],
                    layout=cfg['layout'], features=cfg['features'], activation=cfg['activation'],
                    device='cuda', backend=kw.pop('backend', 'fused'), seed=1234, **kw)
    if params is not None:
        solver.load_flat_params(params)
    elif 'log_scale' in cfg:
        with torch.no_grad():
            solver.model.log_scale.fill_(cfg['log_scale'])
    return solver


def _lap2(u, x, y, D, V):                       # (2, 2): five jet channels
    return D(D(u, x), x) + D(D(u, y), y) - x * u


# ---- 1. placement --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(PW.PROBLEMS))
def test_example_networks_refused_by_the_thread_kernel_take_the_128_class(name, monkeypatch):
    monkeypatch.delenv('PINN_FORCE_KERNEL', raising=False)
    eng = _solver(name)._get_engine()
    assert eng.info.tensor_core == 2 and eng.info.threads_per_cta == 512
    assert eng.info.small_batch_points == 0 and eng.lib.pinn_multi_step_max_points(eng.plan) == 0
    rc, _ = _create_rc(eng.spec, 'thread')
    assert rc == N.E_UNSUPPORTED, 'the thread kernel holds %s (rc %d): not a network the library refused' % (name, rc)
    rc, _ = _create_rc(eng.spec, 'wide')            # the 64-wide class does not cover it either
    assert rc == N.E_UNSUPPORTED


@pytest.mark.parametrize('hidden', [[65, 16], [128, 128], [128, 72, 100], [100, 128], [128, 16, 128]])
def test_networks_the_thread_kernel_holds_keep_it(hidden):
    cfg = TG._problem(_lap2, 2, [(w, 'Tanh') for w in hidden], bc=0.0)
    spec, _ = TG._spec(cfg)
    rc, info = _create_rc(spec, None)
    assert rc == 0 and info.tensor_core == 0, hidden
    rc, info = _create_rc(spec, 'wide128')           # ... and the 128-wide class can be forced on them
    assert rc == 0 and info.tensor_core == 2, hidden


def _refused(kind):
    if kind == 'width129':
        return TG._problem(_lap2, 2, [(129, 'Tanh'), (16, 'Tanh')], bc=0.0), None
    if kind == 'seven_layers':
        return TG._problem(_lap2, 2, [(100, 'Tanh')] * 6, bc=0.0), None
    if kind == 'width64':                        # the 64-wide class covers it: nothing above 64 units
        return TG._problem(_lap2, 2, [(64, 'Tanh'), (64, 'Tanh')], bc=0.0), None
    if kind in ('gelu', 'sin', 'softplus', 'silu'):
        return TG._problem(_lap2, 2, [(100, 'Tanh'), (100, kind)], bc=0.0), None
    if kind == 'residual':
        return TG._problem(_lap2, 2, [(100, 'Tanh')] * 3, bc=0.0), [None, 0, None, None]
    if kind == 'order3':
        return TG._problem(lambda u, x, t, D, V: D(u, t) + D(D(D(u, x), x), x) + u * D(u, x), 2, [(100, 'Tanh')],
                           bc=0.0), None
    raise KeyError(kind)


@pytest.mark.parametrize('kind', ['width129', 'seven_layers', 'width64', 'residual', 'gelu', 'sin', 'softplus', 'silu',
                                  'order3'])
def test_forced_128_class_refuses_what_it_does_not_cover(kind):
    cfg, skips = _refused(kind)
    traced = TG._trace(cfg)
    spec = N.build_spec([cfg['total']] + TG._features(cfg), TG._acts_names(cfg), cfg['ndims'], cfg['nparams'], True,
                        cfg['bc'], False, cfg['domain'], traced, skips=skips)
    rc, _ = _create_rc(spec, 'wide128')
    assert rc == N.E_UNSUPPORTED, (kind, rc)


def test_too_large_for_every_kernel_is_still_refused():
    cfg = TG._problem(_lap2, 2, [(200, 'Tanh'), (200, 'Tanh'), (200, 'Tanh')], bc=0.0)
    spec, _ = TG._spec(cfg)
    rc, _ = _create_rc(spec, None)
    assert rc == N.E_UNSUPPORTED


# ---- 2. every jet set ----------------------------------------------------------------------------------------------
P_ = TG._problem
JET_SETS = {
    (0, 0): P_(lambda u, x, t, D, V: u * u - torch.sin(x) * t + V('k', 0.5) * u, 2,
               [(128, 'Tanh')], ic=TG._icf_a, variables={'k': 0.5, 'a': 0.4}),
    (1, 0): P_(lambda u, x, D, V: D(u, x) - torch.cos(x) * u, 1, [(9, 'Sigmoid'), (100, None)], bc=0.3),
    (1, 1): P_(lambda u, x, t, D, V: D(D(u, x), x) + u - t, 2, [(65, 'Tanh'), (1, 'Tanh'), (127, 'Sigmoid')],
               ic=0.5, bc=-0.2),
    (2, 0): P_(lambda u, x, t, D, V: D(u, t) + x * D(u, x) - torch.exp(-u), 2,
               [(16, 'Tanh'), (127, 'Sigmoid'), (8, None), (72, 'Tanh'), (96, 'Tanh')], ic=TG._icf_ab,
               variables={'a': 0.4, 'b': -0.2}),
    (2, 1): P_(lambda u, x, t, D, V: D(u, x) - D(D(u, t), t) * V('k', 0.7), 2, [(96, 'Sigmoid'), (100, 'Tanh')],
               bc=0.1, variables={'k': 0.7}),
    (2, 2): P_(lambda u, x, y, D, V: D(D(u, x), x) + D(D(u, y), y) - x * u, 2, [(128, 'Tanh')], bc=0.0),
    (3, 0): P_(lambda u, x, y, t, D, V: D(u, t) + D(u, x) * u - D(u, y) - 0.3, 3,
               [(128, 'Tanh'), (128, None), (128, 'Tanh')], ic=TG._icf_a, variables={'a': 0.4}),
    (3, 1): P_(lambda u, x, y, p, D, V: D(u, x) + p * D(u, y) - D(D(u, p), p), 2, [(72, 'Tanh'), (9, 'Sigmoid')],
               nparams=1, bc=0.2),
    (3, 2): P_(lambda u, x, y, t, D, V: D(u, t) - D(D(u, x), x) - D(D(u, y), y) * V('c', 0.3), 3,
               [(127, 'Sigmoid'), (65, 'Tanh'), (16, None)], ic=TG._icf_ab, bc=0.0,
               variables={'a': 0.4, 'b': -0.2, 'c': 0.3}),
    (3, 3): P_(lambda u, x, y, D, V: D(D(u, x), y) + 0.5 * D(u, y) * u - 0.3, 2,
               [(72, 'Tanh'), (65, 'Sigmoid'), (96, 'Tanh'), (8, None), (100, 'Tanh')], bc=0.4),
    (4, 0): P_(lambda u, x, y, z, t, D, V: D(u, t) + D(u, x) - y * D(u, y) + D(u, z) * u, 4, [(65, 'Tanh')], ic=0.7),
    (4, 1): P_(lambda u, x, y, z, t, D, V: D(u, x) + D(u, y) + D(u, z) - D(D(u, t), t) + u ** 2, 4,
               [(100, 'Tanh'), (127, 'Sigmoid')], bc=-0.1),
    (4, 2): P_(lambda u, x, y, p, q, D, V: D(u, x) + D(u, y) * V('k', 0.7) - D(D(u, p), p) - D(D(u, q), q), 2,
               [(128, 'Tanh'), (96, None), (33, 'Sigmoid'), (72, 'Tanh')], nparams=2, bc=0.0, variables={'k': 0.7}),
    (4, 3): P_(lambda u, x, y, t, D, V: D(u, t) + D(D(u, x), y) - 0.2 * D(u, x) * u, 3,
               [(9, 'Tanh'), (128, 'Sigmoid'), (1, None), (100, 'Tanh'), (16, 'Sigmoid')], ic=TG._icf_a,
               variables={'a': 0.4}),
    (4, 4): P_(lambda u, x, y, z, D, V: D(D(u, x), y) + D(D(u, z), z) + torch.sin(x) * u - y, 3,
               [(128, 'Tanh'), (128, 'Sigmoid'), (128, None), (128, 'Tanh')], bc=0.0),
}


@pytest.mark.parametrize('jet', list(JET_SETS), ids=lambda j: 'nf%d_ns%d' % j)
def test_every_jet_set_matches_fp64_oracle(jet, monkeypatch):
    cfg = JET_SETS[jet]
    spec, _ = TG._spec(cfg)
    assert (spec.nf, spec.ns) == jet, 'the equation traces to (%d, %d)' % (spec.nf, spec.ns)
    params = TG._params(cfg, spec)
    with _plan128(spec, monkeypatch) as p:
        cuts = [1, 63, 64, 65, 64 * p.info.sm_count + 1]
        pts = TG._points(cfg, max(cuts), seed=11)
        ref = TG._oracle_prefixes(('jet128', jet), cfg, params, pts, cuts)
        for n in cuts:
            loss, res, grads, _ = p.step(params, pts[:n])
            TG._check('%s n=%d' % (TG._tag(cfg, spec), n), spec, (loss, res, grads), ref[n])


# ---- 3. seeded random problems -------------------------------------------------------------------------------------
def _random_wide_problem(seed):
    """ test_gpu_tile's random problem generator (equation, columns, ansatz, variables, criterion, batch) on hidden
    widths of the 128-wide class: at the block edges or uniform in 1..128, at least one above 64 """
    cfg, crit, n, _ = TG._random_tile_problem(400 + seed)
    rng = np.random.RandomState(520000 + seed)
    hidden = [(int(rng.choice(EDGE_WIDTHS)) if rng.rand() < 0.6 else int(rng.randint(1, 129)), a)
              for _, a in cfg['hidden']]
    if max(w for w, _ in hidden) <= 64:
        k = int(rng.randint(len(hidden)))
        hidden[k] = (int(rng.choice(EDGE_WIDTHS)), hidden[k][1])
    if all(a is None for _, a in hidden):           # a linear network has no second derivatives for the oracle to take
        hidden[-1] = (hidden[-1][0], 'Tanh')
    cfg['hidden'] = hidden
    return cfg, crit, {127: 63, 129: 65}.get(n, n)


@pytest.mark.parametrize('seed', list(range(30)))
def test_random_problem_matches_fp64_oracle(seed, monkeypatch):
    cfg, crit, n = _random_wide_problem(seed)
    if n < 0:
        n = 64 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    pts = TG._points(cfg, n, seed=6000 + seed)
    params = TG._oracle_problem(cfg).flat_params().numpy().astype(np.float32)
    key, module, inv_n, weight, slack = None, None, None, 1.0, 1.0
    if crit is not None:
        kind, red = crit
        prob = TG._oracle_problem(cfg)
        prob.load_flat(torch.as_tensor(params, dtype=torch.float64))
        _, r64, _ = prob.loss_and_grads(pts.astype(np.float64))
        thr = float(np.float32(np.median(np.abs(r64))))
        key, module = {'l1': (('l1',), torch.nn.L1Loss()), 'huber': (('huber', thr), torch.nn.HuberLoss(delta=thr)),
                       'smooth_l1': (('smooth_l1', thr), torch.nn.SmoothL1Loss(beta=thr))}[kind]
        if red == 'sum':
            inv_n, weight = 1.0, 1.0 / n
        kink = 0.0 if kind == 'l1' else thr         # residuals within fp32 rounding of a kink (test_gpu_tile.py)
        near = np.abs(np.abs(r64) - kink) <= 1e-5 * np.maximum(np.abs(r64), kink)
        slack = 1.0 + 1e4 * float(near.mean()) * (1.0 if kind == 'l1' else 1e-5)
    spec, _ = TG._spec(cfg, key)
    assert spec.nf <= 4 and spec.n_params == params.size
    with _plan128(spec, monkeypatch) as p:
        loss, res, grads, _ = p.step(params, pts, inv_n=inv_n)
    ref = TG._oracle_prefixes(('random128', seed), cfg, params, pts, [n], criterion=module)[n]
    if crit is not None:
        ref = (ref[0], r64, ref[2])
    tag = 'seed %d %s %s criterion=%s n=%d' % (seed, cfg['eq_name'], TG._tag(cfg, spec), crit, n)
    TG._check(tag, spec, (loss, res, grads), ref, weight=weight, residual=crit is None, slack=slack)


def test_largest_network_the_128_class_claims(monkeypatch):
    """ 6 linear layers, every hidden width 128, 8 point columns, 4 variables (two of them in the initial condition);
    the default selection takes it """
    cfg = TG._problem(lambda u, x, y, t, p1, p2, p3, p4, p5, D, V: D(u, t) - D(D(u, x), x) * V('k', 0.7)
                      - D(D(u, y), y) * (p1 + p2 * p3) + V('c', 0.3) * u * p4 - p5, 3,
                      [(128, 'Tanh'), (128, 'Sigmoid'), (128, 'Tanh'), (128, None), (128, 'Tanh')], nparams=5,
                      ic=TG._icf_ab, bc=0.0, variables={'a': 0.4, 'b': -0.2, 'c': 0.3, 'k': 0.7})
    spec, _ = TG._spec(cfg)
    assert spec.n_layers == 6 and spec.n_vars == 4 and spec.ndims + spec.nparams == 8
    params = TG._params(cfg, spec)
    with _plan128(spec, monkeypatch, force=False) as p:
        cuts = [1, 65, 64 * p.info.sm_count + 1]
        pts = TG._points(cfg, max(cuts), seed=41)
        ref = TG._oracle_prefixes(('largest128',), cfg, params, pts, cuts)
        for n in cuts:
            loss, res, grads, _ = p.step(params, pts[:n])
            TG._check('largest %s n=%d' % (TG._tag(cfg, spec), n), spec, (loss, res, grads), ref[n])


# ---- 4. tile and grid edges ----------------------------------------------------------------------------------------
EDGE = {
    'wide128': P_(lambda u, x, y, t, D, V: D(D(u, t), t) - D(D(u, x), x) - D(D(u, y), y) + 0.2 * D(u, x) * u, 3,
                  [(128, 'Tanh'), (128, 'Tanh'), (128, 'Sigmoid')], ic=TG._icf_a, bc=0.0, variables={'a': 0.4}),
    'mixed': P_(lambda u, x, t, D, V: D(u, t) - D(D(u, x), x) * V('k', 0.7) + u ** 3, 2,
                [(65, 'Tanh'), (128, 'Sigmoid'), (100, None)], ic=TG._icf_ab, bc=0.1,
                variables={'a': 0.4, 'b': -0.2, 'k': 0.7}),
}
MANY_TILES = 2503                     # about 40 tiles of 64 points through one CTA


def _edge_cuts(sm):
    r = 64 * sm
    return [1, 2, 63, 64, 65, r - 1, r, r + 1, MANY_TILES, 2 * r + 1]


def _edge_oracle(name, p):
    cfg = EDGE[name]
    params = TG._params(cfg, p.spec)
    cuts = _edge_cuts(p.info.sm_count)
    pts = TG._points(cfg, max(cuts), seed=23)
    return cfg, params, pts, TG._oracle_prefixes(('edge128', name, tuple(cuts)), cfg, params, pts, cuts)


@pytest.mark.parametrize('name', list(EDGE))
def test_tile_and_grid_edges_match_fp64_oracle(name, monkeypatch):
    spec, _ = TG._spec(EDGE[name])
    with _plan128(spec, monkeypatch) as p:
        cfg, params, pts, ref = _edge_oracle(name, p)
        for n in _edge_cuts(p.info.sm_count):
            loss, res, grads, _ = p.step(params, pts[:n])
            TG._check('%s %s n=%d' % (name, TG._tag(cfg, spec), n), spec, (loss, res, grads), ref[n])


@pytest.mark.parametrize('ctas', [1, 7])
@pytest.mark.parametrize('name', list(EDGE))
def test_many_tiles_per_cta_match_fp64_oracle(name, ctas, monkeypatch):
    """ PINN_WIDE_CTAS caps the grid: each CTA walks 40 (1 CTA) or 5-6 (7 CTAs) tiles into one set of accumulators,
    the hidden->hidden ones in the workspace """
    spec, _ = TG._spec(EDGE[name])
    with _plan128(spec, monkeypatch) as p:
        cfg, params, pts, ref = _edge_oracle(name, p)
        monkeypatch.setenv('PINN_WIDE_CTAS', str(ctas))
        loss, res, grads, _ = p.step(params, pts[:MANY_TILES])
        TG._check('%s %s n=%d ctas=%d' % (name, TG._tag(cfg, spec), MANY_TILES, ctas), spec, (loss, res, grads),
                  ref[MANY_TILES])


# ---- 5. bit level --------------------------------------------------------------------------------------------------
def _sampling_problem(total):
    return TG._problem(lambda u, x, y, t, *ps, D, V: D(u, t) - D(D(u, x), x) - D(D(u, y), y) * (1.0 + sum(ps)) + u * x,
                       3, [(128, 'Tanh'), (100, 'Tanh')], nparams=total - 3, ic=TG._icf_a, bc=0.0,
                       variables={'a': 0.4})


@pytest.mark.parametrize('total', [5, 8])
def test_in_kernel_sampling_equals_explicit_points(total, monkeypatch):
    cfg = _sampling_problem(total)
    spec, _ = TG._spec(cfg)
    params = TG._params(cfg, spec)
    cols = TG._columns(total)
    n, seed, step, offset = 3001, 4242, (3 << 32) | 17, 123457
    with _plan128(spec, monkeypatch) as p:
        _, res_s, _, out_s = p.step(params, None, n=n, cols=cols, seed=seed, step=step, offset=offset)
        out_s = out_s.clone()
        pts = p.sample(n, cols, seed, step, offset)
        assert not torch.equal(pts, p.sample(n, cols, seed, step, 0)), 'point_offset has no effect'
        _, res_e, _, out_e = p.step(params, pts)
    assert torch.isfinite(out_s).all()
    assert torch.equal(out_s, out_e), 'sampled and explicit steps differ in %d of %d outputs' % (
        int((out_s != out_e).sum()), out_s.numel())
    assert np.array_equal(res_s, res_e)


@pytest.mark.parametrize('ctas', [None, 1])
def test_step_is_bit_reproducible(ctas, monkeypatch):
    cfg = EDGE['wide128']
    spec, _ = TG._spec(cfg)
    params = TG._params(cfg, spec)
    pts = TG._points(cfg, 20011 if ctas is None else 3001, seed=31)
    with _plan128(spec, monkeypatch, force=False) as p:
        if ctas is not None:
            monkeypatch.setenv('PINN_WIDE_CTAS', str(ctas))
        runs = [p.step(params, pts) for _ in range(3)]
    assert np.isfinite(runs[0][2]).all()
    for r in runs[1:]:
        assert torch.equal(r[3], runs[0][3]), 'outputs differ in %d of %d' % (int((r[3] != runs[0][3]).sum()), r[3].numel())
        assert np.array_equal(r[1], runs[0][1])


# ---- 6. Adam in the step, CUDA graphs ------------------------------------------------------------------------------
ADAM = dict(lr=0.003, beta1=0.85, beta2=0.995, eps=1e-7, weight_decay=0.01)


class _AdamState:
    def __init__(self, n_params, params, rng):
        dev = torch.device('cuda:0')
        self.p = torch.from_numpy(params.copy()).to(dev)
        self.m = torch.from_numpy((0.01 * rng.randn(n_params)).astype(np.float32)).to(dev)
        self.v = torch.from_numpy((1e-4 * rng.uniform(0.5, 2.0, n_params)).astype(np.float32)).to(dev)
        mask = np.ones(n_params, dtype=np.float32)
        mask[rng.choice(n_params, n_params // 7, replace=False)] = 0.0
        self.mask = torch.from_numpy(mask).to(dev)
        self.steps = torch.full((3,), 37.0, dtype=torch.float32, device=dev)
        self.counter = torch.zeros(1, dtype=torch.int64, device=dev)
        self.out = torch.zeros(n_params + 4, dtype=torch.float32, device=dev)

    def clone(self):
        c = object.__new__(_AdamState)
        for k, v in self.__dict__.items():
            setattr(c, k, v.clone())
        return c


def _step_adam(p, st, pts):
    n = pts.shape[0]
    need = int(p.lib.pinn_workspace_bytes(p.plan, n))
    if p.ws is None or p.ws.numel() < need:
        p.ws = torch.zeros(need, dtype=torch.uint8, device=p.dev)
    adam = N.PinnAdam(st.m.data_ptr(), st.v.data_ptr(), st.mask.data_ptr(), st.steps.data_ptr(), st.steps.numel(),
                      ADAM['lr'], ADAM['beta1'], ADAM['beta2'], ADAM['eps'], ADAM['weight_decay'], None, 0)
    N.check(p.lib.pinn_step_adam(p.plan, None, C.c_void_p(st.p.data_ptr()), C.c_void_p(pts.data_ptr()), None,
                                 C.c_uint64(0), C.c_void_p(st.counter.data_ptr()), C.c_uint64(0), C.c_int64(n),
                                 C.c_float(1.0 / n), C.c_void_p(st.out.data_ptr()), None, C.c_void_p(p.ws.data_ptr()),
                                 C.c_size_t(p.ws.numel()), C.byref(adam), p._stream()))


def test_adam_step_equals_step_then_oracle_adam(monkeypatch):
    cfg = EDGE['mixed']
    spec, _ = TG._spec(cfg)
    params = TG._params(cfg, spec)
    rng = np.random.RandomState(9)
    with _plan128(spec, monkeypatch) as p:
        st = _AdamState(spec.n_params, params, rng)
        mask = st.mask.cpu().numpy()
        for s in range(4):
            pts = torch.from_numpy(TG._points(cfg, 4099, seed=90 + s)).cuda()
            p_prev, m_prev, v_prev = (t.cpu().numpy().copy() for t in (st.p, st.m, st.v))
            loss, _, g, _ = p.step(p_prev, pts)
            _step_adam(p, st, pts)
            torch.cuda.synchronize()
            p_o, m_o, v_o = oracle_adam.adam_step(p_prev.copy(), g, m_prev.copy(), v_prev.copy(), 37 + s + 1,
                                                  lr=ADAM['lr'], beta1=ADAM['beta1'], beta2=ADAM['beta2'],
                                                  eps=ADAM['eps'], weight_decay=ADAM['weight_decay'], mask=mask)
            p_k, m_k, v_k = (t.cpu().numpy() for t in (st.p, st.m, st.v))
            assert float(st.out[spec.n_params]) == loss, s             # the same step, the same loss bits
            assert rel_l2(m_k, m_o) <= 1e-5 and rel_l2(v_k, v_o) <= 1e-5, s
            assert rel_l2(p_k - p_prev, p_o - p_prev) <= 1e-4, s
            frozen = mask == 0
            for a, b in ((p_k, p_prev), (m_k, m_prev), (v_k, v_prev)):
                assert np.array_equal(a[frozen], b[frozen]), s
        assert torch.equal(st.steps, torch.full_like(st.steps, 41.0)) and int(st.counter) == 4


def test_graph_replay_equals_plain_launches(monkeypatch):
    cfg = EDGE['wide128']
    spec, _ = TG._spec(cfg)
    params = TG._params(cfg, spec)
    pts = torch.from_numpy(TG._points(cfg, 20011, seed=17)).cuda()
    with _plan128(spec, monkeypatch, force=False) as p:
        st0 = _AdamState(spec.n_params, params, np.random.RandomState(3))
        plain = st0.clone()
        for _ in range(5):
            _step_adam(p, plain, pts)
        torch.cuda.synchronize()
        graphed = st0.clone()
        _step_adam(p, graphed.clone(), pts)                 # warm-up outside the capture (workspace allocated)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            _step_adam(p, graphed, pts)
        for _ in range(5):
            g.replay()
        torch.cuda.synchronize()
    for a, b in ((plain.p, graphed.p), (plain.m, graphed.m), (plain.v, graphed.v), (plain.out, graphed.out)):
        assert torch.equal(a, b), int((a != b).sum())
    assert int(graphed.counter) == 5 and torch.isfinite(plain.p).all()


# ---- 7. forward --------------------------------------------------------------------------------------------------
def _forward(p, params, pts):
    n = pts.shape[0]
    flat = torch.from_numpy(np.ascontiguousarray(params, dtype=np.float32)).to(p.dev)
    x = torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float32)).to(p.dev)
    u = torch.full((n,), float('nan'), dtype=torch.float32, device=p.dev)
    ws = torch.zeros(int(p.lib.pinn_workspace_bytes(p.plan, n)), dtype=torch.uint8, device=p.dev)
    N.check(p.lib.pinn_forward(p.plan, C.c_void_p(flat.data_ptr()), C.c_void_p(x.data_ptr()), C.c_int64(n),
                               C.c_void_p(u.data_ptr()), C.c_void_p(ws.data_ptr()), C.c_size_t(ws.numel()), p._stream()))
    torch.cuda.synchronize()
    return u.cpu().numpy()


@pytest.mark.parametrize('name', list(EDGE))
def test_forward_matches_fp64_oracle(name, monkeypatch):
    """ networks the forward kernel cannot hold: pinn_forward runs the tile kernel's forward-only form """
    cfg = EDGE[name]
    spec, _ = TG._spec(cfg)
    params = TG._params(cfg, spec)
    prob = TG._oracle_problem(cfg)
    prob.load_flat(torch.as_tensor(params, dtype=torch.float64))
    with _plan128(spec, monkeypatch, force=False) as p:
        r = 64 * p.info.sm_count
        pts = TG._points(cfg, 2 * r + 3, seed=29)
        u64 = np.asarray(prob.predict(pts.astype(np.float64)), dtype=np.float64).reshape(-1)
        for n in [1, 63, 64, 65, r + 1, 2 * r + 3]:
            u = _forward(p, params, pts[:n])
            assert np.isfinite(u).all(), n
            assert rel_l2(u, u64[:n]) <= 1e-5, (name, n, rel_l2(u, u64[:n]))


# ---- 8. Solver ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(PW.PROBLEMS))
def test_step_and_predict_match_reference_golden(name):
    g = load_golden(name)
    solver = _solver(name, g['params'])
    eng = solver._get_engine()
    assert eng.info.tensor_core == 2 and eng.n_params == g['params'].size
    loss, grads, residual = solver.loss_and_grads(g['points'])
    grads = grads.cpu().numpy()
    assert abs(loss - float(g['loss'])) <= 1e-5 * abs(float(g['loss']))
    assert rel_l2(residual.cpu().numpy(), g['residual']) <= 1e-5
    assert rel_l2(grads, g['grads']) <= 1e-4
    spec = eng.spec
    for l in range(spec.n_layers):
        w = slice(spec.w_off[l], spec.w_off[l] + spec.widths[l] * spec.widths[l + 1])
        b = slice(spec.b_off[l], spec.b_off[l] + spec.widths[l + 1])
        assert rel_l2(grads[w], g['grads'][w]) <= 1e-4, 'W%d' % l
        assert rel_l2(grads[b], g['grads'][b]) <= 1e-4, 'b%d' % l
    u = solver.predict(*[g['points'][:, i] for i in range(g['points'].shape[1])]).reshape(-1)
    assert rel_l2(u, g['u']) <= 1e-5


@pytest.mark.parametrize('adam', ['kernel', 'torch'])
@pytest.mark.parametrize('name', list(PW.GOLDEN_TRAJ))
def test_fit_trajectory_matches_reference_fit(name, adam, monkeypatch):
    monkeypatch.setenv('PYDENS_B200_FUSED_ADAM', '1' if adam == 'kernel' else '0')
    g = load_golden(name)
    niters, batch, lr = int(g['traj_meta'][0]), int(g['traj_meta'][1]), float(g['traj_meta'][2])
    solver = _solver(name, g['params'])
    batches = [PW.make_points(name, batch, seed=1000 + i) for i in range(niters)]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        solver.fit(niters=niters, batch_size=batch, sampler=Replay(batches), lr=lr)
    assert not [w for w in caught if 'pydens_b200' in str(w.message)], [str(w.message) for w in caught]
    assert solver._engine is not None and solver._engine.info.tensor_core == 2
    losses = np.asarray(solver.losses, dtype=np.float64)
    ref = g['traj_losses'].astype(np.float64)
    assert losses.shape == ref.shape
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 2e-3
    assert abs(losses[-1] - ref[-1]) <= 1e-5 * max(1.0, abs(ref[-1]))
    final = solver.flat_params().cpu().numpy()
    assert np.linalg.norm(final - g['traj_params']) / np.linalg.norm(g['traj_params']) <= 1e-3


def test_tiny_batches_train_stepwise_without_a_warning():
    solver = _solver('poisson_wide128')
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        solver.fit(niters=40, batch_size=50, lr=0.001)
    assert not [w for w in caught if 'pydens_b200' in str(w.message)], [str(w.message) for w in caught]
    eng = solver._engine
    assert eng is not None and eng.info.tensor_core == 2 and eng.info.small_batch_points == 0
    assert len(solver.losses) == 40 and np.isfinite(solver.losses).all()
    assert np.mean(solver.losses[-5:]) < np.mean(solver.losses[:5])


def test_fused_constraint_matches_autograd_constraint(monkeypatch):
    """ a variable in the initial condition and a constraint at t = 0.5 on a 3 x 128 network: the constraint is one
    more launch of the 128-wide tile kernel (a plan with the value channel only); the autograd constraint is the
    yardstick """
    def odevar(u, t):
        return D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t)

    def initial(*args):
        return V('init', data=torch.Tensor([3.0]))

    def make():
        torch.manual_seed(0)
        return Solver(odevar, ndims=1, initial_condition=initial, layout='fafafaf', features=[128, 128, 128, 1],
                      activation='Tanh', constraints=lambda u, t: u(torch.tensor([0.5])) - 0.25)
    rng = np.random.RandomState(5)
    batches = [rng.uniform(size=(150, 1)).astype(np.float32) for _ in range(30)]
    fused = make()
    fused.fit(niters=30, batch_size=150, lr=0.005, sampler=Replay(batches), loss_terms=['equation', 'constraint_0'])
    eng = fused._engine
    assert eng is not None and eng.info.tensor_core == 2 and eng._constraint_plans[0] is not None
    cinfo = N.PinnPlanInfo()
    N.check(eng.lib.pinn_plan_info(eng._constraint_plans[0]['plan'], C.byref(cinfo)))
    assert cinfo.tensor_core == 2 and cinfo.nf == 0
    monkeypatch.setenv('PYDENS_B200_FUSED_CONSTRAINTS', '0')
    hybrid = make()
    hybrid.fit(niters=30, batch_size=150, lr=0.005, sampler=Replay(batches), loss_terms=['equation', 'constraint_0'])
    assert hybrid._engine._constraint_plans[0] is None
    a, b = np.asarray(fused.losses, dtype=np.float64), np.asarray(hybrid.losses, dtype=np.float64)
    assert np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-6)) <= 2e-3
    assert abs(float(fused.model.init.detach()) - float(hybrid.model.init.detach())) <= 1e-4
    assert float(fused.model.init.detach()) != 3.0


def test_backend_fused_accepts_the_network():
    solver = _solver('poisson_wide128', backend='fused')
    assert solver._get_engine().info.tensor_core == 2


# ---- 9. two GPUs -------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpu_fit_matches_single_gpu(tmp_path):
    from test_gpu_multi import _run
    one = _run(1, str(tmp_path / 'w1.json'), problem='poisson_wide128')
    two = _run(2, str(tmp_path / 'w2.json'), problem='poisson_wide128')
    assert one['tensor_core'] == 2 and two['tensor_core'] == 2
    a, b = np.asarray(one['losses']), np.asarray(two['losses'])
    assert a.shape == b.shape == (30,)
    assert np.max(np.abs(a - b) / np.abs(a)) <= 1e-4
    assert abs(one['params_norm'] - two['params_norm']) <= 1e-4 * one['params_norm']
