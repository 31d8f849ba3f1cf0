""" The coupled form of the 128-wide tile kernel, wide128_coupled_step_kernel<NF, NS> and its forward-only form
(pydens_b200/csrc/pinn_wide_kernel.cuh, wide_step<…, MULTI = true>): networks with 2..4 outputs whose hidden layers
are 65-128 units wide, against the fp64 oracle and the unmodified reference.

Every bare-ABI test first asserts from pinn_plan_info that this kernel runs (tensor_core == 2, 512 threads, the
intended jet set).  The tolerances are those of test_gpu_tile128.py.  Checked:
- placement: the networks of tests/problems_wide_coupled.py are refused by the thread kernel and by the 64-wide class
  and take this kernel by default; coupled networks the thread kernel holds keep it and accept PINN_FORCE_KERNEL=wide128;
  what the kernel does not cover is refused under wide128;
- the fp64 oracle, tensor by tensor: all 15 jet sets x k in {2, 3, 4} on 2-6 linear layers with hidden widths at the
  block edges, 20 seeded random problems (up to 8 columns, V in the equation and the initial condition, the L1 / Huber /
  SmoothL1 / sum criteria), batch and grid edges around the 64-point tile and about 40 tiles through one CTA, and
  pinn_forward [n, k];
- the reference goldens through the C ABI and through Solver, and the reference's own fit with both Adam forms;
- bit level: in-kernel sampling equals pinn_sample's points, runs are identical, CUDA-graph replay equals plain launches,
  and pinn_step_adam equals pinn_step followed by oracle/adam.py;
- Solver: backend='fused', a constraint added by autograd, tiny batches without a warning, and (two GPUs) the
  data-parallel fit against one GPU. """
import contextlib
import ctypes as C
import os
import warnings

import numpy as np
import pytest
import torch

import problems_wide_coupled as PWC
from helpers import load_golden, rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

if torch.cuda.is_available():
    import test_gpu_tile as TG
    import test_gpu_tile128 as TG128
    from gpu_helpers import Replay
    from oracle import adam as oracle_adam
    from oracle import autograd_port as ap
    from pydens_b200 import Solver, D, V, _native as N
    from pydens_b200 import tracer as T
    from test_coupled import folded, oracle_loss_and_grads, random_coupled, sym_V, tolerances
    from test_oracle_wide_coupled import wide_coupled_oracle

EDGE_WIDTHS = [65, 72, 100, 127, 128]
JET_SETS = [(nf, ns) for nf in range(5) for ns in range(nf + 1)]
# hidden layers (width, activation; None = identity) of the jet-set cases: 2..6 linear layers at the block edges
DEPTHS = [
    [(128, 'Tanh')],
    [(65, 'Tanh'), (127, 'Sigmoid')],
    [(100, 'Tanh'), (72, None), (128, 'Tanh')],
    [(127, 'Sigmoid'), (65, 'Tanh'), (100, 'Tanh'), (72, 'Tanh')],
    [(128, 'Tanh'), (100, 'Sigmoid'), (128, None), (65, 'Tanh'), (72, 'Tanh')],
]


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    for k, v in kv.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _plan(spec, force=True):
    """ A plan on the coupled 128-wide tile kernel (forced, or by default); asserts from pinn_plan_info that it runs. """
    with env(PINN_FORCE_KERNEL='wide128' if force else None):
        p = TG._Plan(spec)
    try:
        assert p.info.tensor_core == 2, 'the 128-wide tile kernel does not run this plan (%d)' % p.info.tensor_core
        assert (p.info.nf, p.info.ns) == (spec.nf, spec.ns), ((p.info.nf, p.info.ns), (spec.nf, spec.ns))
        assert p.info.threads_per_cta == 512
        assert spec.widths[spec.n_layers] >= 2
    except AssertionError:
        p.__exit__(None, None, None)
        raise
    return p


def _create_rc(spec, force):
    """ pinn_plan_create's return code and plan info under PINN_FORCE_KERNEL=force (None: default selection) """
    lib = N.load()
    plan = C.c_void_p()
    with env(PINN_FORCE_KERNEL=force):
        rc = lib.pinn_plan_create(C.byref(spec), 0, C.byref(plan))
    info = None
    if rc == 0:
        info = N.PinnPlanInfo()
        N.check(lib.pinn_plan_info(plan, C.byref(info)))
        lib.pinn_plan_destroy(plan)
    return rc, info


def _forward(p, params, pts, k):
    """ pinn_forward -> u [n, k] """
    n = pts.shape[0]
    flat = torch.from_numpy(np.ascontiguousarray(params, dtype=np.float32)).to(p.dev)
    x = torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float32)).to(p.dev)
    u = torch.full((n, k), float('nan'), dtype=torch.float32, device=p.dev)
    ws = torch.zeros(int(p.lib.pinn_workspace_bytes(p.plan, n)), dtype=torch.uint8, device=p.dev)
    N.check(p.lib.pinn_forward(p.plan, C.c_void_p(flat.data_ptr()), C.c_void_p(x.data_ptr()), C.c_int64(n),
                               C.c_void_p(u.data_ptr()), C.c_void_p(ws.data_ptr()), C.c_size_t(ws.numel()), p._stream()))
    torch.cuda.synchronize()
    return u.cpu().numpy()


# ---- problems -------------------------------------------------------------------------------------------------------
class Case:
    """ A random coupled problem of test_coupled.random_coupled (equation, ansatz, variables, criterion) on the hidden
    layers `hidden`: the fp64 oracle, fp32 parameters, points, the criterion and the spec. """

    def __init__(self, seed, hidden, n=None, nparams=None, skips=None, **fixed):
        cfg = random_coupled(seed, **fixed)
        if nparams is not None:                       # more point columns: parameters the network takes as inputs
            cfg['nparams'], cfg['total'] = nparams, cfg['ndims'] + nparams
        self.cfg, self.hidden, self.k = cfg, hidden, cfg['k']
        acts = [a for _, a in hidden if a]
        layout = ''.join('fa' if a else 'f' for _, a in hidden) + 'f'
        features = [w for w, _ in hidden] + [cfg['k']]
        holder = {}
        ic = cfg['ic'](lambda nm, init: holder['prob'].V(nm, init)) if callable(cfg['ic']) else cfg['ic']
        prob = ap.Problem(cfg['eq'], ndims=cfg['ndims'], nparams=cfg['nparams'], initial_condition=ic,
                          boundary_condition=cfg['bc'], domain=cfg['domain'], features=features, activation=acts,
                          dtype=torch.float64, variables=cfg['variables'], seed=seed, layout=layout)
        holder['prob'] = prob
        with torch.no_grad():
            prob.log_scale.fill_(cfg['log_scale'])
        self.params = prob.flat_params().numpy().astype(np.float32)
        prob.load_flat(torch.from_numpy(self.params.astype(np.float64)))
        self.prob = prob
        self.n = cfg['n'] if n is None else n
        rng = np.random.RandomState(430000 + seed)
        ranges = list(cfg['domain']) + [(0.0, 1.0)] * cfg['nparams']
        self.pts = np.concatenate([rng.uniform(lo + 1e-3 * (hi - lo), hi - 1e-3 * (hi - lo), size=(self.n, 1))
                                   for lo, hi in ranges], axis=1).astype(np.float32)
        _, r64, _ = oracle_loss_and_grads(prob, self.pts.astype(np.float64))
        self.r64, self.thr = r64, float(np.float32(np.median(np.abs(r64))))
        kind = cfg['kind']
        self.key, self.crit = {
            'mse': (('mse',), torch.nn.MSELoss()), 'mse_sum': (('mse', 'sum'), torch.nn.MSELoss(reduction='sum')),
            'l1': (('l1',), torch.nn.L1Loss()), 'huber': (('huber', self.thr), torch.nn.HuberLoss(delta=self.thr)),
            'smooth_l1': (('smooth_l1', self.thr), torch.nn.SmoothL1Loss(beta=self.thr))}[kind]
        self.weight = float(self.n) if kind == 'mse_sum' else 1.0
        sym_ic = cfg['ic'](sym_V) if callable(cfg['ic']) else cfg['ic']
        nsp = cfg['ndims'] - 1 if cfg['ic'] is not None else cfg['ndims']
        traced = T.trace(lambda u, *xs: cfg['eq'](u, *xs, D=T.sym_D, V=sym_V), cfg['total'], None,
                         initial_condition=sym_ic, ndims_spatial=nsp, criterion=self.key, n_out=cfg['k'])
        assert (traced.nf, traced.ns) == (cfg['nf'], cfg['ns']), cfg['tag']
        layer_acts = [(a.lower() if a else 'none') for _, a in hidden] + ['none']
        self.spec = N.build_spec([cfg['total']] + features, layer_acts, cfg['ndims'], cfg['nparams'],
                                 cfg['bc'] is not None, cfg['bc'] if cfg['bc'] is not None else 0.0,
                                 cfg['ic'] is not None, cfg['domain'], traced, skips=skips)
        self.tag = '%s cols=%d hidden=%s' % (cfg['tag'], cfg['total'], [(w, a or 'id') for w, a in hidden])

    def oracle(self, pts=None):
        pts = self.pts if pts is None else pts
        loss, res, grads = oracle_loss_and_grads(self.prob, pts.astype(np.float64), criterion=self.crit)
        return loss, np.asarray(res), grads.numpy()

    def check(self, got, ref=None):
        """ loss, residual (the MSE criteria), the whole gradient and every tensor against the fp64 oracle """
        loss, res, grads = got
        ref_loss, ref_res, ref_g = self.oracle() if ref is None else ref
        loss, grads = loss * self.weight, grads * np.float32(self.weight)
        cond, slack = tolerances(self.cfg, self.r64, self.thr)
        _check(self.tag, self.spec, (loss, res, grads), (ref_loss, ref_res, ref_g), self.k, cond, slack,
               self.key if self.cfg['kind'].startswith('mse') else None)


def _check(tag, spec, got, ref, k, cond, slack=1.0, key=None):
    """ test_gpu_tile._check for k outputs: the residual is the per-point folded residual the kernels train on
    (compared for the MSE criteria, `key`) """
    loss, res, grads = got
    ref_loss, ref_res, ref_g = ref
    assert np.isfinite(grads).all(), tag
    assert abs(loss - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), '%s: loss %r vs %r' % (tag, loss, ref_loss)
    if key is not None:
        assert rel_l2(res, folded(ref_res, k, key)) <= 2e-5 * cond, tag
    assert rel_l2(grads[:ref_g.size], ref_g) <= 1e-4 * cond * slack, tag
    scale = 1e-3 * np.linalg.norm(ref_g)
    for name, sl in TG._tensors(spec):
        err = np.linalg.norm(grads[sl] - ref_g[sl]) / max(np.linalg.norm(ref_g[sl]), scale, 1e-30)
        assert err <= 1e-4 * cond * slack, '%s: %s rel err %.2e' % (tag, name, err)


def crit_key(name):
    return PWC.PROBLEMS[name].get('criterion')


def wide_coupled_spec(name):
    cfg = PWC.PROBLEMS[name]
    nsp = cfg['ndims'] - 1 if PWC.has_ic(name) else cfg['ndims']
    traced = T.trace(PWC.bind(name, T.sym_D, sym_V), cfg['ndims'] + cfg['nparams'], None,
                     initial_condition=PWC.make_ic(name, sym_V), ndims_spatial=nsp, criterion=crit_key(name),
                     n_out=cfg['k'])
    acts, skips = PWC.layer_plan(name)
    return N.build_spec([cfg['ndims'] + cfg['nparams']] + list(cfg['features']), acts, cfg['ndims'], cfg['nparams'],
                        cfg['bc'] is not None, cfg['bc'] if cfg['bc'] is not None else 0.0, PWC.has_ic(name),
                        cfg['domain'], traced, skips=skips)


def make_solver(name, backend='fused', **kw):
    cfg = PWC.PROBLEMS[name]
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)           # the [N, m] vs [N, 1] broadcast of the throw-away run
        solver = Solver(PWC.bind(name, D, lambda n, init: V(n, data=torch.Tensor([init]))), ndims=cfg['ndims'],
                        nparams=cfg['nparams'], initial_condition=PWC.make_ic(name, lambda n, init: V(n, data=torch.Tensor([init]))),
                        boundary_condition=cfg['bc'], domain=cfg['domain'], layout=cfg['layout'],
                        features=cfg['features'], activation=cfg['activation'], device='cuda', backend=backend,
                        seed=1234, **kw)
    if 'log_scale' in cfg:
        with torch.no_grad():
            solver.model.log_scale.fill_(cfg['log_scale'])
    return solver


# ---- 1. placement ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(PWC.PROBLEMS))
def test_fixture_networks_refused_by_the_thread_kernel_take_the_128_class(name):
    spec = wide_coupled_spec(name)
    rc, info = _create_rc(spec, None)
    assert rc == 0 and info.tensor_core == 2 and info.threads_per_cta == 512, (rc, info and info.tensor_core)
    assert info.small_batch_points == 0
    assert _create_rc(spec, 'thread')[0] == N.E_UNSUPPORTED
    assert _create_rc(spec, 'wide')[0] == N.E_UNSUPPORTED          # the 64-wide class never takes k > 1
    eng = make_solver(name)._get_engine()
    assert eng.info.tensor_core == 2 and eng.lib.pinn_multi_step_max_points(eng.plan) == 0


@pytest.mark.parametrize('hidden', [[128, 128], [100, 72], [65, 16], [128, 16, 128]])
def test_coupled_networks_the_thread_kernel_holds_keep_it(hidden):
    spec = Case(7, [(w, 'Tanh') for w in hidden], k=3, jet=(2, 2), kind='mse').spec
    rc, info = _create_rc(spec, None)
    assert rc == 0 and info.tensor_core == 0, hidden
    rc, info = _create_rc(spec, 'wide128')
    assert rc == 0 and info.tensor_core == 2, hidden


REFUSED = ['width129', 'residual', 'gelu', 'silu', 'sin', 'softplus', 'order3', 'five_directions', 'width64']


@pytest.mark.parametrize('kind', REFUSED)
def test_forced_128_class_refuses_what_it_does_not_cover(kind):
    hidden, skips, jet = [(100, 'Tanh'), (100, 'Tanh')], None, (2, 2)
    if kind == 'width129':
        hidden = [(129, 'Tanh'), (16, 'Tanh')]
    elif kind == 'width64':
        hidden = [(64, 'Tanh'), (64, 'Tanh')]
    elif kind == 'residual':
        hidden, skips = [(100, 'Tanh')] * 3, [None, 0, None, None]
    elif kind in ('gelu', 'silu', 'sin', 'softplus'):
        hidden = [(100, 'Tanh'), (100, {'gelu': 'GELU', 'silu': 'SiLU', 'sin': 'Sin', 'softplus': 'Softplus'}[kind])]
    elif kind == 'order3':
        jet = (1, 0)
    spec = _refused_spec(hidden, skips, jet)
    if kind == 'order3':
        spec.order = 3
    elif kind == 'five_directions':
        spec.nf, spec.ns = 5, 5
    assert _create_rc(spec, 'wide128')[0] == N.E_UNSUPPORTED, kind


def _refused_spec(hidden, skips, jet):
    cfg = random_coupled(7, k=3, jet=jet, kind='mse')
    sym_ic = cfg['ic'](sym_V) if callable(cfg['ic']) else cfg['ic']
    nsp = cfg['ndims'] - 1 if cfg['ic'] is not None else cfg['ndims']
    traced = T.trace(lambda u, *xs: cfg['eq'](u, *xs, D=T.sym_D, V=sym_V), cfg['total'], None,
                     initial_condition=sym_ic, ndims_spatial=nsp, criterion=('mse',), n_out=3)
    return N.build_spec([cfg['total']] + [w for w, _ in hidden] + [3], [a.lower() for _, a in hidden] + ['none'],
                        cfg['ndims'], cfg['nparams'], cfg['bc'] is not None, cfg['bc'] if cfg['bc'] is not None else 0.0,
                        cfg['ic'] is not None, cfg['domain'], traced, skips=skips)


# ---- 2. every jet set x k ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('k', [2, 3, 4])
@pytest.mark.parametrize('jet', JET_SETS, ids=['nf%d_ns%d' % j for j in JET_SETS])
def test_every_jet_set_and_output_count_matches_fp64_oracle(jet, k):
    i = JET_SETS.index(jet)
    case = Case(1000 + 17 * i + k, DEPTHS[(3 * i + k) % len(DEPTHS)], n=[1, 63, 64, 65, 130][(i + k) % 5],
                k=k, jet=jet, kind='mse')
    with _plan(case.spec) as p:
        loss, res, grads, _ = p.step(case.params, case.pts)
        u = _forward(p, case.params, case.pts, k)
    case.check((loss, res, grads))
    u64 = case.prob.predict(case.pts.astype(np.float64)).reshape(-1, k)
    assert rel_l2(u, u64) <= 1e-5, case.tag


# ---- 3. seeded random problems ----------------------------------------------------------------------------------------
def _random_case(seed):
    """ random_coupled's equation, ansatz, variables, criterion and k on 1..5 hidden layers of the 128-wide class (at
    the block edges or uniform in 1..128, at least one above 64; tanh, sigmoid or identity) and up to 8 columns """
    rng = np.random.RandomState(530000 + seed)
    hidden = []
    for _ in range(int(rng.randint(1, 6))):
        w = int(rng.choice(EDGE_WIDTHS)) if rng.rand() < 0.6 else int(rng.randint(1, 129))
        hidden.append((w, [None, 'Tanh', 'Sigmoid'][int(rng.randint(3))]))
    if max(w for w, _ in hidden) <= 64:
        j = int(rng.randint(len(hidden)))
        hidden[j] = (int(rng.choice(EDGE_WIDTHS)), hidden[j][1])
    if all(a is None for _, a in hidden):
        hidden[-1] = (hidden[-1][0], 'Tanh')
    probe = random_coupled(300 + seed)
    nparams = int(rng.randint(0, 8 - probe['ndims'] + 1))
    kinds = ['mse', 'l1', 'huber', 'smooth_l1', 'mse_sum']
    return Case(300 + seed, hidden, n=int(rng.choice([1, 40, 63, 65, 129, 300])), nparams=nparams,
                kind=kinds[seed % len(kinds)])


@pytest.mark.parametrize('seed', list(range(20)))
def test_random_problem_matches_fp64_oracle(seed):
    case = _random_case(seed)
    assert case.spec.n_params == case.params.size
    with _plan(case.spec) as p:
        loss, res, grads, _ = p.step(case.params, case.pts)
    case.check((loss, res, grads))


def test_random_problems_cover_columns_variables_and_criteria():
    cases = [_random_case(s) for s in range(20)]
    assert max(c.cfg['total'] for c in cases) == 8
    assert {c.cfg['kind'] for c in cases} == {'mse', 'l1', 'huber', 'smooth_l1', 'mse_sum'}
    assert any(c.spec.n_vars and c.spec.ic_has_vars for c in cases) and {c.k for c in cases} >= {2, 3}


# ---- 4. tile and grid edges, forward ----------------------------------------------------------------------------------
MANY_TILES = 2503                     # about 40 tiles of 64 points through one CTA


def _prefix_oracle(prob, pts, cuts, criterion=None):
    """ {n: (loss, residual [n, m], grads)} on the prefixes `cuts` of `pts` (means over points: the sums add) """
    bounds = sorted(set([0] + list(cuts)))
    out, res, l_acc, g_acc = {}, [], 0.0, 0.0
    for a, b in zip(bounds[:-1], bounds[1:]):
        l, r, g = oracle_loss_and_grads(prob, pts[a:b].astype(np.float64), criterion=criterion)
        l_acc, g_acc = l_acc + l * (b - a), g_acc + g.numpy() * (b - a)
        res.append(np.asarray(r).reshape(b - a, -1))
        out[b] = (l_acc / b, np.concatenate(res), g_acc / b)
    return out


_EDGE = {}


def _edge(sm):
    """ the Navier-Stokes fixture at its golden parameters on points up to two rounds of tiles: (params, points,
    {n: oracle}) """
    if sm not in _EDGE:
        name = 'navier_stokes2d_wide'
        params = load_golden(name)['params']
        r = 64 * sm
        cuts = [1, 2, 63, 64, 65, r - 1, r, r + 1, MANY_TILES, 2 * r + 1]
        pts = PWC.make_points(name, max(cuts), seed=23)
        pts = np.clip(pts, 1e-3, 1.0 - 1e-3)
        _EDGE[sm] = (params, pts, cuts, _prefix_oracle(wide_coupled_oracle(name, params=params.astype(np.float64)),
                                                      pts, cuts))
    return _EDGE[sm]


def test_tile_and_grid_edges_match_fp64_oracle():
    spec = wide_coupled_spec('navier_stokes2d_wide')
    with _plan(spec, force=False) as p:
        params, pts, cuts, ref = _edge(p.info.sm_count)
        for n in cuts:
            loss, res, grads, _ = p.step(params, pts[:n])
            r64 = ref[n][1]
            cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(r64)))), 1e-30))
            _check('n=%d' % n, spec, (loss, res, grads), ref[n], 3, cond, key=('mse',))


@pytest.mark.parametrize('ctas', [1, 7])
def test_many_tiles_per_cta_match_fp64_oracle(ctas):
    """ PINN_WIDE_CTAS caps the grid: each CTA walks 40 (1 CTA) or 5-6 (7 CTAs) tiles into one set of accumulators """
    spec = wide_coupled_spec('navier_stokes2d_wide')
    with _plan(spec, force=False) as p:
        params, pts, _, ref = _edge(p.info.sm_count)
        with env(PINN_WIDE_CTAS=str(ctas)):
            loss, res, grads, _ = p.step(params, pts[:MANY_TILES])
    r64 = ref[MANY_TILES][1]
    cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(r64)))), 1e-30))
    _check('ctas=%d' % ctas, spec, (loss, res, grads), ref[MANY_TILES], 3, cond, key=('mse',))


@pytest.mark.parametrize('name', list(PWC.PROBLEMS))
def test_forward_writes_n_by_k_matching_fp64_oracle(name):
    """ networks the forward kernel cannot hold: pinn_forward runs the coupled tile kernel's forward-only form """
    cfg, g = PWC.PROBLEMS[name], load_golden(name)
    prob = wide_coupled_oracle(name, params=g['params'].astype(np.float64))
    with _plan(wide_coupled_spec(name), force=False) as p:
        r = 64 * p.info.sm_count
        pts = PWC.make_points(name, 2 * r + 3, seed=29)
        u64 = np.asarray(prob.predict(pts.astype(np.float64)), dtype=np.float64).reshape(-1, cfg['k'])
        for n in [1, 63, 64, 65, r + 1, 2 * r + 3]:
            u = _forward(p, g['params'], pts[:n], cfg['k'])
            assert u.shape == (n, cfg['k']) and np.isfinite(u).all(), n
            assert rel_l2(u, u64[:n]) <= 1e-5, (name, n, rel_l2(u, u64[:n]))


# ---- 5. the reference goldens ----------------------------------------------------------------------------------------
def _check_golden(spec, g, name, loss, residual, grads):
    assert abs(loss - float(g['loss'])) <= 1e-5 * abs(float(g['loss']))
    assert rel_l2(residual, folded(g['residual'], PWC.PROBLEMS[name]['m'], crit_key(name))) <= 1e-5
    assert rel_l2(grads, g['grads']) <= 1e-4
    for tname, sl in TG._tensors(spec):
        err =np.linalg.norm(grads[sl] - g['grads'][sl]) / max(np.linalg.norm(g['grads'][sl]),
                                                               1e-3 * np.linalg.norm(g['grads']))
        assert err <= 1e-4, (name, tname, err)


@pytest.mark.parametrize('name', list(PWC.PROBLEMS))
def test_c_abi_matches_reference_golden(name):
    g = load_golden(name)
    spec = wide_coupled_spec(name)
    with _plan(spec, force=False) as p:
        loss, residual, grads, _ = p.step(g['params'], g['points'])
        u = _forward(p, g['params'], g['points'], PWC.PROBLEMS[name]['k'])
    _check_golden(spec, g, name, loss, residual, grads)
    assert rel_l2(u, g['u']) <= 1e-5


@pytest.mark.parametrize('name', list(PWC.PROBLEMS))
def test_solver_matches_reference_golden_and_predicts_n_by_k(name):
    g = load_golden(name)
    solver = make_solver(name)
    solver.load_flat_params(g['params'])
    assert solver._fused_possible(PWC.torch_criterion(name), ('equation',))[0]     # the fused plan of this criterion
    eng = solver._get_engine()
    assert eng.info.tensor_core == 2 and eng.n_params == g['params'].size
    loss, grads, residual = solver.loss_and_grads(g['points'])
    _check_golden(eng.spec, g, name, loss, residual.cpu().numpy().reshape(-1), grads.cpu().numpy()[:g['grads'].size])
    u = solver.predict(*[g['points'][:, i] for i in range(g['points'].shape[1])])
    assert isinstance(u, np.ndarray) and u.shape == g['u'].shape and rel_l2(u, g['u']) <= 1e-5


@pytest.mark.parametrize('fused_adam', ['1', '0'])
@pytest.mark.parametrize('name', list(PWC.GOLDEN_TRAJ))
def test_fit_follows_the_reference_fit(name, fused_adam):
    g = load_golden(name)
    niters, batch, lr = int(g['traj_meta'][0]), int(g['traj_meta'][1]), float(g['traj_meta'][2])
    solver = make_solver(name)
    solver.load_flat_params(g['params'])
    batches = [PWC.make_points(name, batch, seed=1000 + i) for i in range(niters)]
    with env(PYDENS_B200_FUSED_ADAM=fused_adam), warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        solver.fit(niters=niters, batch_size=batch, sampler=Replay(batches), lr=lr, criterion=PWC.torch_criterion(name))
    assert not [w for w in caught if 'pydens_b200' in str(w.message)], [str(w.message) for w in caught]
    assert solver._engine is not None and solver._engine.info.tensor_core == 2
    losses, ref = np.asarray(solver.losses, dtype=np.float64), g['traj_losses'].astype(np.float64)
    assert losses.shape == ref.shape
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 2e-3
    flat = solver.flat_params().cpu().numpy()[:g['traj_params'].size]
    assert rel_l2(flat, g['traj_params']) <= 1e-3


# ---- 6. bit level ----------------------------------------------------------------------------------------------------
def test_in_kernel_sampling_equals_explicit_points_and_runs_are_bit_identical():
    eng = make_solver('react_diff_wide')._get_engine()
    assert eng.info.tensor_core == 2
    n = 30011
    outs = []
    for _ in range(2):
        eng._step(None, None, n, 1.0 / n, 0, use_counter=False, step_value=5)
        torch.cuda.synchronize()
        outs.append(eng.out.clone())
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])
    pts = eng.sample(n, step=5)
    eng._step(pts, None, n, 1.0 / n, 0, use_counter=False)
    torch.cuda.synchronize()
    assert torch.equal(eng.out, outs[0]), int((eng.out != outs[0]).sum())


def test_step_is_bit_reproducible_on_one_cta():
    spec = wide_coupled_spec('quad_wide128_huber')
    params = load_golden('quad_wide128_huber')['params']
    pts = PWC.make_points('quad_wide128_huber', 3001, seed=31)
    with _plan(spec, force=False) as p, env(PINN_WIDE_CTAS='1'):
        runs = [p.step(params, pts) for _ in range(3)]
    assert np.isfinite(runs[0][2]).all()
    for r in runs[1:]:
        assert torch.equal(r[3], runs[0][3]) and np.array_equal(r[1], runs[0][1])


def test_adam_step_equals_step_then_oracle_adam():
    name = 'react_diff_wide'
    spec, params = wide_coupled_spec(name), load_golden(name)['params']
    rng = np.random.RandomState(9)
    with _plan(spec, force=False) as p:
        st = TG128._AdamState(spec.n_params, params, rng)
        mask = st.mask.cpu().numpy()
        A = TG128.ADAM
        for s in range(4):
            pts = torch.from_numpy(PWC.make_points(name, 4099, seed=90 + s)).cuda()
            p_prev, m_prev, v_prev = (t.cpu().numpy().copy() for t in (st.p, st.m, st.v))
            loss, _, g, _ = p.step(p_prev, pts)
            TG128._step_adam(p, st, pts)
            torch.cuda.synchronize()
            p_o, m_o, v_o = oracle_adam.adam_step(p_prev.copy(), g, m_prev.copy(), v_prev.copy(), 37 + s + 1,
                                                  lr=A['lr'], beta1=A['beta1'], beta2=A['beta2'], eps=A['eps'],
                                                  weight_decay=A['weight_decay'], mask=mask)
            p_k, m_k, v_k = (t.cpu().numpy() for t in (st.p, st.m, st.v))
            assert float(st.out[spec.n_params]) == loss, s
            assert rel_l2(m_k, m_o) <= 1e-5 and rel_l2(v_k, v_o) <= 1e-5, s
            assert rel_l2(p_k - p_prev, p_o - p_prev) <= 1e-4, s
            frozen = mask == 0
            for a, b in ((p_k, p_prev), (m_k, m_prev), (v_k, v_prev)):
                assert np.array_equal(a[frozen], b[frozen]), s
        assert torch.equal(st.steps, torch.full_like(st.steps, 41.0)) and int(st.counter) == 4


def test_graph_replay_equals_plain_launches():
    name = 'navier_stokes2d_wide'
    spec, params = wide_coupled_spec(name), load_golden(name)['params']
    pts = torch.from_numpy(PWC.make_points(name, 20011, seed=17)).cuda()
    with _plan(spec, force=False) as p:
        st0 = TG128._AdamState(spec.n_params, params, np.random.RandomState(3))
        plain = st0.clone()
        for _ in range(5):
            TG128._step_adam(p, plain, pts)
        torch.cuda.synchronize()
        graphed = st0.clone()
        TG128._step_adam(p, graphed.clone(), pts)            # warm-up outside the capture (workspace allocated)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            TG128._step_adam(p, graphed, pts)
        for _ in range(5):
            g.replay()
        torch.cuda.synchronize()
    for a, b in ((plain.p, graphed.p), (plain.m, graphed.m), (plain.v, graphed.v), (plain.out, graphed.out)):
        assert torch.equal(a, b), int((a != b).sum())
    assert int(graphed.counter) == 5 and torch.isfinite(plain.p).all()


# ---- 7. Solver -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(PWC.PROBLEMS))
def test_backend_fused_builds_the_network(name):
    solver = make_solver(name, backend='fused')
    assert solver._get_engine().info.tensor_core == 2


def test_constraint_is_added_by_autograd_on_top_of_the_fused_equation():
    name = 'navier_stokes2d_wide'
    batches = [PWC.make_points(name, 256, seed=2000 + i) for i in range(8)]
    cons = lambda u, x, y: u(torch.tensor([0.5]), torch.tensor([0.5]))[:, 2:3] - 0.1     # pin the pressure at a point
    curves = []
    for backend in ('fused', 'torch'):
        solver = make_solver(name, backend=backend, constraints=[cons])
        with warnings.catch_warnings():
            warnings.simplefilter('ignore', UserWarning)
            solver.fit(niters=8, batch_size=256, sampler=Replay(list(batches)), lr=0.002,
                       loss_terms=['equation', 'constraint_0'])
        if backend == 'fused':
            assert solver._engine is not None and solver._engine.info.tensor_core == 2
        curves.append(np.asarray(solver.losses, dtype=np.float64))
    assert np.max(np.abs(curves[0] - curves[1]) / np.abs(curves[1])) <= 1e-4


def test_tiny_batch_trains_step_by_step_without_a_warning():
    solver = make_solver('react_diff_wide')
    eng = solver._get_engine()
    assert eng.info.tensor_core == 2
    assert eng.info.small_batch_points == 0 and eng.lib.pinn_multi_step_max_points(eng.plan) == 0
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        solver.fit(niters=40, batch_size=50, lr=0.001)
    assert not [w for w in caught if 'pydens_b200' in str(w.message)], [str(w.message) for w in caught]
    assert len(solver.losses) == 40 and np.isfinite(solver.losses).all()
    assert np.mean(solver.losses[-5:]) < np.mean(solver.losses[:5])


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpu_fit_matches_single_gpu(tmp_path):
    from test_gpu_multi import _run
    one = _run(1, str(tmp_path / 'w1.json'), problem='navier_stokes2d_wide')
    two = _run(2, str(tmp_path / 'w2.json'), problem='navier_stokes2d_wide')
    assert one['tensor_core'] == 2 and two['tensor_core'] == 2
    a, b = np.asarray(one['losses']), np.asarray(two['losses'])
    assert a.shape == b.shape == (30,)
    assert np.max(np.abs(a - b) / np.abs(a)) <= 1e-4
    assert abs(one['params_norm'] - two['params_norm']) <= 1e-4 * one['params_norm']
