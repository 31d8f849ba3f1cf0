""" The tensor-core tile kernel wide_step_kernel<NF, NS> (pydens_b200/csrc/pinn_wide_kernel.cuh) against the fp64
oracle, at every jet set, width, depth and tile edge it accepts.

The host emulation (tests/emul) never runs this kernel's own code: its 3xTF32 GEMMs, the zero-padding to 64 units,
the slab layout, the exchange area, the shared-memory accumulators that live across the tiles of a CTA and their
readout.  So every test here runs it on the GPU, through the bare C ABI (plans built by `N.build_spec`, as
test_gpu_fuzz.py does), with `PINN_FORCE_KERNEL=wide`, and first asserts from pinn_plan_info that the tile kernel
is the one that runs, with the jet set it asked for and 512 threads per CTA.

Checked against the fp64 oracle with the tolerances and the cancellation factor of test_gpu_placement.py: the loss,
the residual, the whole gradient and every tensor of it (each W_l, each b_l including the output bias, log_scale and
each V), a tensor whose gradient is 1000x below the whole held to 1e-3 of the whole.  The oracle runs once per
problem over one batch and is cut at each prefix.
- every (NF, NS) with 0 <= NS <= NF <= 4 (the 15 instantiated jet sets), on networks of 2 to 6 linear layers with
  hidden widths at the 16-column block edges and tanh / sigmoid / identity layers; batches of 1, 127, 128, 129 and
  128 * sm_count + 1 points (one tile past a full round, so one CTA walks two tiles);
- 60 seeded random tile-eligible problems: point columns 1-8 (parameter columns too), bc / ic ansatz with ic callables
  that use V, 0-4 variables, log_scale != 0, and on some seeds the criteria tracer.apply_criterion lowers, and batches
  up to 128 * sm_count + 1 points;
- tile and grid edges around 128 * sm_count, and about 40 tiles through one CTA (PINN_WIDE_CTAS=1 / 7): the
  accumulators are zeroed once per launch and summed over every tile of the CTA;
- bit level: in-kernel sampling equals pinn_sample's points (5 and 8 columns: the second Philox block), and steps
  are identical run to run;
- where the kernel is placed by default, which networks it refuses, and that the largest network it claims (6
  linear layers, every hidden width 64, 8 columns, 4 variables) gets a plan and runs on it. """
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import rel_l2

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200)]

if torch.cuda.is_available():
    from oracle import autograd_port as ap
    from pydens_b200 import _native as N, tracer as T


# ---- problems ---------------------------------------------------------------------------------------------------
# A problem: equation(u, *xs, D, V); ndims / nparams; ic: None, a number, or a factory V -> callable of the spatial
# coordinates; bc: None or a number; hidden: [(width, activation or None for identity)]; variables: {name: init},
# kept sorted by name, the order of the flat parameter vector.
def _problem(eq, ndims, hidden, nparams=0, ic=None, bc=None, variables=None, log_scale=0.15, domain=None,
             param_range=(0.5, 2.0), seed=0):
    domain = domain or [(-0.3 - 0.1 * k, 1.1 + 0.2 * k) for k in range(ndims)]
    return dict(eq=eq, ndims=ndims, nparams=nparams, total=ndims + nparams, hidden=list(hidden), ic=ic, bc=bc,
                variables=dict(sorted((variables or {}).items())), log_scale=log_scale, domain=domain,
                ranges=list(domain) + [param_range] * nparams, seed=seed)


def _ic_of(cfg, V):
    return cfg['ic'](V) if callable(cfg['ic']) else cfg['ic']


def _layout(cfg):
    return ' '.join('fa' if a else 'f' for _, a in cfg['hidden']) + ' f'


def _features(cfg):
    return [w for w, _ in cfg['hidden']] + [1]


def _acts_names(cfg):
    return [a.lower() if a else 'none' for _, a in cfg['hidden']] + ['none']


def _trace(cfg, criterion=None):
    sym_V = lambda n, init: T.Sym(T.var(n))
    nsp = cfg['ndims'] - 1 if cfg['ic'] is not None else cfg['ndims']
    return T.trace(lambda u, *xs: cfg['eq'](u, *xs, D=T.sym_D, V=sym_V), cfg['total'], None,
                   initial_condition=_ic_of(cfg, sym_V), ndims_spatial=nsp, criterion=criterion)


def _spec(cfg, criterion=None):
    traced = _trace(cfg, criterion)
    return N.build_spec([cfg['total']] + _features(cfg), _acts_names(cfg), cfg['ndims'], cfg['nparams'],
                        cfg['bc'] is not None, cfg['bc'] if cfg['bc'] is not None else 0.0, cfg['ic'] is not None,
                        cfg['domain'], traced), traced


def _oracle_problem(cfg):
    holder = {}
    ic = _ic_of(cfg, lambda n, init: holder['prob'].V(n, init))
    prob = ap.Problem(cfg['eq'], ndims=cfg['ndims'], nparams=cfg['nparams'], initial_condition=ic,
                      boundary_condition=cfg['bc'], domain=cfg['domain'], features=_features(cfg),
                      activation=[a for _, a in cfg['hidden'] if a] or 'Tanh', dtype=torch.float64,
                      variables=cfg['variables'] or None, seed=cfg['seed'], layout=_layout(cfg))
    holder['prob'] = prob
    with torch.no_grad():
        prob.log_scale.fill_(cfg['log_scale'])
    return prob


def _points(cfg, n, seed):
    rng = np.random.RandomState(seed)
    return np.concatenate([rng.uniform(lo, hi, size=(n, 1)) for lo, hi in cfg['ranges']], axis=1).astype(np.float32)


def _tag(cfg, spec):
    return 'nf=%d ns=%d cols=%d widths=%s acts=%s ic=%s bc=%s vars=%s' % (
        spec.nf, spec.ns, cfg['total'], _features(cfg)[:-1], [a or 'id' for _, a in cfg['hidden']],
        'V' if callable(cfg['ic']) else cfg['ic'], cfg['bc'], sorted(cfg['variables']))


# ---- the fp64 oracle on prefixes of one batch -------------------------------------------------------------------
_ORACLE = {}


def _oracle_prefixes(key, cfg, params, pts, cuts, criterion=None):
    """ {n: (loss, residual [n], grads)} on the prefixes `cuts` of `pts`, the sums cut at each prefix (the loss and
    the gradients are means over the points: their sums add over segments).  Cached under `key`. """
    if key in _ORACLE:
        return _ORACLE[key]
    prob = _oracle_problem(cfg)
    prob.load_flat(torch.as_tensor(params, dtype=torch.float64))
    pts = pts.astype(np.float64)
    bounds = sorted(set([0] + list(cuts)))
    sums, res = {}, []
    l_acc, g_acc = 0.0, None
    import warnings
    for a, b in zip(bounds[:-1], bounds[1:]):
        for c0 in range(a, b, 20000):
            c1 = min(b, c0 + 20000)
            with warnings.catch_warnings():
                warnings.simplefilter('ignore', UserWarning)
                l, r, g = prob.loss_and_grads(pts[c0:c1], criterion=criterion)
            l_acc += l * (c1 - c0)
            g = g.numpy() * (c1 - c0)
            g_acc = g if g_acc is None else g_acc + g
            res.append(r)
        sums[b] = (l_acc / b, np.concatenate(res), g_acc / b)
    _ORACLE[key] = sums
    return sums


# ---- the tile kernel through the bare C ABI ---------------------------------------------------------------------
class _Plan:
    """ A plan through the bare C ABI (include/pinn_b200.h) and what pinn_plan_info reports about it. """

    def __init__(self, spec):
        self.lib = N.load()
        self.spec = spec
        self.plan = C.c_void_p()
        N.check(self.lib.pinn_plan_create(C.byref(spec), 0, C.byref(self.plan)))
        self.info = N.PinnPlanInfo()
        N.check(self.lib.pinn_plan_info(self.plan, C.byref(self.info)))
        self.dev = torch.device('cuda:0')
        self.ws = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.lib.pinn_plan_destroy(self.plan)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def step(self, params, points, n=None, cols=None, seed=0, step=0, offset=0, inv_n=None):
        """ One step, explicit points (`points`: numpy or a device tensor) or sampled in the kernel (points=None)
        -> (loss, residual [n], grads [n_params], out [n_params + 4] device tensor). """
        n = points.shape[0] if n is None else n
        flat = torch.from_numpy(np.ascontiguousarray(params, dtype=np.float32)).to(self.dev)
        if points is not None and not torch.is_tensor(points):
            points = torch.from_numpy(np.ascontiguousarray(points, dtype=np.float32)).to(self.dev)
        out = torch.zeros(self.spec.n_params + 4, dtype=torch.float32, device=self.dev)
        res = torch.zeros(n, dtype=torch.float32, device=self.dev)
        need = int(self.lib.pinn_workspace_bytes(self.plan, n))
        if self.ws is None or self.ws.numel() < need:
            self.ws = torch.zeros(need, dtype=torch.uint8, device=self.dev)
        N.check(self.lib.pinn_step(
            self.plan, C.c_void_p(flat.data_ptr()), C.c_void_p(points.data_ptr()) if points is not None else None,
            N.make_columns(cols, self.spec.ndims + self.spec.nparams), C.c_uint64(seed), None, C.c_uint64(step),
            C.c_uint64(offset), C.c_int64(n), C.c_float(1.0 / n if inv_n is None else inv_n),
            C.c_void_p(out.data_ptr()), C.c_void_p(res.data_ptr()), C.c_void_p(self.ws.data_ptr()),
            C.c_size_t(self.ws.numel()), self._stream()))
        torch.cuda.synchronize(self.dev)
        o = out.cpu().numpy()
        return float(o[self.spec.n_params]), res.cpu().numpy(), o[:self.spec.n_params].copy(), out

    def sample(self, n, cols, seed, step, offset):
        pts = torch.empty(n, self.spec.ndims + self.spec.nparams, dtype=torch.float32, device=self.dev)
        N.check(self.lib.pinn_sample(self.plan, N.make_columns(cols, pts.shape[1]), C.c_uint64(seed), None,
                                     C.c_uint64(step), C.c_uint64(offset), C.c_int64(n), C.c_void_p(pts.data_ptr()),
                                     self._stream()))
        torch.cuda.synchronize(self.dev)
        return pts


def _abi_step(spec, params, points, **kw):
    """ gpu_helpers.abi_step for the tile kernel: one step through the bare C ABI, explicit points
    -> (pinn_plan_info, loss, residual [n], grads [n_params]). """
    with _Plan(spec) as p:
        loss, res, grads, _ = p.step(params, points, **kw)
        return p.info, loss, res, grads


def _tile_plan(spec, monkeypatch):
    """ A plan forced onto the tile kernel; asserts from pinn_plan_info that this is what runs. """
    monkeypatch.setenv('PINN_FORCE_KERNEL', 'wide')
    p = _Plan(spec)
    info = p.info
    try:
        assert info.tensor_core == 1, 'the tile kernel does not run this plan'
        assert (info.nf, info.ns) == (spec.nf, spec.ns), ((info.nf, info.ns), (spec.nf, spec.ns))
        assert info.threads_per_cta == 512, info.threads_per_cta
    except AssertionError:
        p.__exit__(None, None, None)                 # the caller's `with` never starts: destroy the plan here
        raise
    return p


def _tensors(spec):
    """ (name, slice) of every tensor of the flat gradient: W_l, b_l (the last is the output bias), log_scale, V_i """
    out = []
    for l in range(spec.n_layers):
        out.append(('W%d' % l, slice(spec.w_off[l], spec.w_off[l] + spec.widths[l] * spec.widths[l + 1])))
        out.append(('b%d' % l, slice(spec.b_off[l], spec.b_off[l] + spec.widths[l + 1])))
    out.append(('log_scale', slice(spec.log_scale_off, spec.log_scale_off + 1)))
    out += [('V%d' % i, slice(spec.var_off[i], spec.var_off[i] + 1)) for i in range(spec.n_vars)]
    return out


def _check(tag, spec, got, ref, weight=1.0, residual=True, slack=1.0):
    """ loss, residual, the whole gradient and every tensor against the fp64 oracle (tolerances and cancellation
    factor of test_gpu_placement.test_placement_matches_fp64_oracle) """
    loss, res, grads = got
    ref_loss, ref_res, ref_g = ref
    loss, grads = loss * weight, grads * np.float32(weight)
    cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(ref_res)))), 1e-30))
    assert np.isfinite(grads).all(), tag
    assert abs(loss - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), '%s: loss %r vs %r' % (tag, loss, ref_loss)
    if residual:
        assert rel_l2(res, ref_res) <= 2e-5 * cond, tag
    assert rel_l2(grads[:ref_g.size], ref_g) <= 1e-4 * cond * slack, tag
    scale = 1e-3 * np.linalg.norm(ref_g)           # a tensor whose gradient is 1000x below the whole is held to that
    for name, sl in _tensors(spec):
        err = np.linalg.norm(grads[sl] - ref_g[sl]) / max(np.linalg.norm(ref_g[sl]), scale, 1e-30)
        assert err <= 1e-4 * cond * slack, '%s: %s rel err %.2e' % (tag, name, err)


def _params(cfg, spec):
    params = _oracle_problem(cfg).flat_params().numpy().astype(np.float32)
    assert params.size == spec.n_params, (params.size, spec.n_params)
    return params


# ---- 1. every jet set ---------------------------------------------------------------------------------------------
def _icf_a(V):
    return lambda *x: torch.sin(1.5 * x[0]) * V('a', 0.4) + 0.3


def _icf_ab(V):
    return lambda *x: x[0] * (1.0 - x[-1]) * V('a', 0.4) + V('b', -0.2)


# (NF, NS) -> problem.  Directions: the second-order ones first (D(D(u, x), x), and e_i + e_j for a mixed derivative
# by polarisation), the first-order-only ones after them — several equations name a first-order-only direction
# before a second-order one.  Depth 2 .. 6 linear layers; hidden widths at the 16-column block edges.
JET_SETS = {
    (0, 0): _problem(lambda u, x, t, D, V: u * u - torch.sin(x) * t + V('k', 0.5) * u, 2,
                     [(64, 'Tanh')], ic=_icf_a, variables={'k': 0.5, 'a': 0.4}),
    (1, 0): _problem(lambda u, x, D, V: D(u, x) - torch.cos(x) * u, 1, [(9, 'Sigmoid'), (47, None)], bc=0.3),
    (1, 1): _problem(lambda u, x, t, D, V: D(D(u, x), x) + u - t, 2, [(48, 'Tanh'), (1, 'Tanh'), (17, 'Sigmoid')],
                     ic=0.5, bc=-0.2),
    (2, 0): _problem(lambda u, x, t, D, V: D(u, t) + x * D(u, x) - torch.exp(-u), 2,
                     [(16, 'Tanh'), (63, 'Sigmoid'), (8, None), (33, 'Tanh'), (49, 'Tanh')], ic=_icf_ab,
                     variables={'a': 0.4, 'b': -0.2}),
    (2, 1): _problem(lambda u, x, t, D, V: D(u, x) - D(D(u, t), t) * V('k', 0.7), 2, [(49, 'Sigmoid'), (49, 'Tanh')],
                     bc=0.1, variables={'k': 0.7}),
    (2, 2): _problem(lambda u, x, y, D, V: D(D(u, x), x) + D(D(u, y), y) - x * u, 2, [(33, 'Tanh')], bc=0.0),
    (3, 0): _problem(lambda u, x, y, t, D, V: D(u, t) + D(u, x) * u - D(u, y) - 0.3, 3,
                     [(64, 'Tanh'), (64, None), (64, 'Tanh')], ic=_icf_a, variables={'a': 0.4}),
    (3, 1): _problem(lambda u, x, y, p, D, V: D(u, x) + p * D(u, y) - D(D(u, p), p), 2, [(17, 'Tanh'), (9, 'Sigmoid')],
                     nparams=1, bc=0.2),
    (3, 2): _problem(lambda u, x, y, t, D, V: D(u, t) - D(D(u, x), x) - D(D(u, y), y) * V('c', 0.3), 3,
                     [(63, 'Sigmoid'), (47, 'Tanh'), (16, None)], ic=_icf_ab, bc=0.0,
                     variables={'a': 0.4, 'b': -0.2, 'c': 0.3}),
    (3, 3): _problem(lambda u, x, y, D, V: D(D(u, x), y) + 0.5 * D(u, y) * u - 0.3, 2,
                     [(8, 'Tanh'), (8, 'Sigmoid'), (8, 'Tanh'), (8, None), (8, 'Tanh')], bc=0.4),
    (4, 0): _problem(lambda u, x, y, z, t, D, V: D(u, t) + D(u, x) - y * D(u, y) + D(u, z) * u, 4, [(1, 'Tanh')],
                     ic=0.7),
    (4, 1): _problem(lambda u, x, y, z, t, D, V: D(u, x) + D(u, y) + D(u, z) - D(D(u, t), t) + u ** 2, 4,
                     [(47, 'Tanh'), (63, 'Sigmoid')], bc=-0.1),
    (4, 2): _problem(lambda u, x, y, p, q, D, V: D(u, x) + D(u, y) * V('k', 0.7) - D(D(u, p), p) - D(D(u, q), q), 2,
                     [(64, 'Tanh'), (48, None), (33, 'Sigmoid'), (17, 'Tanh')], nparams=2, bc=0.0,
                     variables={'k': 0.7}),
    (4, 3): _problem(lambda u, x, y, t, D, V: D(u, t) + D(D(u, x), y) - 0.2 * D(u, x) * u, 3,
                     [(9, 'Tanh'), (64, 'Sigmoid'), (1, None), (49, 'Tanh'), (16, 'Sigmoid')], ic=_icf_a,
                     variables={'a': 0.4}),
    (4, 4): _problem(lambda u, x, y, z, D, V: D(D(u, x), y) + D(D(u, z), z) + torch.sin(x) * u - y, 3,
                     [(64, 'Tanh'), (64, 'Sigmoid'), (64, None), (64, 'Tanh')], bc=0.0),
}


@pytest.mark.parametrize('jet', list(JET_SETS), ids=lambda j: 'nf%d_ns%d' % j)
def test_every_jet_set_matches_fp64_oracle(jet, monkeypatch):
    cfg = JET_SETS[jet]
    spec, _ = _spec(cfg)
    assert (spec.nf, spec.ns) == jet, 'the equation traces to (%d, %d)' % (spec.nf, spec.ns)
    params = _params(cfg, spec)
    with _tile_plan(spec, monkeypatch) as p:
        sm = p.info.sm_count
        cuts = [1, 127, 128, 129, 128 * sm + 1]
        pts = _points(cfg, max(cuts), seed=11)
        ref = _oracle_prefixes(('jet', jet), cfg, params, pts, cuts)
        for n in cuts:
            loss, res, grads, _ = p.step(params, pts[:n])
            _check('%s n=%d' % (_tag(cfg, spec), n), spec, (loss, res, grads), ref[n])


# ---- 2. seeded random tile-eligible problems --------------------------------------------------------------------
EDGE_WIDTHS = [1, 8, 9, 16, 17, 33, 47, 48, 49, 63, 64]
CRITERIA = [('l1', 'mean'), ('huber', 'sum'), ('smooth_l1', 'mean'), ('l1', 'sum'), ('huber', 'mean'),
            ('smooth_l1', 'sum')]


def _random_equations(total):
    """ (name, callable) candidates with `total` point columns: test_emul_fuzz._equations, plus the directions that
    reach four """
    from test_emul_fuzz import _equations
    eqs = _equations(total, total)
    if total >= 3:
        eqs += [('mixed_first', lambda u, *xs, D, V: D(u, xs[0]) + D(D(u, xs[1]), xs[2]) - 0.1 * u)]          # (4, 3)
    if total >= 4:
        eqs += [('four_first', lambda u, *xs, D, V: D(u, xs[0]) - D(u, xs[1]) * xs[2] + D(u, xs[2]) * u + D(u, xs[3])),
                ('four_one', lambda u, *xs, D, V: D(u, xs[0]) + D(u, xs[1]) + D(D(u, xs[3]), xs[3]) - D(u, xs[2]) * u),
                ('four_two', lambda u, *xs, D, V: D(u, xs[3]) + D(u, xs[0]) * xs[1] - D(D(u, xs[1]), xs[1])
                 - D(D(u, xs[2]), xs[2])),
                ('four_mixed', lambda u, *xs, D, V: D(D(u, xs[0]), xs[1]) + D(D(u, xs[2]), xs[2]) + 0.3 * xs[3] * u)]
    return eqs


def _random_tile_problem(seed):
    rng = np.random.RandomState(310000 + seed)
    ndims = int(rng.randint(1, 5))
    nparams = int(rng.randint(0, 9 - ndims)) if rng.rand() < 0.5 else 0
    total = ndims + nparams
    depth = int(rng.randint(1, 6))                                      # hidden layers: 2 .. 6 linear layers
    widths = [int(rng.choice(EDGE_WIDTHS)) if rng.rand() < 0.7 else int(rng.randint(1, 65)) for _ in range(depth)]
    acts = [[None, 'Tanh', 'Sigmoid'][int(rng.choice(3, p=[0.2, 0.45, 0.35]))] for _ in range(depth)]
    has_ic = ndims >= 2 and bool(rng.rand() < 0.5)
    nsp = ndims - 1 if has_ic else ndims
    ic, ic_vars = None, {}
    if has_ic:
        kind = int(rng.randint(3))
        if kind == 0:
            ic = float(np.round(rng.uniform(-1, 2), 2))
        elif kind == 1:
            ic, ic_vars = _icf_a, {'a': 0.4}
        else:
            ic, ic_vars = _icf_ab, {'a': 0.4, 'b': -0.2}
    bc = float(np.round(rng.uniform(-1, 1), 2)) if (nsp > 0 and rng.rand() < 0.6) else None
    domain = [(float(np.round(rng.uniform(-1, 0.2), 2)), float(np.round(rng.uniform(0.8, 2.5), 2))) for _ in range(ndims)]
    eqs = _random_equations(total)
    name, base = eqs[int(rng.randint(len(eqs)))]
    variables = dict(ic_vars)
    if name == 'var':
        variables['k'] = 0.7
    n_extra = int(rng.randint(0, 4 - len(variables) + 1))
    extra = [('c', 0.4), ('d', -0.3), ('e', 0.25), ('g', 0.6)][:n_extra]
    variables.update(extra)

    def eq(u, *xs, D, V, base=base, extra=tuple(extra)):
        r = base(u, *xs, D=D, V=V)
        for i, (vn, init) in enumerate(extra):
            r = r + V(vn, init) * (xs[i % len(xs)] if i % 2 == 0 else u)
        return r
    cfg = _problem(eq, ndims, list(zip(widths, acts)), nparams=nparams, ic=ic, bc=bc, variables=variables,
                   log_scale=float(np.round(rng.uniform(0.05, 0.5), 2) * rng.choice([-1, 1])), domain=domain,
                   seed=seed)
    cfg['eq_name'] = name
    crit = CRITERIA[(seed // 6) % len(CRITERIA)] if seed % 6 == 5 else None
    n = int(rng.choice([1, 127, 129, 1000, 4097, -1]))     # -1: 128 * sm_count + 1, one CTA walks two tiles
    return cfg, crit, n


@pytest.mark.parametrize('seed', list(range(60)))
def test_random_tile_problem_matches_fp64_oracle(seed, monkeypatch):
    cfg, crit, n = _random_tile_problem(seed)
    if n < 0:
        n = 128 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    pts = _points(cfg, n, seed=5000 + seed)
    params = _oracle_problem(cfg).flat_params().numpy().astype(np.float32)
    key, module, inv_n, weight, slack = None, None, None, 1.0, 1.0
    if crit is not None:
        kind, red = crit
        prob = _oracle_problem(cfg)
        prob.load_flat(torch.as_tensor(params, dtype=torch.float64))
        _, r64, _ = prob.loss_and_grads(pts.astype(np.float64))
        thr = float(np.float32(np.median(np.abs(r64))))               # both branches of Huber / SmoothL1 are met
        key, module = {'l1': (('l1',), torch.nn.L1Loss()), 'huber': (('huber', thr), torch.nn.HuberLoss(delta=thr)),
                       'smooth_l1': (('smooth_l1', thr), torch.nn.SmoothL1Loss(beta=thr))}[kind]
        if red == 'sum':
            inv_n, weight = 1.0, 1.0 / n          # the kernel sums over the points; the oracle's mean is compared
        # a residual within fp32 rounding of a kink of the criterion lands on the other branch in fp32; its weight in
        # the gradient is 1 / n (test_emul_fuzz.test_random_problem_with_other_criteria_matches_torch_criteria)
        kink = 0.0 if kind == 'l1' else thr
        near = np.abs(np.abs(r64) - kink) <= 1e-5 * np.maximum(np.abs(r64), kink)
        slack = 1.0 + 1e4 * float(near.mean()) * (1.0 if kind == 'l1' else 1e-5)
    spec, _ = _spec(cfg, key)
    assert spec.nf <= 4 and spec.n_params == params.size
    with _tile_plan(spec, monkeypatch) as p:
        loss, res, grads, _ = p.step(params, pts, inv_n=inv_n)
    ref = _oracle_prefixes(('random', seed), cfg, params, pts, [n], criterion=module)[n]
    if crit is not None:
        ref = (ref[0], r64, ref[2])               # the kernel's residual is the criterion's sqrt(rho(r) + eps)
    tag = 'seed %d %s %s criterion=%s n=%d' % (seed, cfg['eq_name'], _tag(cfg, spec), crit, n)
    _check(tag, spec, (loss, res, grads), ref, weight=weight, residual=crit is None, slack=slack)


# ---- 3. tile and grid edges ---------------------------------------------------------------------------------------
EDGE = {
    'wide64': _problem(lambda u, x, y, t, D, V: D(D(u, t), t) - D(D(u, x), x) - D(D(u, y), y) + 0.2 * D(u, x) * u, 3,
                       [(64, 'Tanh'), (64, 'Tanh'), (64, 'Sigmoid')], ic=_icf_a, bc=0.0, variables={'a': 0.4}),
    'narrow9': _problem(lambda u, x, t, D, V: D(u, t) - D(D(u, x), x) * V('k', 0.7) + u ** 3, 2,
                        [(9, 'Tanh'), (9, 'Sigmoid'), (9, None)], ic=_icf_ab, bc=0.1,
                        variables={'a': 0.4, 'b': -0.2, 'k': 0.7}),
}
MANY_TILES = 5003                     # about 40 tiles through one CTA


def _edge_cuts(sm):
    r = 128 * sm
    return [1, 2, 127, 128, 129, r - 1, r, r + 1, MANY_TILES, 2 * r + 1]


def _edge_oracle(name, p):
    cfg = EDGE[name]
    spec = p.spec
    params = _params(cfg, spec)
    cuts = _edge_cuts(p.info.sm_count)
    pts = _points(cfg, max(cuts), seed=23)
    return cfg, params, pts, _oracle_prefixes(('edge', name, tuple(cuts)), cfg, params, pts, cuts)


@pytest.mark.parametrize('name', list(EDGE))
def test_tile_and_grid_edges_match_fp64_oracle(name, monkeypatch):
    spec, _ = _spec(EDGE[name])
    with _tile_plan(spec, monkeypatch) as p:
        cfg, params, pts, ref = _edge_oracle(name, p)
        for n in _edge_cuts(p.info.sm_count):
            loss, res, grads, _ = p.step(params, pts[:n])
            _check('%s %s n=%d' % (name, _tag(cfg, spec), n), spec, (loss, res, grads), ref[n])


@pytest.mark.parametrize('ctas', [1, 7])
@pytest.mark.parametrize('name', list(EDGE))
def test_many_tiles_per_cta_match_fp64_oracle(name, ctas, monkeypatch):
    """ PINN_WIDE_CTAS caps the grid: each CTA walks 40 (1 CTA) or 5-6 (7 CTAs) tiles into one set of accumulators """
    spec, _ = _spec(EDGE[name])
    with _tile_plan(spec, monkeypatch) as p:
        cfg, params, pts, ref = _edge_oracle(name, p)
        monkeypatch.setenv('PINN_WIDE_CTAS', str(ctas))
        n = MANY_TILES
        loss, res, grads, _ = p.step(params, pts[:n])
        _check('%s %s n=%d ctas=%d' % (name, _tag(cfg, spec), n, ctas), spec, (loss, res, grads), ref[n])


# ---- 4. bit level -------------------------------------------------------------------------------------------------
def _sampling_problem(total):
    """ a 64-wide problem with `total` point columns (three of them spatial, the rest parameters) """
    return _problem(lambda u, x, y, t, *ps, D, V: D(u, t) - D(D(u, x), x) - D(D(u, y), y) * (1.0 + sum(ps)) + u * x, 3,
                    [(64, 'Tanh'), (64, 'Tanh')], nparams=total - 3, ic=_icf_a, bc=0.0, variables={'a': 0.4})


def _columns(total):
    base = [(N.COL_UNIFORM, 0.0, 1.0), (N.COL_NORMAL, 0.5, 0.2), (N.COL_UNIFORM, 0.0, 2.0),
            (N.COL_TNORMAL, 0.2, 0.3, 0.0, 0.5),
            ('mix', 'a', [(1.0, N.COL_UNIFORM, 0.1, 1.0), (2.0, N.COL_UNIFORM, 2.0, 4.0)]),
            (N.COL_UNIFORM, -1.0, 1.0), (N.COL_NORMAL, 1.0, 0.5), (N.COL_UNIFORM, 0.5, 1.5)]
    return base[:total]


@pytest.mark.parametrize('total', [5, 8])
def test_in_kernel_sampling_equals_explicit_points(total, monkeypatch):
    """ columns 4 .. 7 come from the second Philox block; a nonzero point_offset shifts the counter """
    cfg = _sampling_problem(total)
    spec, _ = _spec(cfg)
    params = _params(cfg, spec)
    cols = _columns(total)
    n, seed, step, offset = 3001, 4242, (3 << 32) | 17, 123457
    with _tile_plan(spec, monkeypatch) as p:
        _, res_s, _, out_s = p.step(params, None, n=n, cols=cols, seed=seed, step=step, offset=offset)
        out_s = out_s.clone()
        pts = p.sample(n, cols, seed, step, offset)
        assert torch.isfinite(pts).all()
        assert not torch.equal(pts, p.sample(n, cols, seed, step, 0)), 'point_offset has no effect'
        _, res_e, _, out_e = p.step(params, pts)
    assert torch.isfinite(out_s).all()
    assert torch.equal(out_s, out_e), 'sampled and explicit steps differ in %d of %d outputs' % (
        int((out_s != out_e).sum()), out_s.numel())
    assert np.array_equal(res_s, res_e)


@pytest.mark.parametrize('ctas', [None, 1])
def test_step_is_bit_reproducible(ctas, monkeypatch):
    cfg = EDGE['wide64']
    spec, _ = _spec(cfg)
    params = _params(cfg, spec)
    pts = _points(cfg, 20011 if ctas is None else 3001, seed=31)
    with _tile_plan(spec, monkeypatch) as p:
        if ctas is not None:
            monkeypatch.setenv('PINN_WIDE_CTAS', str(ctas))
        runs = [p.step(params, pts) for _ in range(3)]
    assert np.isfinite(runs[0][2]).all()
    for r in runs[1:]:
        assert torch.equal(r[3], runs[0][3]), 'outputs differ in %d of %d' % (int((r[3] != runs[0][3]).sum()), r[3].numel())
        assert np.array_equal(r[1], runs[0][1])


# ---- 5. placement and refusals ----------------------------------------------------------------------------------
def _lap2(u, x, y, D, V):                       # (2, 2): five jet channels
    return D(D(u, x), x) + D(D(u, y), y) - x * u


def _first_second(u, x, y, D, V):               # (2, 1): four jet channels
    return D(u, x) - D(D(u, y), y) + u


@pytest.mark.parametrize('eq,width,tile', [(_lap2, 47, False), (_lap2, 48, True), (_first_second, 64, False),
                                           (_lap2, 64, True)])
def test_default_selection_at_its_boundary(eq, width, tile, monkeypatch):
    """ by default the tile kernel takes networks with a hidden layer of 48 units or more and at least 5 channels """
    monkeypatch.delenv('PINN_FORCE_KERNEL', raising=False)
    cfg = _problem(eq, 2, [(width, 'Tanh'), (16, 'Tanh')], bc=0.0)
    spec, traced = _spec(cfg)
    with _Plan(spec) as p:
        assert p.info.tensor_core == int(tile), (width, traced.channels)
        if tile:
            assert p.info.threads_per_cta == 512


def _refused(kind):
    if kind == 'seven_layers':
        return _problem(_lap2, 2, [(16, 'Tanh')] * 6, bc=0.0), None
    if kind == 'width65':
        return _problem(_lap2, 2, [(65, 'Tanh'), (16, 'Tanh')], bc=0.0), None
    if kind in ('gelu', 'sin', 'softplus', 'silu'):
        return _problem(_lap2, 2, [(32, 'Tanh'), (32, kind)], bc=0.0), None
    if kind == 'residual':
        return _problem(_lap2, 2, [(32, 'Tanh'), (32, 'Tanh'), (32, 'Tanh')], bc=0.0), [None, 0, None, None]
    if kind == 'order3':
        return _problem(lambda u, x, t, D, V: D(u, t) + D(D(D(u, x), x), x) + u * D(u, x), 2, [(32, 'Tanh')], bc=0.0), None
    raise KeyError(kind)


@pytest.mark.parametrize('kind', ['seven_layers', 'width65', 'residual', 'gelu', 'sin', 'softplus', 'silu', 'order3'])
def test_forced_tile_kernel_refuses_what_it_does_not_cover(kind, monkeypatch):
    cfg, skips = _refused(kind)
    traced = _trace(cfg)
    acts = _acts_names(cfg)
    spec = N.build_spec([cfg['total']] + _features(cfg), acts, cfg['ndims'], cfg['nparams'], True, cfg['bc'], False,
                        cfg['domain'], traced, skips=skips)
    lib = N.load()
    plan = C.c_void_p()
    monkeypatch.delenv('PINN_FORCE_KERNEL', raising=False)
    assert lib.pinn_plan_create(C.byref(spec), 0, C.byref(plan)) == 0, lib.pinn_last_error()   # the thread kernel runs it
    lib.pinn_plan_destroy(plan)
    monkeypatch.setenv('PINN_FORCE_KERNEL', 'wide')
    plan = C.c_void_p()
    rc = lib.pinn_plan_create(C.byref(spec), 0, C.byref(plan))
    if rc == 0:
        lib.pinn_plan_destroy(plan)
    assert rc == N.E_UNSUPPORTED, (kind, rc)


def test_largest_network_the_tile_kernel_claims(monkeypatch):
    """ 6 linear layers, every hidden width 64, 8 point columns, 4 variables (two of them in the initial condition) """
    cfg = _problem(lambda u, x, y, t, p1, p2, p3, p4, p5, D, V: D(u, t) - D(D(u, x), x) * V('k', 0.7)
                   - D(D(u, y), y) * (p1 + p2 * p3) + V('c', 0.3) * u * p4 - p5, 3,
                   [(64, 'Tanh'), (64, 'Sigmoid'), (64, 'Tanh'), (64, None), (64, 'Tanh')], nparams=5, ic=_icf_ab,
                   bc=0.0, variables={'a': 0.4, 'b': -0.2, 'c': 0.3, 'k': 0.7})
    spec, _ = _spec(cfg)
    assert spec.n_layers == 6 and spec.n_vars == 4 and spec.ndims + spec.nparams == 8
    params = _params(cfg, spec)
    with _tile_plan(spec, monkeypatch) as p:
        cuts = [1, 129, 128 * p.info.sm_count + 1]
        pts = _points(cfg, max(cuts), seed=41)
        ref = _oracle_prefixes(('largest',), cfg, params, pts, cuts)
        for n in cuts:
            loss, res, grads, _ = p.step(params, pts[:n])
            _check('largest %s n=%d' % (_tag(cfg, spec), n), spec, (loss, res, grads), ref[n])
