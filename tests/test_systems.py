""" Equations whose residual has several columns, `torch.cat([r_1, …, r_m], dim=1)`, on a network with one output.
The reference trains them with `criterion(residual[N, m], zeros[N, 1])` (model_torch.py:448), which broadcasts: the loss
is the criterion over all N m entries.  The tracer folds the columns into the one residual per point the kernels train
on (tracer.residual_outputs), so these run on every kernel with no change to the device code.  CPU only: the tracer,
the device math (host build, tests/emul) against the reference goldens and the fp64 oracle.  The GPU twin is
test_gpu_systems.py. """
import hashlib
import json
import os
import warnings

import numpy as np
import pytest
import torch

import emul_harness as E
import problems as P
import problems_systems as PS
import test_emul_fuzz as F
from helpers import GOLDEN, load_golden, rel_l2
from oracle import autograd_port as ap
from oracle.adam import adam_step
from pydens_b200 import _native as N
from pydens_b200 import tracer as T

sym_V = lambda n, init: T.Sym(T.var(n))


def traced_system(name, criterion=None):
    cfg = PS.PROBLEMS[name]
    nsp = cfg['ndims'] - 1 if PS.has_ic(name) else cfg['ndims']
    return T.trace(PS.bind(name, T.sym_D, sym_V), cfg['ndims'] + cfg['nparams'], None,
                   initial_condition=PS.make_ic(name, sym_V), ndims_spatial=nsp, criterion=criterion)


def system_spec(name, criterion=None):
    cfg = PS.PROBLEMS[name]
    dom = cfg['domain']
    if isinstance(dom[0], (int, float)):
        dom = [tuple(dom)] * cfg['ndims']
    acts, skips = PS.layer_plan(name)
    return N.build_spec([cfg['ndims'] + cfg['nparams']] + list(cfg['features']), acts, cfg['ndims'], cfg['nparams'],
                        cfg['bc'] is not None, cfg['bc'] if cfg['bc'] is not None else 0.0, PS.has_ic(name), dom,
                        traced_system(name, criterion), skips=skips)


def system_oracle(name, dtype=torch.float64, params=None):
    cfg = PS.PROBLEMS[name]
    holder = {}
    ic = PS.make_ic(name, lambda n, init: holder['prob'].V(n, init))
    prob = ap.Problem(lambda u, *xs, D, V: cfg['equation'](u, *xs, D=D, V=V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                      initial_condition=ic, boundary_condition=cfg['bc'], domain=cfg['domain'], features=cfg['features'],
                      activation=cfg['activation'], dtype=dtype, variables=cfg.get('variables'), layout=cfg['layout'])
    holder['prob'] = prob
    if params is not None:
        prob.load_flat(torch.as_tensor(params))
    return prob


def oracle_loss_and_grads(prob, pts, criterion=None):
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)          # torch's [N, m] vs [N, 1] broadcast warning, as in the reference
        return prob.loss_and_grads(pts, criterion=criterion)


# ------------------------------------------------------------------------------------------------------------------
# tracer
# ------------------------------------------------------------------------------------------------------------------
def _digest(tr):
    parts = [None if prog is None else ([list(i) for i in prog.instrs], list(prog.outs), prog.n_slots)
             for prog in (tr.eq_prog, tr.ic_prog)]
    parts.append((tr.dirs, tr.dir_vecs, tr.ns, tr.var_names, tr.order, tr.n_slots))
    return hashlib.sha256(json.dumps(parts).encode()).hexdigest()


def test_scalar_equations_trace_to_the_programs_they_had_before():
    """ Every registry problem under five criteria traces to the byte-identical programs it traced to before residuals
    of several columns existed (digests recorded then). """
    with open(os.path.join(GOLDEN, 'traced_program_digests.json')) as fh:
        want = json.load(fh)
    got = {'%s|%s' % (name, key): _digest(E.traced_problem(name, key))
           for name in P.PROBLEMS for key in (None, ('l1',), ('huber', 0.5), ('smooth_l1', 0.25, 'sum'), ('mse', 'sum'))}
    assert got == want


SELECT = {'plain': lambda f: f, 'slice': lambda f: f[:, 0:1], 'list': lambda f: f[:, [0]], 'ellipsis': lambda f: f[..., 0:1],
          'last': lambda f: f[:, [-1]], 'split': lambda f: torch.split(f, 1, dim=1)[0], 'split_method': lambda f: f.split(1, 1)[0],
          'split_kw': lambda f: f.split(1, dim=-1)[0], 'chunk': lambda f: torch.chunk(f, 1, dim=1)[0],
          'chunk_method': lambda f: f.chunk(1, -1)[0]}
CONCAT = {'cat': lambda cols: torch.cat(cols, dim=1), 'cat_neg': lambda cols: torch.cat(cols, -1),
          'cat_tuple': lambda cols: torch.cat(tuple(cols), 1), 'concat': lambda cols: torch.concat(cols, dim=1),
          'hstack': lambda cols: torch.hstack(cols), 'column_stack': lambda cols: torch.column_stack(cols),
          'nested': lambda cols: torch.cat([cols[0], torch.cat(cols[1:], dim=1)], dim=1) if len(cols) > 1 else cols[0]}


@pytest.mark.parametrize('select', list(SELECT))
def test_column_selection_of_a_one_output_network_is_the_identity(select):
    def eq(f, x, t):
        return T.sym_D(f, t) - T.sym_D(T.sym_D(f, x), x) + f * torch.sin(x)
    plain = T.trace(eq, 2, None)
    picked = T.trace(lambda f, x, t: eq(SELECT[select](f), x, t), 2, None)
    assert _digest(picked) == _digest(plain)


@pytest.mark.parametrize('concat', list(CONCAT))
def test_concatenation_forms_give_the_same_program(concat):
    cols = lambda f, x, t: [T.sym_D(f, t) - T.sym_D(T.sym_D(f, x), x), f * x - 0.5, T.sym_D(f, x) + torch.cos(t)]
    want = T.trace(lambda f, x, t: torch.cat(cols(f, x, t), dim=1), 2, None)
    got = T.trace(lambda f, x, t: CONCAT[concat](cols(f, x, t)), 2, None)
    assert _digest(got) == _digest(want)
    assert len(want.eq_prog.outs) == 1 + want.channels


def test_one_column_concatenation_is_the_scalar_program():
    eq = lambda f, x, t: T.sym_D(f, t) + f * T.sym_D(f, x) - 0.01 * T.sym_D(T.sym_D(f, x), x)
    for key in (None, ('mse', 'sum'), ('huber', 0.3)):
        assert _digest(T.trace(lambda f, x, t: torch.cat([eq(f, x, t)], dim=1), 2, None, criterion=key)) == \
            _digest(T.trace(eq, 2, None, criterion=key))


REJECTED = {
    'one_dimensional': lambda f, x: T.sym_D(f[:, 0], x),                          # [N]: broadcasts to [N, N] in torch
    'missing_column': lambda f, x: T.sym_D(f[:, 1:2], x),                         # empty in torch
    'row_index': lambda f, x: f[0] - x,
    'step_slice': lambda f, x: f[:, 0:1:2] - x,
    'stack': lambda f, x: torch.stack([T.sym_D(f, x), f], dim=1),                 # [N, 2, 1]
    'cat_rows': lambda f, x: torch.cat([T.sym_D(f, x), f], dim=0),                # [2N, 1]
    'cat_default_dim': lambda f, x: torch.cat([T.sym_D(f, x), f]),
    'arithmetic_on_columns': lambda f, x: 2.0 * torch.cat([T.sym_D(f, x), f], dim=1),
    'math_on_columns': lambda f, x: torch.sin(torch.cat([T.sym_D(f, x), f], dim=1)),
    'D_of_columns': lambda f, x: T.sym_D(torch.cat([f, f * x], dim=1), x),
    'split_rows': lambda f, x: torch.split(f, 1)[0] - x,
    'chunk_rows': lambda f, x: f.chunk(2)[0] - x,
    # a V(...) variable is a one-element tensor and a constant a number in the reference, not [N, 1] columns
    'index_variable': lambda f, x: T.sym_D(f, x) - T.Sym(T.var('k'))[:, 0:1],
    'split_variable': lambda f, x: T.sym_D(f, x) - torch.split(T.Sym(T.var('k')), 1, dim=1)[0],
    'cat_variable': lambda f, x: torch.cat([T.sym_D(f, x), T.Sym(T.var('k'))], dim=1),
    'cat_constant': lambda f, x: torch.cat([T.sym_D(f, x), torch.ones_like(x)], dim=1),
}


def test_coordinates_and_expressions_of_the_points_are_columns():
    """ x[:, 0:1] and (u * x)[:, [0]] are [N, 1] columns in the reference: the identity here too. """
    eq = lambda f, x: T.sym_D(f, x) * x - f * T.Sym(T.var('k'))
    want = T.trace(eq, 1, None)
    got = T.trace(lambda f, x: (T.sym_D(f, x) * x[:, 0:1])[..., 0:1] - (f * T.Sym(T.var('k')))[:, [0]], 1, None)
    assert _digest(got) == _digest(want)


@pytest.mark.parametrize('form', list(REJECTED))
def test_forms_with_other_semantics_stay_on_autograd(form):
    with pytest.raises(T.NotLowerable):
        T.trace(REJECTED[form], 1, None)


def test_forms_with_other_semantics_keep_the_solver_on_the_reference_loop():
    """ f[:, 0] is one-dimensional in the reference, so `D(f, x) - f[:, 0] * cos(x)` is an [N, N] residual there.  It
    does not lower: the Solver keeps such an equation on its autograd path, which computes what the reference does. """
    from pydens_b200 import Solver, D
    eq = lambda f, x: D(f, x) - f[:, 0] * torch.cos(x)
    one_dim = Solver(eq, ndims=1, boundary_condition=0.0, layout='fafaf', features=[8, 8, 1], activation='Tanh',
                     device='cpu', backend='auto')
    assert one_dim._traced is None and 'one-dimensional' in one_dim._lower_error
    with pytest.raises(RuntimeError):
        Solver(eq, ndims=1, boundary_condition=0.0, layout='fafaf', features=[8, 8, 1], activation='Tanh', device='cpu',
               backend='fused')
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        one_dim.fit(niters=3, batch_size=16)
    assert len(one_dim.losses) == 3 and np.isfinite(np.asarray(one_dim.losses, dtype=np.float64)).all()


@pytest.mark.parametrize('name', list(PS.PROBLEMS))
def test_system_problems_lower_through_the_solver(name):
    """ Solver(..., backend='fused') accepts them: only tracing runs here (plans are created on a GPU). """
    from pydens_b200 import Solver, D, V
    cfg = PS.PROBLEMS[name]
    pkg_V = lambda n, init: V(n, data=torch.Tensor([init]))
    with warnings.catch_warnings():
        warnings.simplefilter('ignore', UserWarning)
        solver = Solver(PS.bind(name, D, pkg_V), ndims=cfg['ndims'], nparams=cfg['nparams'],
                        initial_condition=PS.make_ic(name, pkg_V), boundary_condition=cfg['bc'], domain=cfg['domain'],
                        layout=cfg['layout'], features=cfg['features'], activation=cfg['activation'], device='cpu',
                        backend='fused')
    assert solver._traced is not None
    assert solver._traced.var_names == sorted(cfg.get('variables', {}))
    want = traced_system(name)
    assert _digest(solver._traced) == _digest(want)


def test_folded_residual_program_on_the_host_interpreter():
    """ The residual program (tracer.run_program) against numpy: r~ = sqrt(mean_j r_j^2 + eps) and its partials, by
    finite differences of that formula in fp64. """
    eq = lambda f, x: torch.cat([T.sym_D(f, x) - f, f * f - x, torch.sin(f) + 0.2 * T.sym_D(f, x)], dim=1)
    tr = T.trace(eq, 1, None)
    assert tr.channels == 2 and len(tr.eq_prog.outs) == 3
    rng = np.random.RandomState(0)
    u, ux, x = rng.uniform(-1, 1, size=(3, 50))

    def rt(u, ux):
        cols = [ux - u, u * u - x, np.sin(u) + 0.2 * ux]
        return np.sqrt(sum(c * c for c in cols) / 3.0 + 1e-30)
    out = T.run_program(tr.eq_prog, np.stack([u, ux]), x[None, :].copy(), [])
    h = 1e-6
    assert np.allclose(out[0], rt(u, ux), rtol=1e-12)
    assert np.allclose(out[1], (rt(u + h, ux) - rt(u - h, ux)) / (2 * h), rtol=1e-6, atol=1e-9)
    assert np.allclose(out[2], (rt(u, ux + h) - rt(u, ux - h)) / (2 * h), rtol=1e-6, atol=1e-9)


# ------------------------------------------------------------------------------------------------------------------
# device math (host build) against the reference goldens
# ------------------------------------------------------------------------------------------------------------------
def _reference_fp32_error(name, g):
    """ rel-L2 distance of the reference's own fp32 folded residual and gradients from the fp64 oracle: nested autograd
    of order 3 loses digits in fp32, so a comparison against the golden carries that much slack (as in test_emul.py) """
    m = PS.PROBLEMS[name]['m']
    _, r64, g64 = oracle_loss_and_grads(system_oracle(name, params=g['params'].astype(np.float64)), g['points'].astype(np.float64))
    return rel_l2(PS.folded_residual(g['residual'], m), PS.folded_residual(r64, m)), rel_l2(g['grads'], g64.numpy())


@pytest.mark.parametrize('name', list(PS.PROBLEMS))
def test_device_math_matches_reference_goldens(name):
    g = load_golden(name)
    m = PS.PROBLEMS[name]['m']
    assert g['residual'].shape == (g['points'].shape[0], m)
    spec = system_spec(name)
    assert spec.n_params == g['params'].size
    loss, residual, grads = E.emul_step(spec, g['params'], g['points'])
    slack_r, slack_g = _reference_fp32_error(name, g) if name == 'kdv_two_residuals' else (0.0, 0.0)
    assert abs(loss - float(g['loss'])) <= (1e-5 + 2.0 * slack_r) * abs(float(g['loss']))
    assert rel_l2(residual, PS.folded_residual(g['residual'], m)) <= 1e-5 + 1.5 * slack_r
    assert rel_l2(grads, g['grads']) <= 1e-4 + 1.5 * slack_g
    # per tensor: every weight and bias, log_scale, every variable
    for l in range(spec.n_layers):
        n_in, n_out = spec.widths[l], spec.widths[l + 1]
        for off, size in ((spec.w_off[l], n_in * n_out), (spec.b_off[l], n_out)):
            assert rel_l2(grads[off:off + size], g['grads'][off:off + size]) <= 1e-4 + 1.5 * slack_g, (l, off)
    tails = [spec.log_scale_off] + [spec.var_off[i] for i in range(spec.n_vars)]
    for off in tails:
        if PS.has_ic(name) or off != spec.log_scale_off:
            assert abs(grads[off] - g['grads'][off]) <= (1e-4 + 1.5 * slack_g) * max(abs(g['grads'][off]), 1e-3 * np.abs(g['grads']).max()), off
    u = E.emul_forward(spec, g['params'], g['points'])
    assert rel_l2(u, g['u']) <= 1e-5


@pytest.mark.parametrize('name', list(PS.GOLDEN_TRAJ))
def test_emulated_fit_follows_the_reference_fit(name):
    """ The whole loop on the CPU: device math for loss and gradients, the oracle's Adam for optimizer.step(), on the
    batches the reference's own Solver.fit saw. """
    g = load_golden(name)
    niters, batch, lr = int(g['traj_meta'][0]), int(g['traj_meta'][1]), float(g['traj_meta'][2])
    spec = system_spec(name)
    params = g['params'].astype(np.float32).copy()
    m, v = np.zeros_like(params), np.zeros_like(params)
    losses = []
    for i in range(niters):
        loss, _, grads = E.emul_step(spec, params, PS.make_points(name, batch, seed=1000 + i))
        losses.append(loss)
        adam_step(params, grads, m, v, i + 1, lr=lr)
    losses, ref = np.asarray(losses, dtype=np.float64), g['traj_losses'].astype(np.float64)
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 2e-3
    assert abs(losses[-1] - ref[-1]) <= 1e-5 * max(1.0, abs(ref[-1]))
    assert np.linalg.norm(params - g['traj_params']) / np.linalg.norm(g['traj_params']) <= 1e-3


CRITERIA = {'mse_sum': (('mse', 'sum'), lambda d: torch.nn.MSELoss(reduction='sum')),
            'l1': (('l1',), lambda d: torch.nn.L1Loss()),
            'huber': (('huber', None), lambda d: torch.nn.HuberLoss(delta=d)),
            'smooth_l1_sum': (('smooth_l1', None, 'sum'), lambda d: torch.nn.SmoothL1Loss(beta=d, reduction='sum'))}


@pytest.mark.parametrize('kind', list(CRITERIA))
@pytest.mark.parametrize('name', ['burgers_penalty', 'heat_pair_skip', 'kdv_two_residuals'])
def test_system_problems_under_other_criteria_match_torch_criteria(name, kind):
    g = load_golden(name)
    thr = float(np.float32(np.median(np.abs(g['residual']))))
    key, make = CRITERIA[kind]
    key = tuple(thr if k is None else k for k in key)
    spec = system_spec(name, criterion=key)
    loss, _, grads = E.emul_step(spec, g['params'], g['points'])
    weight = float(g['points'].shape[0]) if key[-1] == 'sum' else 1.0
    l64, _, g64 = oracle_loss_and_grads(system_oracle(name, params=g['params'].astype(np.float64)),
                                        g['points'].astype(np.float64), criterion=make(thr))
    assert abs(loss * weight - l64) <= 2e-5 * abs(l64)
    assert rel_l2(grads * np.float32(weight), g64.numpy()) <= 1e-4


# ------------------------------------------------------------------------------------------------------------------
# random systems against the fp64 oracle
# ------------------------------------------------------------------------------------------------------------------
def _extra_columns(total, has_var):
    cols = [lambda u, xs, D, V: u - 0.5 * xs[0],
            lambda u, xs, D, V: 0.3 * D(u, xs[0]) + torch.sin(xs[-1]),
            lambda u, xs, D, V: u * u - 0.25,
            lambda u, xs, D, V: torch.tanh(u) * xs[0] + 0.1]
    if has_var:
        cols.append(lambda u, xs, D, V: V('k', 0.7) * u - xs[-1])
    return cols


def _random_system(seed):
    rng = np.random.RandomState(310000 + seed)
    family = int(rng.randint(3))
    cfg = [F._random_problem, F._random_many_direction_problem, F._random_high_order_problem][family](int(rng.randint(100000)))
    m = int(rng.randint(1, 5))
    pool = _extra_columns(cfg['total'], bool(cfg['variables']))
    extra = [pool[int(i)] for i in rng.randint(len(pool), size=m - 1)]
    select = list(SELECT)[int(rng.randint(len(SELECT)))]
    concat = list(CONCAT)[int(rng.randint(len(CONCAT)))]
    base = cfg['eq']

    def eq(f, *xs, D, V):
        u = SELECT[select](f)
        return CONCAT[concat]([base(u, *xs, D=D, V=V)] + [c(u, xs, D, V) for c in extra])
    kind = ['mse', 'l1', 'huber', 'smooth_l1'][int(rng.randint(4))]
    use_sum = bool(rng.rand() < 0.4)
    n = int(rng.choice([1, 5, 33, 70]))
    return cfg, eq, m, kind, use_sum, n, '%s m=%d %s %s' % (cfg['eq_name'], m, select, concat)


@pytest.mark.parametrize('seed', list(range(240)))
def test_random_system_matches_fp64_oracle(seed):
    cfg, eq, m, kind, use_sum, n, tag = _random_system(seed)
    nsp = cfg['ndims'] - 1 if cfg['ic'] is not None else cfg['ndims']
    nparams = cfg.get('nparams', 0)
    prob = ap.Problem(eq, ndims=cfg['ndims'], nparams=nparams, initial_condition=cfg['ic'], boundary_condition=cfg['bc'],
                      domain=cfg['domain'], features=cfg['features'], activation=cfg['acts'] or 'Tanh',
                      dtype=torch.float64, variables=cfg['variables'], seed=seed, layout=cfg['layout'])
    with torch.no_grad():
        prob.log_scale.fill_(cfg['log_scale'])
    params = prob.flat_params().numpy().astype(np.float32)
    prob.load_flat(torch.from_numpy(params.astype(np.float64)))
    rng = np.random.RandomState(320000 + seed)
    # points 1e-3 of the width away from the faces, as in test_emul_fuzz.py (the oracle's nested torch.prod backward)
    pts = np.concatenate([rng.uniform(lo + 1e-3 * (hi - lo), hi - 1e-3 * (hi - lo), size=(n, 1)) for lo, hi in cfg['ranges']],
                         axis=1).astype(np.float32)
    _, r64, _ = oracle_loss_and_grads(prob, pts.astype(np.float64))
    thr = float(np.float32(np.median(np.abs(r64))))
    red = 'sum' if use_sum else 'mean'
    key, crit = {'mse': (('mse',), torch.nn.MSELoss(reduction=red)), 'l1': (('l1',), torch.nn.L1Loss(reduction=red)),
                 'huber': (('huber', thr), torch.nn.HuberLoss(delta=thr, reduction=red)),
                 'smooth_l1': (('smooth_l1', thr), torch.nn.SmoothL1Loss(beta=thr, reduction=red))}[kind]
    if use_sum:
        key = key + ('sum',)
    traced = T.trace(lambda u, *xs: eq(u, *xs, D=T.sym_D, V=sym_V), cfg['total'], None, initial_condition=cfg['ic'],
                     ndims_spatial=nsp, criterion=key)
    acts, skips = F._layer_plan(cfg)
    spec = N.build_spec([cfg['total']] + cfg['features'], acts, cfg['ndims'], nparams, cfg['bc'] is not None,
                        cfg['bc'] if cfg['bc'] is not None else 0.0, cfg['ic'] is not None, cfg['domain'], traced, skips=skips)
    loss, residual, grads = E.emul_step(spec, params, pts)
    weight = float(n) if use_sum else 1.0
    ref_loss, ref_res, ref_grads = oracle_loss_and_grads(prob, pts.astype(np.float64), criterion=crit)
    tag = '%s %s %s %s n=%d' % (kind, red, tag, cfg['layout'], n)
    # the tolerances of test_emul_fuzz.py: relaxed by the cancellation factor of a residual far below its O(1) terms,
    # and for the non-smooth criteria by the share of entries within fp32 rounding of a kink
    near_kink = np.abs(np.abs(r64) - (0.0 if kind in ('l1', 'mse') else thr)) <= 1e-5 * np.maximum(np.abs(r64), thr)
    slack = 1.0 if kind == 'mse' else 1.0 + 1e4 * float(near_kink.mean()) * (1.0 if kind == 'l1' else 1e-5)
    cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(r64)))), 1e-30))
    if cfg['eq_name'] in ('biharmonic', 'mixed3'):
        cond *= 5.0
    assert abs(loss * weight - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), tag
    assert rel_l2(grads * np.float32(weight), ref_grads.numpy()) <= 1e-4 * cond * slack, tag
    if kind == 'mse':           # one column: the plain residual (today's program); several: the folded one
        want = ref_res if m == 1 else PS.folded_residual(ref_res, m, red)
        assert rel_l2(residual, want) <= 2e-5 * cond, tag
