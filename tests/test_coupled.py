""" Coupled systems: networks with k = 2..4 outputs (tests/problems_coupled.py).  The tracer selects component j of the
[N, k] output, gives every component the same jet set and leaves the partials of the residual in one contiguous block
(include/pinn_b200.h, PinnSpec); the k-output form of the per-thread device code (host build, tests/emul) is checked
against the reference goldens, the reference's own fit, and random coupled problems on the fp64 oracle.  The GPU twin
is test_gpu_coupled.py. """
import warnings

import numpy as np
import pytest
import torch

import emul_coupled as EC
import emul_harness as E
import problems_coupled as PC
from helpers import load_golden, rel_l2
from oracle import autograd_port as ap
from oracle.adam import adam_step
from pydens_b200 import _native as N
from pydens_b200 import tracer as T

sym_V = lambda n, init: T.Sym(T.var(n))


def crit_key(name):
    return PC.PROBLEMS[name].get('criterion')


def traced_coupled(name, criterion=None):
    cfg = PC.PROBLEMS[name]
    nsp = cfg['ndims'] - 1 if PC.has_ic(name) else cfg['ndims']
    return T.trace(PC.bind(name, T.sym_D, sym_V), cfg['ndims'] + cfg['nparams'], None, initial_condition=PC.make_ic(name, sym_V),
                   ndims_spatial=nsp, criterion=criterion if criterion is not None else crit_key(name), n_out=cfg['k'])


def coupled_spec(name, criterion=None):
    cfg = PC.PROBLEMS[name]
    dom = cfg['domain']
    if isinstance(dom[0], (int, float)):
        dom = [tuple(dom)] * cfg['ndims']
    acts, skips = PC.layer_plan(name)
    return N.build_spec([cfg['ndims'] + cfg['nparams']] + list(cfg['features']), acts, cfg['ndims'], cfg['nparams'],
                        cfg['bc'] is not None, cfg['bc'] if cfg['bc'] is not None else 0.0, PC.has_ic(name), dom,
                        traced_coupled(name, criterion), skips=skips)


def coupled_oracle(name, dtype=torch.float64, params=None):
    cfg = PC.PROBLEMS[name]
    holder = {}
    ic = PC.make_ic(name, lambda n, init: holder['prob'].V(n, init))
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


def folded(residual, m, key=None):
    """ The per-point residual the kernels train on, from an [N, m] residual: sqrt(mean_j rho(r_j)) (tracer.residual_outputs) """
    r = np.asarray(residual, dtype=np.float64).reshape(-1, m)
    if key is None or key[0] == 'mse':
        rho = r * r
    else:                                                    # Huber
        a, d = np.abs(r), key[1]
        rho = np.where(a <= d, 0.5 * r * r, d * (a - 0.5 * d))
    return np.sqrt(rho.sum(axis=1) if key is not None and key[-1] == 'sum' else rho.mean(axis=1))


def _digest(tr):
    return (tuple(tr.eq_prog.instrs), tuple(tr.eq_prog.outs), tr.n_slots, tuple(tr.dirs), tr.ns)


# ------------------------------------------------------------------------------------------------------------------
# tracer: selection forms, the slot convention, what stays on autograd
# ------------------------------------------------------------------------------------------------------------------
SELECT = {
    'slice': lambda f: (f[:, 0:1], f[:, 1:2], f[:, 2:3]),
    'list': lambda f: (f[:, [0]], f[:, [1]], f[:, [2]]),
    'ellipsis': lambda f: (f[..., 0:1], f[..., 1:2], f[..., 2:3]),
    'split': lambda f: torch.split(f, 1, dim=1),
    'split_sizes': lambda f: torch.split(f, [1, 1, 1], dim=1),
    'chunk': lambda f: torch.chunk(f, 3, dim=1),
    'method_split': lambda f: f.split(1, dim=1),
    'method_split_pos': lambda f: f.split(1, 1),
    'method_chunk': lambda f: f.chunk(3, dim=-1),
}


def _ns_like(f, x, y):
    u, v, p = f
    return torch.cat([u * T.sym_D(u, x) + v * T.sym_D(u, y) + T.sym_D(p, x) - 0.1 * T.sym_D(T.sym_D(u, y), y),
                      T.sym_D(u, x) + T.sym_D(v, y), p * v - torch.sin(x)], dim=1)


@pytest.mark.parametrize('form', list(SELECT))
def test_every_selection_form_gives_the_same_program(form):
    ref = T.trace(lambda f, x, y: _ns_like(SELECT['slice'](f), x, y), 2, None, n_out=3)
    tr = T.trace(lambda f, x, y: _ns_like(SELECT[form](f), x, y), 2, None, n_out=3)
    assert _digest(tr) == _digest(ref)
    assert tr.n_out == 3


def test_tuple_unpacking_of_split():
    def eq(f, x, y):
        u, v, p = torch.split(f, 1, dim=1)
        return torch.cat([T.sym_D(u, x) - v, p * u], dim=1)
    tr = T.trace(eq, 2, None, n_out=3)
    assert tr.nf == 1 and tr.n_out == 3


def test_slot_convention_on_the_host_interpreter():
    """ Slots j*C + c hold channel c of component j; the partials land in the block eq_out[1] + j*C + c. """
    def eq(f, x, t):
        u, v = f[:, 0:1], f[:, 1:2]
        return torch.cat([T.sym_D(u, t) - u * v + T.sym_D(T.sym_D(v, x), x), T.sym_D(v, t) + torch.sin(u) * x], dim=1)
    tr = T.trace(eq, 2, None, n_out=2)
    C = tr.channels
    assert (tr.nf, tr.ns, C) == (2, 1, 4)
    prog = tr.eq_prog
    assert prog.outs[1:1 + C] == [prog.outs[1] + c for c in range(C)]
    rng = np.random.RandomState(0)
    n = 50
    jet = rng.randn(2 * C, n)
    coords = rng.rand(2, n)
    outs = T.run_program(prog, jet, coords, [])
    # program slots -> (u, v) channels: [value, d/dx_dir0, d/dx_dir1, second along dir0]; dir0 = x (second order), dir1 = t
    x, u, v = coords[0], jet[0], jet[C]
    ut, vt, vxx = jet[2], jet[C + 2], jet[C + 3]
    r1, r2 = ut - u * v + vxx, vt + np.sin(u) * x
    assert np.allclose(outs[0], np.sqrt(0.5 * (r1 * r1 + r2 * r2) + 1e-30))
    slots = np.zeros((prog.n_slots, n))
    slots[:2 * C] = jet
    # the whole block, read from the slots the convention names
    full = T.Program(prog.instrs, [prog.outs[1] + s for s in range(2 * C)], prog.n_slots)
    block = T.run_program(full, jet, coords, [])
    g = 1.0 / (2.0 * outs[0])                       # d r~ / d r_j^2 ... r~ = sqrt((r1^2 + r2^2) / 2)
    want = {0: g * r1 * -v, 2: g * r1, C + 0: g * (r1 * -u) + g * r2 * np.cos(u) * x * 0 + g * r2 * 0,
            C + 2: g * r2, C + 3: g * r1}
    want[0] = want[0] + g * r2 * np.cos(u) * x
    for s in range(2 * C):
        assert np.allclose(block[s], want.get(s, 0.0), atol=1e-12), s


def test_one_output_programs_are_unchanged_by_the_output_count_argument():
    def eq(f, x, t):
        return T.sym_D(f, t) - 0.3 * T.sym_D(T.sym_D(f, x), x) + f * f
    assert _digest(T.trace(eq, 2, None)) == _digest(T.trace(eq, 2, None, n_out=1))


REJECTED = {
    'one_dimensional_index': lambda f, x, y: f[:, 0] * x,
    'component_past_k': lambda f, x, y: f[:, 2:3] - x,
    'list_past_k': lambda f, x, y: f[:, [5]] - x,
    'arithmetic_on_whole': lambda f, x, y: f * x,
    'D_on_whole': lambda f, x, y: T.sym_D(f, x),
    'torch_on_whole': lambda f, x, y: torch.sin(f),
    'split_two_wide': lambda f, x, y: torch.split(f, 2, dim=1)[0],
    'chunk_too_few': lambda f, x, y: torch.chunk(f, 1, dim=1)[0],
    'split_rows': lambda f, x, y: torch.split(f, 1, dim=0)[0],
    'wide_slice': lambda f, x, y: f[:, 0:2],
    'iterate': lambda f, x, y: list(f)[0],
}


@pytest.mark.parametrize('form', list(REJECTED))
def test_forms_outside_the_selection_stay_on_autograd(form):
    with pytest.raises(T.NotLowerable):
        T.trace(REJECTED[form], 2, None, n_out=2)


def test_order_three_and_five_directions_stay_on_autograd():
    def kdv(f, x, t):
        u, v = f[:, 0:1], f[:, 1:2]
        return torch.cat([T.sym_D(T.sym_D(T.sym_D(u, x), x), x) + v, T.sym_D(v, t)], dim=1)
    with pytest.raises(T.NotLowerable, match='order'):
        T.trace(kdv, 2, None, n_out=2)

    def lap5(f, a, b, c, d, e):
        u, v = f[:, 0:1], f[:, 1:2]
        return torch.cat([sum(T.sym_D(u, z) for z in (a, b, c, d, e)), v], dim=1)
    with pytest.raises(T.NotLowerable, match='directions'):
        T.trace(lap5, 5, None, n_out=2)


def test_running_out_of_slots_is_reported_as_slots():
    def eq(f, x, y, z, w):
        cols = torch.split(f, 1, dim=1)
        terms = []
        for q, u in enumerate(cols):
            e = u
            for a in (x, y, z, w):
                e = e + torch.sin(T.sym_D(T.sym_D(u, a), a) * (q + 1.5)) * torch.exp(T.sym_D(u, a) * a) * torch.cos(u * a)
            terms.append(e * torch.tanh(cols[(q + 1) % 4] * e) + torch.sqrt(e * e + 1.0))
        return torch.cat(terms, dim=1)
    with pytest.raises(T.NotLowerable, match='slots|instructions'):
        T.trace(eq, 4, None, n_out=4)


def test_solver_lowers_coupled_problems_and_keeps_constraints_on_autograd():
    from pydens_b200 import Solver, D
    s = Solver(lambda f, x, y: torch.cat([D(f[:, 0:1], x) - f[:, 1:2], D(f[:, 1:2], y)], dim=1), ndims=2,
               layout='fafaf', features=[8, 8, 2], activation='Tanh', device='cpu', backend='auto',
               constraints=[lambda u, x, y: u(torch.tensor([0.5]), torch.tensor([0.5]))[:, 0:1]])
    assert s._traced is not None and s._traced.n_out == 2
    assert s._lower_constraint(0) is None
    s5 = Solver(lambda f, x, y: D(f[:, 0:1], x), ndims=2, layout='fafaf', features=[8, 8, 5], activation='Tanh',
                device='cpu', backend='auto')
    assert s5._traced is None and 'four' in s5._lower_error


def test_plan_refuses_what_the_coupled_kernels_do_not_cover():
    """ build_dev_plan (shared by the library and the host build): k in 2..4, order <= 2, <= 4 directions, the partial block. """
    spec = coupled_spec('navier_stokes2d')
    g = load_golden('navier_stokes2d')
    EC.emul_coupled_step(spec, g['params'], g['points'][:4])
    with pytest.raises(RuntimeError, match='output width'):          # the one-output code still refuses k outputs
        E.emul_step(spec, g['params'], g['points'][:4])
    bad = coupled_spec('navier_stokes2d')
    bad.eq_out[2] = bad.eq_out[1] + 3
    with pytest.raises(RuntimeError, match='eq_out'):
        EC.emul_coupled_step(bad, g['params'], g['points'][:4])
    bad = coupled_spec('navier_stokes2d')
    bad.order = 3
    with pytest.raises(RuntimeError, match='order'):
        EC.emul_coupled_step(bad, g['params'], g['points'][:4])
    bad = coupled_spec('navier_stokes2d')
    bad.widths[bad.n_layers] = 5
    with pytest.raises(RuntimeError, match='output width'):
        EC.emul_coupled_step(bad, g['params'], g['points'][:4])


# ------------------------------------------------------------------------------------------------------------------
# device math (host build) against the reference goldens
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(PC.PROBLEMS))
def test_device_math_matches_reference_goldens(name):
    g = load_golden(name)
    cfg = PC.PROBLEMS[name]
    m, k = cfg['m'], cfg['k']
    assert g['residual'].shape == (g['points'].shape[0], m) and g['u'].shape == (g['points'].shape[0], k)
    spec = coupled_spec(name)
    assert spec.n_params == g['params'].size
    loss, residual, grads = EC.emul_coupled_step(spec, g['params'], g['points'])
    assert abs(loss - float(g['loss'])) <= 1e-5 * abs(float(g['loss']))
    assert rel_l2(residual, folded(g['residual'], m, crit_key(name))) <= 1e-5
    assert rel_l2(grads, g['grads']) <= 1e-4
    for l in range(spec.n_layers):
        n_in, n_out = spec.widths[l], spec.widths[l + 1]
        for off, size in ((spec.w_off[l], n_in * n_out), (spec.b_off[l], n_out)):
            assert rel_l2(grads[off:off + size], g['grads'][off:off + size]) <= 1e-4, (l, off)
    tails = [spec.log_scale_off] + [spec.var_off[i] for i in range(spec.n_vars)]
    for off in tails:
        if PC.has_ic(name) or off != spec.log_scale_off:
            assert abs(grads[off] - g['grads'][off]) <= 1e-4 * max(abs(g['grads'][off]), 1e-3 * np.abs(g['grads']).max()), off
    u = EC.emul_coupled_forward(spec, g['params'], g['points'])
    assert u.shape == g['u'].shape and rel_l2(u, g['u']) <= 1e-5


@pytest.mark.parametrize('name', list(PC.GOLDEN_TRAJ))
def test_emulated_fit_follows_the_reference_fit(name):
    """ The whole loop on the CPU: device math for loss and gradients, the oracle's Adam for optimizer.step(), on the
    batches the reference's own Solver.fit saw. """
    g = load_golden(name)
    niters, batch, lr = int(g['traj_meta'][0]), int(g['traj_meta'][1]), float(g['traj_meta'][2])
    spec = coupled_spec(name)
    params = g['params'].astype(np.float32).copy()
    m, v = np.zeros_like(params), np.zeros_like(params)
    losses = []
    for i in range(niters):
        loss, _, grads = EC.emul_coupled_step(spec, params, PC.make_points(name, batch, seed=1000 + i))
        losses.append(loss)
        adam_step(params, grads, m, v, i + 1, lr=lr)
    losses, ref = np.asarray(losses, dtype=np.float64), g['traj_losses'].astype(np.float64)
    assert np.max(np.abs(losses - ref) / np.maximum(np.abs(ref), 1e-6)) <= 2e-3
    assert np.linalg.norm(params - g['traj_params']) / np.linalg.norm(g['traj_params']) <= 1e-3


# ------------------------------------------------------------------------------------------------------------------
# random coupled problems against the fp64 oracle
# ------------------------------------------------------------------------------------------------------------------
JET_SETS = [(nf, ns) for nf in range(5) for ns in range(nf + 1)]
PICK = {
    'slice': lambda f, k: [f[:, j:j + 1] for j in range(k)],
    'list': lambda f, k: [f[:, [j]] for j in range(k)],
    'ellipsis': lambda f, k: [f[..., j:j + 1] for j in range(k)],
    'split': lambda f, k: list(torch.split(f, 1, dim=1)),
    'chunk': lambda f, k: list(torch.chunk(f, k, dim=1)),
    'method_split': lambda f, k: list(f.split(1, dim=1)),
}
ACTS = ['Tanh', 'Sigmoid', 'SiLU', 'GELU', 'Softplus']


def random_coupled(seed, k=None, jet=None, kind=None, hidden=None, nparams=None, n=None):
    """ A random coupled problem: k outputs, one of the 15 jet sets (axis directions: the first ns carry a second
    derivative), V in the equation and / or the initial condition, dense or residual layout, one of five criteria.
    `k`, `jet` = (nf, ns) and `kind` (criterion) may be fixed by the caller.  So may the hidden widths, the parameter
    columns and the point count; they replace what was drawn after every draw, so a seed draws the same problem
    otherwise.  `hidden`: an int (every hidden layer of the drawn layout) or a list of widths (a dense layout of that
    many layers, the drawn activations in turn). """
    rng = np.random.RandomState(410000 + seed)
    nf, ns = jet if jet is not None else JET_SETS[seed % len(JET_SETS)]
    # k C reserved slots and k C partials: many channels leave room for fewer components in one 192-instruction program
    k_draw = int(rng.randint(2, 2 + max(1, min(3, 24 // (1 + nf + ns) - 1))))
    k = k if k is not None else k_draw
    has_ic = bool(rng.rand() < 0.5)
    ndims = max(nf, 1) + (1 if has_ic and nf == 0 else 0)
    nparams_draw = int(rng.randint(2)) if ndims < 4 else 0
    total = ndims + nparams_draw
    bc = None if rng.rand() < 0.4 else float(np.round(rng.uniform(-0.5, 0.5), 2))
    eq_var, ic_var = bool(rng.rand() < 0.5), bool(has_ic and rng.rand() < 0.5)
    coef = np.round(rng.uniform(0.2, 1.0, size=(k, 6)), 3)
    pick = list(PICK)[int(rng.randint(len(PICK)))]
    width = int(rng.randint(4, 13))
    resnet = bool(rng.rand() < 0.4)
    n_act = 3 if resnet else 2
    acts = [ACTS[int(i)] for i in rng.randint(len(ACTS), size=n_act)]
    layout = 'faR fa fa+ f' if resnet else 'fafaf'
    features = [width] * n_act + [k]
    kind_draw = ['mse', 'l1', 'huber', 'smooth_l1', 'mse_sum'][int(rng.randint(5))]
    kind = kind if kind is not None else kind_draw

    def eq(f, *xs, D, V):
        us = PICK[pick](f, k)
        cols = []
        for j in range(k):
            u, w = us[j], us[(j + 1) % k]
            r = coef[j, 0] * u * w - coef[j, 1] * torch.sin(xs[0])
            for d in range(ns):                          # every component carries every direction's terms
                r = r + coef[j, 2] * D(D(u, xs[d]), xs[d])
            for d in range(ns, nf):
                r = r + coef[j, 3] * D(u, xs[d]) * (w if d == ns else 1.0)
            if eq_var and j == 0:
                r = r + V('c', 0.6) * u
            cols.append(r + coef[j, 4] * torch.tanh(w) if k * (1 + nf + ns) <= 8 else r)
        return torch.cat(cols, dim=1)

    nsp = ndims - 1 if has_ic else ndims
    if not has_ic:
        ic = None
    elif nsp == 0:
        ic = 0.4
    elif ic_var:
        ic = lambda V: (lambda *x: V('a', 0.7) * torch.sin(x[0]) + 0.1)
    else:
        ic = lambda V: (lambda *x: 0.3 * torch.cos(x[0]))
    domain = [(float(np.round(rng.uniform(-1, 0), 2)), float(np.round(rng.uniform(0.5, 2), 2))) for _ in range(ndims)]
    variables = {}
    if eq_var:
        variables['c'] = 0.6
    if ic_var and nsp > 0:
        variables['a'] = 0.7
    n_draw = int(rng.choice([1, 5, 33, 70]))
    log_scale = float(np.round(rng.uniform(-0.3, 0.3), 2))
    # the caller's overrides, after the last draw
    n = n_draw if n is None else n
    if isinstance(hidden, int):
        features = [hidden] * n_act + [k]
    elif hidden is not None:
        acts = [acts[i % n_act] for i in range(len(hidden))]
        layout = 'fa' * len(hidden) + 'f'
        features = list(hidden) + [k]
    if nparams is not None:
        total = ndims + nparams
    nparams = nparams if nparams is not None else nparams_draw
    tag ='k=%d nf=%d ns=%d ic=%s bc=%s %s %s %s %s n=%d' % (k, nf, ns, has_ic, bc, pick, layout, acts, kind, n)
    return dict(eq=eq, k=k, ndims=ndims, nparams=nparams, total=total, bc=bc, ic=ic, domain=domain, features=features,
                acts=acts, layout=layout, variables=dict(sorted(variables.items())), kind=kind, n=n, tag=tag,
                log_scale=log_scale, nf=nf, ns=ns)


def random_setup(seed, dtype=torch.float64, **fixed):
    """ -> (cfg, oracle problem, fp32 params, points, (criterion key, torch criterion), spec); `fixed`: see random_coupled """
    cfg = random_coupled(seed, **fixed)
    holder = {}
    ic = cfg['ic'](lambda n, init: holder['prob'].V(n, init)) if callable(cfg['ic']) else cfg['ic']
    prob = ap.Problem(cfg['eq'], ndims=cfg['ndims'], nparams=cfg['nparams'], initial_condition=ic,
                      boundary_condition=cfg['bc'], domain=cfg['domain'], features=cfg['features'], activation=cfg['acts'],
                      dtype=dtype, variables=cfg['variables'], seed=seed, layout=cfg['layout'])
    holder['prob'] = prob
    with torch.no_grad():
        prob.log_scale.fill_(cfg['log_scale'])
    params = prob.flat_params().numpy().astype(np.float32)
    prob.load_flat(torch.from_numpy(params.astype(np.float64)))
    rng = np.random.RandomState(420000 + seed)
    ranges = list(cfg['domain']) + [(0.0, 1.0)] * cfg['nparams']
    pts = np.concatenate([rng.uniform(lo + 1e-3 * (hi - lo), hi - 1e-3 * (hi - lo), size=(cfg['n'], 1)) for lo, hi in ranges],
                         axis=1).astype(np.float32)
    _, r64, _ = oracle_loss_and_grads(prob, pts.astype(np.float64))
    thr = float(np.float32(np.median(np.abs(r64))))
    kind = cfg['kind']
    red = 'sum' if kind == 'mse_sum' else 'mean'
    key, crit = {'mse': (('mse',), torch.nn.MSELoss()), 'mse_sum': (('mse', 'sum'), torch.nn.MSELoss(reduction='sum')),
                 'l1': (('l1',), torch.nn.L1Loss()),
                 'huber': (('huber', thr), torch.nn.HuberLoss(delta=thr)),
                 'smooth_l1': (('smooth_l1', thr), torch.nn.SmoothL1Loss(beta=thr))}[kind]
    sym_ic = cfg['ic'](sym_V) if callable(cfg['ic']) else cfg['ic']
    nsp = cfg['ndims'] - 1 if cfg['ic'] is not None else cfg['ndims']
    traced = T.trace(lambda u, *xs: cfg['eq'](u, *xs, D=T.sym_D, V=sym_V), cfg['total'], None, initial_condition=sym_ic,
                     ndims_spatial=nsp, criterion=key, n_out=cfg['k'])
    assert (traced.nf, traced.ns) == (cfg['nf'], cfg['ns']), cfg['tag']
    layer_acts = [a.lower() for a in cfg['acts']] + ['none']
    skips = [None, None, 0, None] if cfg['layout'].startswith('faR') else [None] * len(layer_acts)
    spec = N.build_spec([cfg['total']] + cfg['features'], layer_acts, cfg['ndims'], cfg['nparams'], cfg['bc'] is not None,
                        cfg['bc'] if cfg['bc'] is not None else 0.0, cfg['ic'] is not None, cfg['domain'], traced, skips=skips)
    return cfg, prob, params, pts, (key, crit, red, r64, thr), spec


def tolerances(cfg, r64, thr):
    """ The bars of test_systems.py's random systems: relaxed by the cancellation factor of a residual far below its
    O(1) terms, and for the non-smooth criteria by the share of entries within fp32 rounding of a kink. """
    kind = cfg['kind']
    near_kink = np.abs(np.abs(r64) - (0.0 if kind in ('l1', 'mse', 'mse_sum') else thr)) <= 1e-5 * np.maximum(np.abs(r64), thr)
    slack = 1.0 if kind.startswith('mse') else 1.0 + 1e4 * float(near_kink.mean()) * (1.0 if kind == 'l1' else 1e-5)
    cond = max(1.0, 0.05 / max(float(np.sqrt(np.mean(np.square(r64)))), 1e-30))
    return cond, slack


@pytest.mark.parametrize('seed', list(range(225)))
def test_random_coupled_problem_matches_fp64_oracle(seed):
    cfg, prob, params, pts, (key, crit, red, r64, thr), spec = random_setup(seed)
    loss, residual, grads = EC.emul_coupled_step(spec, params, pts)
    weight = float(cfg['n']) if red == 'sum' else 1.0
    ref_loss, ref_res, ref_grads = oracle_loss_and_grads(prob, pts.astype(np.float64), criterion=crit)
    cond, slack = tolerances(cfg, r64, thr)
    tag = cfg['tag']
    assert abs(loss * weight - ref_loss) <= 2e-5 * cond * max(abs(ref_loss), 1e-6), tag
    assert rel_l2(grads * np.float32(weight), ref_grads.numpy()) <= 1e-4 * cond * slack, tag
    if cfg['kind'].startswith('mse'):
        assert rel_l2(residual, folded(ref_res, cfg['k'], key)) <= 2e-5 * cond, tag
    u = EC.emul_coupled_forward(spec, params, pts)
    assert rel_l2(u, prob.predict(pts.astype(np.float64)).reshape(-1, cfg['k'])) <= 1e-5, tag
