""" Constraints that differentiate the solution at their own points (`D(u(t0), t0)`, reference model_torch.py:451-457):
what the tracer lowers and what it leaves to autograd, the programs of constraints without derivatives (unchanged:
digests recorded before derivatives were lowered), every constraint plan on the host build of the device code against
fp64 autograd at the constraint's points, and the persistent kernels' term points (point_step<…, TERMS = true>) in the
equation's jet set.  The GPU side is tests/test_gpu_constraint_derivatives.py. """
import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest
import torch

import problems as P
import emul_harness as E
from helpers import load_golden, oracle_problem, rel_l2
from pydens_b200 import tracer as T, _native as N
from pydens_b200.model import D

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, 'golden')
TERMS_SRC = os.path.join(HERE, 'emul', 'pinn_emul_terms.cpp')
sym_V = lambda n, init=None: T.Sym(T.var(n))          # noqa: E731


def grad_tensor(values):
    return torch.tensor(values, requires_grad=True)


# ------------------------------------------------------------------------------------------------------------------
# the cases: (golden problem, constraint on u, the same expression as an equation of the fp64 oracle, its points)
# ------------------------------------------------------------------------------------------------------------------
def _velocity(u, x):                                   # u'(0) of a one-column problem
    t0 = grad_tensor([0.0])
    return D(u(t0), t0)


FLUX_Y = np.linspace(0.05, 0.95, 16).astype(np.float32)


def _flux(u, x, y):                                    # Neumann data on the face x = 1, 16 points
    x0 = grad_tensor(np.ones(16, dtype=np.float32))
    return D(u(x0, torch.tensor(FLUX_Y)), x0) - 0.3


def _mixed(u, x, y):
    x0, y0 = grad_tensor([0.3, 0.7]), grad_tensor([0.6, 0.2])
    return D(D(u(x0, y0), x0), y0)


def _beam_end(u, x, t):                                # u'' and u''' at the free end x = 1 of the beam
    x0 = grad_tensor([1.0, 1.0, 1.0])
    ux = D(D(u(x0, torch.tensor([0.2, 0.5, 0.9])), x0), x0)
    return ux + 0.5 * D(ux, x0)


def _heat_vars(u, x, t, V=sym_V):                      # V in the constraint; the problem's ic has V too
    x0 = grad_tensor([0.0, 0.0, 1.0])
    return D(u(x0, torch.tensor([0.3, 0.6, 0.8])), x0) * V('src') - V('shift')


CASES = {
    'velocity': ('ode_var', _velocity, lambda u, x, D, V: D(u, x), np.array([[0.0]])),
    'flux': ('poisson2d', _flux, lambda u, x, y, D, V: D(u, x) - 0.3, np.stack([np.ones(16), FLUX_Y], 1)),
    'mixed': ('poisson2d', _mixed, lambda u, x, y, D, V: D(D(u, x), y), np.array([[0.3, 0.6], [0.7, 0.2]])),
    'beam_end': ('beam', _beam_end, lambda u, x, t, D, V: D(D(u, x), x) + 0.5 * D(D(D(u, x), x), x),
                 np.array([[1.0, 0.2], [1.0, 0.5], [1.0, 0.9]])),
    'heat_vars': ('heat1d_icvar', _heat_vars, lambda u, x, t, D, V: D(u, x) * V('src') - V('shift'),
                  np.array([[0.0, 0.3], [0.0, 0.6], [1.0, 0.8]])),
    'mixed_in_layout': ('mixed2d', _mixed, lambda u, x, y, D, V: D(D(u, x), y), np.array([[0.3, 0.6], [0.7, 0.2]])),
}
# case -> (nf, ns, order, in the equation's jet set)
LOWERED = {'velocity': (1, 0, 2, True), 'flux': (2, 2, 2, True), 'mixed': (3, 3, 2, False), 'beam_end': (1, 0, 3, False),
           'heat_vars': (2, 1, 2, True), 'mixed_in_layout': (3, 3, 2, True)}


def _total(name):
    cfg = P.PROBLEMS[name]
    return cfg['ndims'] + cfg['nparams']


def _nsp(name):
    return P.PROBLEMS[name]['ndims'] - 1 if P.has_ic(name) else P.PROBLEMS[name]['ndims']


def trace_case(case, criterion=None, layout=True):
    name, constraint = CASES[case][:2]
    eq = E.traced_problem(name, criterion) if layout else None
    return T.trace_constraint(constraint, _total(name), initial_condition=P.make_ic(name, sym_V), ndims_spatial=_nsp(name),
                              criterion=criterion, layout=eq)


def term_spec(name, tr, criterion=None):
    """ The constraint's plan next to the golden problem's: its network, parameter layout and ansatz. """
    cfg = P.PROBLEMS[name]
    main, main_tr = E.spec_for(name, criterion), E.traced_problem(name, criterion)
    var_offsets = {n: main.var_off[i] for i, n in enumerate(main_tr.var_names)}
    acts, skips = P.layer_plan(name)
    dom = cfg['domain']
    if isinstance(dom[0], (int, float)):
        dom = [tuple(dom)] * cfg['ndims']
    n_layers = len(cfg['features'])
    return main, N.build_spec([_total(name)] + list(cfg['features']), acts, cfg['ndims'], cfg['nparams'], cfg['bc'] is not None,
                              cfg['bc'] if cfg['bc'] is not None else 0.0, P.has_ic(name), dom, tr, var_offsets=var_offsets,
                              w_off=list(main.w_off[:n_layers]), b_off=list(main.b_off[:n_layers]),
                              log_scale_off=main.log_scale_off, n_params=main.n_params, skips=skips)


def oracle(case, params, criterion=None):
    name, _, expr, pts = CASES[case]
    prob = oracle_problem(name, torch.float64, params.astype(np.float64))
    prob.equation = expr
    return prob.loss_and_grads(pts.astype(np.float64), criterion=criterion)


# ------------------------------------------------------------------------------------------------------------------
# lowering
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', list(CASES))
def test_derivative_constraints_lower_with_their_jet_set(case):
    """ nf / ns / order of the plan, and whether it is the equation's jet set (the persistent kernels run only those). """
    name = CASES[case][0]
    tr, args = trace_case(case)
    eq = E.traced_problem(name)
    nf, ns, order, shared = LOWERED[case]
    assert (tr.nf, tr.ns, tr.order) == (nf, ns, order)
    assert ((tr.dirs, tr.dir_vecs, tr.ns) == (eq.dirs, eq.dir_vecs, eq.ns)) == shared
    assert len(args) == _total(name) and not T.leaves(tr.residual, ('coord',))
    own, _ = trace_case(case, layout=False)            # without a layout: the jet set the derivatives call for
    assert own.nf <= tr.nf and own.order == order


def test_constraints_that_stay_on_autograd_are_refused():
    p, q, plain = grad_tensor([0.5]), grad_tensor([0.5]), torch.tensor([0.5])
    refused = {
        'p not among the arguments': lambda u, x, y: D(u(p, 0.5), q),
        'p passed as two columns': lambda u, x, y: D(u(p, p), p),
        'p without requires_grad': lambda u, x, y: D(u(plain, 0.2), plain),
        'D along the batch points': lambda u, x, y: D(u(p, 0.2), x),
        'p outside D': lambda u, x, y: D(u(p, 0.2), p) * p,
        'two model evaluations': lambda u, x, y: D(u(p, 0.2), p) - u(0.1, 0.2),
        'the batch points': lambda u, x, y: D(u(p, 0.2), p) * x,
        'order 5': lambda u, x, y: D(D(D(D(D(u(p, 0.2), p), p), p), p), p),
    }
    for why, c in refused.items():
        with pytest.raises(T.NotLowerable):
            T.trace_constraint(c, 2, layout=E.traced_problem('poisson2d'))
            pytest.fail(why)


def test_a_derivative_the_equation_lacks_gets_its_own_jet_set():
    """ u_y on a problem whose equation differentiates x only: own jet set, not the equation's. """
    eq = T.trace(lambda u, x, y: T.sym_D(T.sym_D(u, x), x) - y, 2, None)
    y0 = grad_tensor([0.5])
    tr, _ = T.trace_constraint(lambda u, x, y: D(u(0.2, y0), y0), 2, layout=eq)
    assert tr.dirs == [1] and tr.ns == 0 and eq.dirs == [0]


VALUE_CONSTRAINTS = {
    'point': lambda u, *xs: u(*[torch.tensor([0.5])] * len(xs)),
    'square': lambda u, *xs: u(*[torch.tensor([0.25, 0.75])] * len(xs)) ** 2 - 0.3,
    'var': lambda u, *xs: torch.sin(u(*[torch.tensor([0.1, 0.4, 0.9])] * len(xs))) * sym_V('amp') - 1.0,
}
DIGEST_PROBLEMS = ['poisson2d', 'ode_var', 'heat1d_icvar', 'beam', 'mixed2d']
DIGEST_CRITERIA = [None, ('l1',), ('huber', 0.5), ('mse', 'sum')]


def _digest(tr):
    parts = [None if prog is None else ([list(i) for i in prog.instrs], list(prog.outs), prog.n_slots)
             for prog in (tr.eq_prog, tr.ic_prog)]
    parts.append((tr.dirs, tr.dir_vecs, tr.ns, tr.var_names, tr.order, tr.n_slots))
    return hashlib.sha256(json.dumps(parts).encode()).hexdigest()


def value_constraint_digests(layout):
    got = {}
    for name in DIGEST_PROBLEMS:
        for cname, c in VALUE_CONSTRAINTS.items():
            if cname == 'var' and name != 'heat1d_icvar':
                continue
            for key in DIGEST_CRITERIA:
                kw = dict(layout=E.traced_problem(name, key)) if layout else {}
                tr, _ = T.trace_constraint(c, _total(name), initial_condition=P.make_ic(name, sym_V),
                                           ndims_spatial=_nsp(name), criterion=key, **kw)
                got['%s|%s|%s' % (name, cname, key)] = _digest(tr)
    return got


def test_constraints_without_derivatives_trace_to_the_programs_they_had():
    """ C = 1 and the same program bytes as before derivatives were lowered (digests recorded then), with or without
    the equation's jet set on offer. """
    with open(os.path.join(GOLDEN, 'constraint_program_digests.json')) as fh:
        want = json.load(fh)
    assert value_constraint_digests(layout=True) == want


# ------------------------------------------------------------------------------------------------------------------
# the stepwise plan on the host build, against fp64 autograd at the constraint's points
# ------------------------------------------------------------------------------------------------------------------
def _criteria():
    return {'mse': (None, None), 'huber': (('huber', 0.05), torch.nn.HuberLoss(delta=0.05))}


@pytest.mark.parametrize('crit', ['mse', 'huber'])
@pytest.mark.parametrize('case', list(CASES))
def test_constraint_plan_matches_fp64_autograd(case, crit):
    """ Loss, residual and every gradient tensor — weights, biases, log_scale and the variables. """
    key, torch_crit = _criteria()[crit]
    name, _, _, pts = CASES[case]
    g = load_golden(name)
    tr, _ = trace_case(case, key)
    _, spec = term_spec(name, tr, key)
    loss, res, grads = E.emul_step(spec, g['params'], pts.astype(np.float32))
    l64, r64, g64 = oracle(case, g['params'], torch_crit)
    assert abs(loss - l64) <= 2e-5 * abs(l64) + 1e-9
    assert rel_l2(res, r64) <= 2e-5 or crit != 'mse'
    g64 = g64.numpy()
    for off, n in _tensor_spans(name, spec):
        assert rel_l2(grads[off:off + n], g64[off:off + n]) <= 1e-4 or np.abs(g64[off:off + n]).max() < 1e-7, (off, n)


def _tensor_spans(name, spec):
    """ (offset, length) of every parameter tensor in the flat layout: W_l, b_l, log_scale, each variable. """
    widths = [_total(name)] + list(P.PROBLEMS[name]['features'])
    spans = []
    for l in range(len(widths) - 1):
        spans += [(spec.w_off[l], widths[l] * widths[l + 1]), (spec.b_off[l], widths[l + 1])]
    spans.append((spec.log_scale_off, 1))
    spans += [(spec.var_off[i], 1) for i in range(spec.n_vars)]
    return spans


def test_sum_reduction_weights_each_constraint_point_by_one():
    """ MSELoss(reduction='sum'): the same program, point weight 1 instead of 1 / n. """
    name = 'poisson2d'
    g = load_golden(name)
    tr, _ = trace_case('flux', ('mse', 'sum'))
    _, spec = term_spec(name, tr, ('mse', 'sum'))
    pts = CASES['flux'][3]
    loss, _, grads = E.emul_step(spec, g['params'], pts.astype(np.float32))
    l64, _, g64 = oracle('flux', g['params'], torch.nn.MSELoss(reduction='sum'))
    n = pts.shape[0]
    assert abs(loss * n - l64) <= 2e-5 * abs(l64)
    assert rel_l2(grads * n, g64.numpy()) <= 1e-4


# ------------------------------------------------------------------------------------------------------------------
# the persistent kernels' term points, in the equation's jet set
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def terms_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('terms') / 'libterms.so')
    subprocess.check_call(['g++', '-O2', '-mfma', '-std=c++17', '-shared', '-fPIC', '-x', 'c++', '-Wno-unknown-pragmas',
                           '-o', out, TERMS_SRC])
    return C.CDLL(out)


def term_step(lib, main, spec, params, pts, weight):
    params = np.ascontiguousarray(params, dtype=np.float32)
    pts = np.ascontiguousarray(pts, dtype=np.float32)
    out = np.zeros(main.n_params + 4, dtype=np.float32)
    res = np.zeros(pts.shape[0], dtype=np.float32)
    msg = C.create_string_buffer(256)
    rc = lib.emul_term_step(C.byref(main), C.byref(spec), params.ctypes.data_as(C.c_void_p), pts.ctypes.data_as(C.c_void_p),
                            C.c_longlong(pts.shape[0]), C.c_float(weight), out.ctypes.data_as(C.c_void_p),
                            res.ctypes.data_as(C.c_void_p), msg, 256)
    assert rc == 0, msg.value
    return float(out[main.n_params]), res, out[:main.n_params]


SHARED = [c for c in CASES if LOWERED[c][3]]


@pytest.mark.parametrize('crit', ['mse', 'huber'])
@pytest.mark.parametrize('case', SHARED)
def test_term_points_in_the_equation_jet_set_match_fp64_autograd(terms_lib, case, crit):
    """ point_step<…, TERMS> at a term point: the term's program on every channel of the equation's jet, its own
    weight, seeds on every channel, the initial condition's variables — against fp64 autograd, and equal to the
    stepwise plan (the same per-point code) up to summation order. """
    key, torch_crit = _criteria()[crit]
    name, _, _, pts = CASES[case]
    g = load_golden(name)
    tr, _ = trace_case(case, key)
    main, spec = term_spec(name, tr, key)
    n = pts.shape[0]
    loss, res, grads = term_step(terms_lib, main, spec, g['params'], pts, 1.0 / n)
    l64, r64, g64 = oracle(case, g['params'], torch_crit)
    assert abs(loss - l64) <= 2e-5 * abs(l64) + 1e-9
    g64 = g64.numpy()
    for off, m in _tensor_spans(name, main):
        assert rel_l2(grads[off:off + m], g64[off:off + m]) <= 1e-4 or np.abs(g64[off:off + m]).max() < 1e-7, (off, m)
    sl, sres, sgrads = E.emul_step(spec, g['params'], pts.astype(np.float32))
    np.testing.assert_allclose(res, sres, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(grads, sgrads, rtol=1e-4, atol=1e-6)
    l1, _, g1 = term_step(terms_lib, main, spec, g['params'], pts, 1.0)        # reduction='sum': weight 1
    assert abs(l1 - loss * n) <= 1e-5 * abs(l1) + 1e-9


def test_value_terms_keep_their_single_channel(terms_lib):
    """ A constraint without derivatives next to a plan with a jet set: its program reads slot 0 only, seeds only u. """
    name = 'heat1d_icvar'
    g = load_golden(name)
    tr, _ = T.trace_constraint(VALUE_CONSTRAINTS['var'], 2, initial_condition=P.make_ic(name, sym_V), ndims_spatial=1,
                               layout=E.traced_problem(name))
    assert tr.nf == 0
    main, spec = term_spec(name, tr)
    pts = np.array([[0.1, 0.1], [0.4, 0.4], [0.9, 0.9]], dtype=np.float32)
    loss, res, grads = term_step(terms_lib, main, spec, g['params'], pts, 1.0 / 3)
    sl, sres, sgrads = E.emul_step(spec, g['params'], pts)
    assert abs(loss - sl) <= 1e-6 * abs(sl)
    np.testing.assert_allclose(grads, sgrads, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize('case', [c for c in CASES if not LOWERED[c][3]])
def test_a_term_plan_with_another_jet_set_is_refused(terms_lib, case):
    """ build_dev_term — pinn_multi_step_terms' check — takes no directions or the plan's, nothing else. """
    name = CASES[case][0]
    tr, _ = trace_case(case)
    main, spec = term_spec(name, tr)
    msg = C.create_string_buffer(256)
    assert terms_lib.emul_term_check(C.byref(main), C.byref(spec), msg, 256) == N.E_INVALID
    assert b'derivative directions' in msg.value
    shared, _ = trace_case('flux')
    main, spec = term_spec('poisson2d', shared)
    assert terms_lib.emul_term_check(C.byref(main), C.byref(spec), msg, 256) == 0
