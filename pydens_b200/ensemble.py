""" `fit_ensemble` — train several Solvers of one problem side by side in the persistent multi-step kernels.

People who fit small problems rarely fit just one: they run several seeds, sweep the initial value of a `V(...)`
variable, or solve one equation for many values of a frozen coefficient.  Each such fit alone runs on one CTA or one
cluster of at most 8 CTAs; `fit_ensemble` puts up to PINN_MAX_MEMBERS of them into one launch
(pinn_multi_step_ensemble), one CTA or cluster per member.  It means exactly "call `s.fit(...)` on every solver": every
member keeps its own seed, optimizer state, frozen mask, loss list and step counter, and its result is bit-identical to
its solo fit.  Each member may also take its own Adam hyper-parameters (a learning-rate sweep: `lr=[...]`), which the
kernels read from the member's row of the table (pinn_multi_step_ensemble_adam).  L-BFGS fits whose solo fits run in
the cluster kernel go to its L-BFGS form the same way (pinn_lbfgs_multi_ensemble), each with its own lr.
"""
import warnings

import numpy as np
import torch
from torch import nn

from . import _native
from .engine import (_AUTO_PERSISTENT_STEPS, _dist, adam_steps_equal, auto_persistent, plain_adam, run_lbfgs_persistent,
                     run_persistent, sampler_columns)

# what each part of the problem's spec describes, for the error that names the difference between two members
_SPEC_PARTS = (
    ('network', ('n_layers', 'widths', 'act', 'skip_src', 'w_off', 'b_off', 'n_params', 'log_scale_off')),
    ('domain', ('ndims', 'nparams', 'dom_lo', 'dom_hi')),
    ('ansatz', ('has_bc', 'has_ic', 'bc_value', 'n_ic', 'ic_prog', 'ic_out', 'ic_has_vars')),
    ('equation program', ('abi_version', 'order', 'nf', 'ns', 'dir_col', 'dir_vec', 'n_eq', 'eq_prog', 'eq_out',
                          'n_slots', 'n_vars', 'var_off')),
)


def spec_difference(a, b):
    """ None when the two PinnSpecs are byte-identical, else the part that differs: 'network (widths)', ... """
    raw_a, raw_b = bytes(a), bytes(b)
    if raw_a == raw_b:
        return None
    for part, fields in _SPEC_PARTS:
        for name in fields:
            f = getattr(_native.PinnSpec, name)
            if raw_a[f.offset:f.offset + f.size] != raw_b[f.offset:f.offset + f.size]:
                return '%s (%s)' % (part, name)
    return 'spec padding'


def check_members(solvers):
    """ The solvers of an ensemble: at least one, each once, all on one device.  Raises ValueError. """
    if not solvers:
        raise ValueError('fit_ensemble: no solvers')
    seen = {}
    for j, s in enumerate(solvers):
        if id(s) in seen:
            raise ValueError('fit_ensemble: solvers %d and %d are the same Solver' % (seen[id(s)], j))
        seen[id(s)] = j
        if s.device != solvers[0].device:
            raise ValueError('fit_ensemble: solver %d is on %s, solver 0 on %s' % (j, s.device, solvers[0].device))


def member_samplers(sampler, n):
    """ One sampler per member: a list of n samplers, or the one sampler shared by all. """
    if isinstance(sampler, (list, tuple)):
        if len(sampler) != n:
            raise ValueError('fit_ensemble: %d samplers for %d solvers' % (len(sampler), n))
        return list(sampler)
    return [sampler] * n


def _per_member(v):
    return isinstance(v, (list, tuple)) or (isinstance(v, np.ndarray) and v.ndim > 0)


def member_hyper(n, lr, kwargs):
    """ Each member's (lr, optimizer kwargs): `lr`, `eps` and `weight_decay` are one value for all or a sequence of n,
    `betas` one pair for all or a sequence of n pairs.  Raises ValueError for a sequence of another length. """
    def spread(name, v, pairs=False):
        if not _per_member(v) or (pairs and not (len(v) and _per_member(v[0]))):
            return [v] * n
        if len(v) != n:
            raise ValueError('fit_ensemble: %d values of %s for %d solvers' % (len(v), name, n))
        return list(v)
    kws = [dict(kwargs) for _ in range(n)]
    for name in ('betas', 'eps', 'weight_decay'):
        if name in kwargs:
            for kw, v in zip(kws, spread(name, kwargs[name], pairs=name == 'betas')):
                kw[name] = v
    return spread('lr', lr), kws


def fit_ensemble(solvers, niters, batch_size, sampler=None, loss_terms='equation', optimizer='Adam',
                 criterion=nn.MSELoss(), lr=0.005, steps_per_launch=None, **kwargs):
    """ `s.fit(niters, batch_size, sampler, loss_terms, optimizer, criterion, lr, ...)` for every solver in `solvers`,
    in one persistent launch per `steps_per_launch` steps for all of them when each fit is one that `Solver.fit` sends
    to the persistent multi-step kernels by itself (or with steps_per_launch): plain Adam, one device, the equation
    term, fused constraints, a batch the kernels take.  L-BFGS fits (optimizer='LBFGS') run together in the L-BFGS form
    of the cluster kernel when each member's solo fit runs there and the members share every setting but lr.  The solvers must share the problem byte for byte (equation,
    network, domain, ansatz, constraints); they differ in their parameters, seeds, optimizer states and frozen masks.

    sampler   None, one sampler shared by all members, or a list with one per member.  In-kernel samplers draw each
              member's batch from its own seed; a shared host sampler gives each member its batches in member order,
              launch by launch.
    lr        one learning rate, or a sequence with one per member; so are `eps` and `weight_decay` among the optimizer
              kwargs, and `betas` is one pair or a sequence of one pair per member.  Member j then fits as
              `s.fit(..., lr=lr[j], betas=betas[j], ...)`, and its optimizer keeps its own settings for a later
              `fit(optimizer=None)`.  With optimizer=None every member keeps its existing optimizer, whatever its
              settings.
    Anything the persistent path cannot take fits the solvers one after another with their own `fit`, after one
    UserWarning giving the reason; decoupled weight decay (decoupled_weight_decay=True with weight_decay > 0) is one
    such fit, it runs on torch's Adam.  Raises ValueError for the same Solver twice, solvers on different devices,
    solvers whose problems differ, or a per-member sequence whose length is not the number of solvers.
    """
    solvers = list(solvers)
    check_members(solvers)
    samplers = member_samplers(sampler, len(solvers))
    lrs, kws = member_hyper(len(solvers), lr, kwargs)
    loss_terms = tuple(loss_terms) if isinstance(loss_terms, (tuple, list)) else (loss_terms,)
    why = None
    if niters > 0:
        why = _fit_together(solvers, niters, batch_size, samplers, loss_terms, optimizer, criterion, lr,
                            steps_per_launch, kwargs)
        if why is None:
            return
        warnings.warn('pydens_b200.fit_ensemble: fitting the solvers one after another (%s)' % why, UserWarning,
                      stacklevel=2)
    for s, smp, lr_j, kw in zip(solvers, samplers, lrs, kws):
        if steps_per_launch is not None:
            kw['steps_per_launch'] = steps_per_launch
        s.fit(niters, batch_size, smp, list(loss_terms), optimizer, criterion, lr_j, **kw)


def _fit_together(solvers, niters, batch_size, samplers, loss_terms, optimizer, criterion, lr, steps_per_launch, kwargs):
    """ The ensemble fit, each member with the optimizer of its own values of `lr` and `kwargs` (member_hyper), or the
    reason it cannot run (nothing has been trained then). """
    if _dist() is not None:
        return 'torch.distributed runs several ranks'
    engines = []
    for j, s in enumerate(solvers):
        ok, why = s._fused_possible(criterion, loss_terms)
        if not ok:
            return 'solver %d: %s' % (j, why)
        eng = s._get_engine()
        if eng is None:
            return 'solver %d: %s' % (j, s._lower_error)
        engines.append(eng)
    for j, eng in enumerate(engines[1:], 1):
        diff = spec_difference(engines[0].spec, eng.spec)
        if diff is not None:
            raise ValueError('fit_ensemble: solver %d differs from solver 0 in its %s' % (j, diff))
    e0 = engines[0]
    k = int(steps_per_launch or 0)
    if k <= 0:                                            # the rule of FusedEngine.fit for tiny batches
        if not auto_persistent(niters, batch_size, e0.info):
            return ('a solo fit of batch %d x %d steps does not take the persistent kernels by itself '
                    '(pass steps_per_launch)' % (batch_size, niters))
        k = _AUTO_PERSISTENT_STEPS
    if batch_size <= 0:
        return 'batch_size %d' % batch_size
    terms = [eng._persistent_terms(loss_terms, batch_size) for eng in engines]
    if any(t is None for t in terms):
        return ('the constraints do not all run fused (at most %d, with %d points in all), or batch + constraint points '
                'exceed %d' % (_native.MAX_TERMS, _native.MAX_TERM_POINTS, e0.lib.pinn_multi_step_max_points(e0.plan)))
    for j, t in enumerate(terms[1:], 1):
        for i, (a, b) in enumerate(zip(terms[0], t)):
            diff = spec_difference(a['spec'], b['spec'])
            if diff is None and a['host_points'].numpy().tobytes() != b['host_points'].numpy().tobytes():
                diff = 'points'
            if diff is not None:
                raise ValueError('fit_ensemble: solver %d differs from solver 0 in constraint %d: %s' % (j, i, diff))
    total = solvers[0].model.total
    if len({sampler_columns(smp, total)[0] for smp in samplers}) > 1:
        return 'the members\' samplers differ in their in-kernel columns, or some sample on the host'
    opts = [eng._optimizer_for(optimizer, lr_j, kw)[0]
            for eng, lr_j, kw in zip(engines, *member_hyper(len(solvers), lr, kwargs))]
    if all(type(opt) is torch.optim.LBFGS and len(opt.param_groups) == 1 for opt in opts):
        return _fit_lbfgs_together(engines, opts, samplers, loss_terms, niters, batch_size, k, int(steps_per_launch or 0))
    for opt in opts:
        if not plain_adam(opt):
            return ('the optimizer is not plain torch.optim.Adam with one parameter group and L2 weight decay '
                    '(decoupled weight decay runs on torch\'s Adam)')
        if not adam_steps_equal(opt):
            return 'the optimizer has taken different numbers of steps for different parameters'
    return run_persistent(engines, opts, samplers, terms[0], niters, batch_size, k, table=True)


# the settings of torch.optim.LBFGS the members of one launch share (lr is each member's own)
_LBFGS_SHARED = ('max_iter', 'max_eval', 'tolerance_grad', 'tolerance_change', 'history_size', 'line_search_fn')


def _fit_lbfgs_together(engines, opts, samplers, loss_terms, niters, batch_size, k, steps_per_launch):
    """ The L-BFGS ensemble fit in the L-BFGS form of the cluster kernel (run_lbfgs_persistent), when each member's
    solo fit would run there, or the reason it cannot (nothing has been trained then). """
    for j, (eng, opt) in enumerate(zip(engines, opts)):
        if eng._lbfgs_persistent_terms(niters, batch_size, loss_terms, opt, steps_per_launch) is None:
            return 'solver %d: its L-BFGS fit does not run in the cluster kernel' % j
        g, g0 = opt.param_groups[0], opts[0].param_groups[0]
        diff = [name for name in _LBFGS_SHARED if g[name] != g0[name]]
        if diff:
            return 'solver %d: its L-BFGS settings differ from solver 0\'s in %s' % (j, ', '.join(diff))
    terms = engines[0]._persistent_terms(loss_terms, batch_size)
    return run_lbfgs_persistent(engines, opts, samplers, terms, niters, batch_size, k, table=True)

