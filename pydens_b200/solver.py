""" `Solver` — the pydens user API (reference pydens/model_torch.py:191-487) on the H100 engine.

Same constructor, `fit`, `predict`, `reshape_and_concat`, attributes (`model`, `losses`, `optimizer`,
`ctx`, `equation`, `constraints`).  What changes is the body of the training loop: where the
reference samples on the host, builds a double-backward autograd graph and calls `loss.backward()`
(model_torch.py:430-460), `fit` here issues ONE CUDA kernel per step through the C ABI
(include/pinn_b200.h: pinn_step), then the (torch) optimizer step — captured together in a CUDA graph
so the Python loop only replays it.

Additions to the reference signature (keyword-only, all optional):
    Solver(..., device=None, backend='auto', seed=None)
    backend: 'auto'  fused kernel when the equation lowers, else the autograd path with a warning
             'fused' fused kernel or raise
             'torch' always the autograd path (device-aware restatement of the reference loop)
"""
import os
import warnings
from contextvars import copy_context

import numpy as np
import torch
from torch import nn

from . import _native, tracer
from .model import ConvBlockModel, TorchModel, current_model, _tracing, D, V   # noqa: F401  (re-exported)

try:                                           # progress bar like the reference (model_torch.py:426)
    from tqdm import tqdm as _tqdm
except ImportError:                            # pragma: no cover
    _tqdm = None

_GRAPH_MIN_ITERS = 8


def _progress(n):
    if _tqdm is None or os.environ.get('PYDENS_B200_PROGRESS', '') == '0':
        return range(n)
    return _tqdm(range(n), mininterval=0.5, disable=None)


class Solver:
    r""" Solver of differential equations with neural networks (PINN / DGM).

    Parameters follow the reference (`pydens.Solver`): `equation` is a callable built from the tokens
    `D` (differentiation) and `V` (trainable variable) and torch / numpy math, e.g.

        def pde(f, x, y):
            return D(D(f, x), x) + D(D(f, y), y) - 5 * torch.sin(np.pi * (x + y))

        solver = Solver(pde, ndims=2, boundary_condition=1, layout='fa fa fa f',
                        activation='Tanh', units=[10, 12, 15, 1])
        solver.fit(batch_size=100, niters=1500)

    `ndims` counts variables, `nparams` parameters with uncertainty (fed to the network, not
    differentiated), `initial_condition` (callable or number) / `boundary_condition` (number) /
    `domain` configure the ansatz, `constraints` are extra loss terms, remaining kwargs configure the
    model (`layout`, `features`/`units`, `activation`).
    """

    def __init__(self, equation, ndims, initial_condition=None, boundary_condition=None, domain=(0, 1),
                 nparams=0, model=ConvBlockModel, constraints=None, device=None, backend='auto', seed=None,
                 **kwargs):
        if backend not in ('auto', 'fused', 'torch'):
            raise ValueError("backend must be 'auto', 'fused' or 'torch'")
        self.equation = equation
        if constraints is None:
            self.constraints = ()
        elif isinstance(constraints, (tuple, list)):
            self.constraints = constraints
        else:
            self.constraints = (constraints,)
        self.losses = []
        self.optimizer = None
        self.backend = backend
        if device is None:
            device = 'cuda' if torch.cuda.is_available() else 'cpu'
        self.device = torch.device(device)
        if self.device.type == 'cuda' and self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.seed = int(seed) if seed is not None else int(torch.initial_seed() & 0x7fffffffffffffff)

        self.model = model(**kwargs, ndims=ndims, initial_condition=initial_condition,
                           boundary_condition=boundary_condition, domain=domain, nparams=nparams)
        self.model.to(self.device)

        current_model.set(self.model)
        self.ctx = copy_context()

        # one throw-away run so that every V() of the equation exists before an optimizer is built
        # (reference :319-325)
        xs = [torch.rand((1, 1), device=self.device).requires_grad_() for _ in range(self.model.total)]
        u_hat = self.ctx.run(self.model, self.reshape_and_concat(xs))
        _ = self.ctx.run(self.equation, u_hat, *xs)

        self._engine = None
        self._traced = None
        self._crit_key = ('mse',)                         # criterion the traced programs (and the engine) are built for
        self._traced_constraints = {}                     # num -> (TracedEquation, points [n, total]) or None
        self._lower_error = None
        self._warned = False
        if backend != 'torch':
            self._try_lower()
            if backend == 'fused' and self._traced is None:
                raise RuntimeError('backend="fused": %s' % self._lower_error)

    # ------------------------------------------------------------------------------------------
    # lowering to the fused engine
    # ------------------------------------------------------------------------------------------
    def _try_lower(self):
        model = self.model
        try:
            if not isinstance(model, ConvBlockModel) or type(model).forward is not ConvBlockModel.forward \
                    or type(model).anzatc is not TorchModel.anzatc:
                raise tracer.NotLowerable('custom model class')
            chain = model.conv_block.dense_chain()
            if chain is None:
                raise tracer.NotLowerable('layout %r is not a plain dense chain' % model.conv_block.layout)
            if chain[-1][1] != 'none' or chain[-1][0].out_features != 1:
                raise tracer.NotLowerable('network must end with a dense layer of one unit')
            if chain[-1][2] is not None:
                raise tracer.NotLowerable('skip connection into the output layer')
            if any(c[0].bias is None for c in chain) or len(chain) > _native.MAX_LAYERS:
                raise tracer.NotLowerable('unsupported dense layers')
            if model.total > _native.MAX_DIMS:
                raise tracer.NotLowerable('more than %d point columns' % _native.MAX_DIMS)
            bc = model.boundary_condition
            if bc is not None and not isinstance(bc, (int, float)):
                raise tracer.NotLowerable('boundary_condition must be a number')

            def run(fn, *args):
                def call():
                    token = _tracing.set(True)
                    try:
                        return fn(*args)
                    finally:
                        _tracing.reset(token)
                return self.ctx.run(call)

            ic = model.raw_initial_condition
            self._traced = tracer.trace(self.equation, model.total, None, initial_condition=ic,
                                        ndims_spatial=model.ndims_spatial, run=run, criterion=self._crit_key)
            self._chain = chain
        except tracer.NotLowerable as exc:
            self._traced = None
            self._lower_error = str(exc)
        except Exception as exc:                          # noqa: BLE001
            # anything else the symbolic proxies choke on (a TypeError from an operator they do not define, an
            # IndexError from user code that indexes its argument ...): the reference accepts such equations, so
            # under backend='auto' they simply stay on autograd; backend='fused' reports the reason
            self._traced = None
            self._lower_error = '%s while tracing: %s' % (type(exc).__name__, exc)

    def _tracing_run(self, fn, *args):
        def call():
            token = _tracing.set(True)
            try:
                return fn(*args)
            finally:
                _tracing.reset(token)
        return self.ctx.run(call)

    def _lower_constraint(self, num):
        """ (traced constraint, its points as a [n, total] fp32 tensor) if constraint `num` can run as a fused
        launch — one model evaluation at fixed points, combined pointwise — else None (autograd adds it). """
        if num not in self._traced_constraints:
            lowered = None
            if self._traced is not None and os.environ.get('PYDENS_B200_FUSED_CONSTRAINTS') != '0':
                model = self.model
                try:
                    traced, args = tracer.trace_constraint(self.constraints[num], model.total,
                                                           initial_condition=model.raw_initial_condition,
                                                           ndims_spatial=model.ndims_spatial, run=self._tracing_run,
                                                           criterion=self._crit_key)
                    pts = self.reshape_and_concat(args).detach().to(torch.float32)
                    if pts.dim() != 2 or pts.shape[1] != model.total or pts.shape[0] < 1:
                        raise tracer.NotLowerable('constraint points do not have %d columns' % model.total)
                    if not set(traced.var_names) <= set(self._traced.var_names):
                        raise tracer.NotLowerable('constraint introduces new variables')
                    lowered = (traced, pts.contiguous())
                except (tracer.NotLowerable, TypeError, ValueError, RuntimeError, IndexError):
                    lowered = None
            self._traced_constraints[num] = lowered
        return self._traced_constraints[num]

    def _get_engine(self):
        if self._engine is None:
            from .engine import FusedEngine
            try:
                self._engine = FusedEngine(self)
            except _native.NativeError as exc:
                # the library understood the request but its kernels do not cover it (e.g. a network whose
                # weights do not fit shared memory): that is a lowering failure, not a crash
                if exc.code == _native.E_UNSUPPORTED and self.backend == 'auto':
                    self._traced, self._lower_error = None, str(exc)
                    return None
                raise
            except _native.LibraryMissing as exc:
                # fresh clone without build(): backend='auto' keeps working on autograd (loudly, fit() warns with
                # this reason); backend='fused' must fail
                if self.backend == 'auto':
                    self._traced, self._lower_error = None, str(exc)
                    return None
                raise
        return self._engine

    @staticmethod
    def _criterion_key(criterion):
        """ The criteria the fused path trains with (reference :448 `criterion(residual, zeros)`): MSELoss natively;
        L1Loss, HuberLoss and SmoothL1Loss through a residual transform (tracer.apply_criterion).  None: autograd. """
        functional = {nn.functional.mse_loss: ('mse',), nn.functional.l1_loss: ('l1',),
                      nn.functional.huber_loss: ('huber', 1.0), nn.functional.smooth_l1_loss: ('smooth_l1', 1.0)}
        try:
            if criterion in functional:                   # the plain functions, with their defaults (mean reduction)
                return functional[criterion]
        except TypeError:                                 # unhashable callable
            pass
        reduction = getattr(criterion, 'reduction', None)
        if reduction not in ('mean', 'sum'):
            return None
        tail = ('sum',) if reduction == 'sum' else ()     # 'sum': the same kernels with weight 1 instead of 1 / batch_size
        kind = type(criterion)
        if kind is nn.MSELoss:
            return ('mse',) + tail
        if kind is nn.L1Loss:
            return ('l1',) + tail
        if kind is nn.HuberLoss and float(criterion.delta) > 0:
            return ('huber', float(criterion.delta)) + tail
        if kind is nn.SmoothL1Loss and float(criterion.beta) >= 0:
            return (('smooth_l1', float(criterion.beta)) if float(criterion.beta) > 0 else ('l1',)) + tail
        return None

    def _switch_criterion(self, key):
        """ Re-trace equation and constraints for another criterion; the engine (plans, graphs, optimizer state) is
        rebuilt on the next use — parameters keep their values. """
        self._release_engine()
        self._crit_key = key
        self._traced_constraints = {}
        self._lower_error = None
        self._try_lower()

    def _fused_possible(self, criterion, loss_terms):
        if self.backend == 'torch':
            return False, 'backend="torch"'
        if self.device.type != 'cuda':
            return False, 'device is %s' % self.device
        key = self._criterion_key(criterion)
        if key is None:
            return False, 'criterion is not MSELoss / L1Loss / HuberLoss / SmoothL1Loss (mean or sum reduction)'
        if key != self._crit_key:
            self._switch_criterion(key)
        if self._traced is None:
            return False, self._lower_error
        if 'equation' not in loss_terms and not self._constraint_numbers(loss_terms):
            return False, 'no loss term'                  # the autograd path fails on it as the reference does
        return True, None

    # ------------------------------------------------------------------------------------------
    # reference API
    # ------------------------------------------------------------------------------------------
    @classmethod
    def reshape_and_concat(cls, tensors):
        """ Cast every element (number, ndarray, list/tuple, tensor) to an (N x 1) tensor — numbers and
        wrong-sized arrays are tiled to the longest element — and concatenate to (N x D).
        Same contract as the reference (:328-362). """
        items = list(tensors)
        lengths = [int(np.prod(t.shape)) for t in items if isinstance(t, (np.ndarray, torch.Tensor))]
        lengths += [int(np.prod(np.array(t).shape)) for t in items if isinstance(t, (tuple, list))]
        n = max(lengths) if lengths else 1
        device = next((t.device for t in items if isinstance(t, torch.Tensor)), None)
        cols = []
        for t in items:
            if isinstance(t, torch.Tensor):
                col = t.view(-1, 1)
            elif isinstance(t, (int, float)):
                col = torch.full((n, 1), float(t), dtype=torch.float32)
            elif isinstance(t, np.ndarray):
                if t.size != n:
                    t = np.tile(t.squeeze()[0] if t.ndim and t.size > 1 else t.reshape(-1)[0], (n, 1))
                col = torch.tensor(np.asarray(t, dtype=np.float32).reshape(n, 1))
            elif isinstance(t, (list, tuple)):
                col = torch.tensor(t, dtype=torch.float32).view(-1, 1)
            else:
                raise TypeError('cannot use %s as a point column' % type(t).__name__)
            cols.append(col)
        if device is not None:
            cols = [c.to(device) for c in cols]
        return torch.cat(cols, dim=1)

    def fit(self, niters, batch_size, sampler=None, loss_terms='equation', optimizer='Adam',
            criterion=nn.MSELoss(), lr=0.005, **kwargs):
        """ Train the model: `niters` optimizer steps on batches of `batch_size` sampled points.

        sampler     object with `.sample(size)`; None = U[0,1) on every column (reference :431).
                    Samplers from pydens_b200.sampler made of independent uniform / normal columns run
                    in-kernel; anything else is sampled on the host and copied per step.
        loss_terms  'equation' and/or 'constraint_{k}' (reference :382-389).
        optimizer   name from torch.optim; None re-uses the existing optimizer (reference :391-393).
        criterion   nn.MSELoss() (default), nn.L1Loss(), nn.HuberLoss(delta), nn.SmoothL1Loss(beta), mean or sum reduction,
                    train on the fused kernels (switching the criterion between fits rebuilds the engine); anything
                    else runs on the autograd path.
        kwargs      forwarded to the optimizer constructor, except
                    steps_per_launch=k  (fused path, small batches): k whole optimizer steps — Adam included — per
                    launch of a persistent kernel.  Batches of at most 1024 points (the launch-bound regime of the
                    README example, batch_size=100, niters=1500) take this path by themselves, 50 steps per launch,
                    whenever the optimizer is plain Adam, there is one device and no constraint term
                    (PYDENS_B200_AUTO_PERSISTENT=0 keeps one launch per step).
        """
        loss_terms = loss_terms if isinstance(loss_terms, (tuple, list)) else (loss_terms,)
        ok, why = self._fused_possible(criterion, loss_terms)
        if not ok:
            kwargs.pop('steps_per_launch', None)            # fused-path option, not an optimizer argument
            if self.backend == 'fused':
                raise RuntimeError('backend="fused" but the fused path cannot run: %s' % why)
            if self.backend == 'auto' and not self._warned and self.device.type == 'cuda':
                warnings.warn('pydens_b200: using the autograd path (%s)' % why, stacklevel=2)
                self._warned = True
            return self._fit_autograd(niters, batch_size, sampler, loss_terms, optimizer, criterion, lr, **kwargs)
        engine = self._get_engine()
        if engine is None:                              # plan creation reported "unsupported": autograd path
            return self.fit(niters, batch_size, sampler, loss_terms, optimizer, criterion, lr, **kwargs)
        return engine.fit(niters, batch_size, sampler, loss_terms, optimizer, criterion, lr, **kwargs)

    def _make_optimizer(self, optimizer, lr, fused_hint=False, **kwargs):
        if optimizer is None:
            if self.optimizer is None:
                raise ValueError('optimizer=None but no optimizer exists yet')
            return
        params = [p for p in self.model.parameters() if p.requires_grad]
        cls = getattr(torch.optim, optimizer)
        if fused_hint and optimizer in ('Adam', 'AdamW') and 'fused' not in kwargs and 'foreach' not in kwargs:
            try:
                self.optimizer = cls(params, lr=lr, fused=True, capturable=True, **kwargs)
                return
            except (TypeError, RuntimeError, ValueError):
                pass
        self.optimizer = cls(params, lr=lr, **kwargs)

    def _sample_host(self, sampler, batch_size):
        if sampler is None:
            return [torch.rand((batch_size, 1), device=self.device) for _ in range(self.model.total)]
        arr = np.asarray(sampler.sample(batch_size)).astype(np.float32)
        return [torch.from_numpy(np.ascontiguousarray(arr[:, i:i + 1])).to(self.device) for i in range(arr.shape[1])]

    def _constraint_loss(self, nums, xs, criterion):
        def _forward(*pts):
            return self.model(self.reshape_and_concat(pts).to(self.device))
        total = 0
        zero = torch.zeros(1, device=self.device)
        for num in nums:
            with warnings.catch_warnings():
                warnings.simplefilter('ignore', UserWarning)      # [1,1] vs [1] target, as in the reference
                total = total + criterion(self.ctx.run(self.constraints[num], _forward, *xs), zero)
        return total

    @staticmethod
    def _constraint_numbers(loss_terms):
        return [int(name.replace('constraint', '').replace('_', '')) for name in loss_terms if 'constraint' in name]

    def _fit_autograd(self, niters, batch_size, sampler, loss_terms, optimizer, criterion, lr, **kwargs):
        """ Device-aware restatement of the reference loop (:419-464) on autograd. """
        self._release_engine()
        self._make_optimizer(optimizer, lr, **kwargs)
        nums = self._constraint_numbers(loss_terms)
        self.model.train()
        for _ in _progress(niters):
            self.optimizer.zero_grad()
            xs = self._sample_host(sampler, batch_size)
            for x in xs:
                x.requires_grad_()
            u_hat = self.ctx.run(self.model, self.reshape_and_concat(xs))
            loss = 0
            if 'equation' in loss_terms:
                loss = loss + criterion(self.ctx.run(self.equation, u_hat, *xs), torch.zeros_like(xs[0]))
            if nums:
                loss = loss + self._constraint_loss(nums, xs, criterion)
            loss.backward()
            self.optimizer.step()
            self.losses.append(loss.detach().cpu().numpy())

    def _release_engine(self):
        """ Detach parameters from the flat buffer of a previous fused fit (autograd path owns them). """
        if self._engine is not None:
            self._engine.release()
            self._engine = None

    def predict(self, *xs):
        """ Solution approximation at the given points; every argument is a tensor / array / number,
        tiled to the longest (reference :466-487).  Returns an (N x 1) numpy array. """
        pts = self.reshape_and_concat(xs).to(self.device, torch.float32)
        self.model.eval()
        if self._traced is not None and self.backend != 'torch' and self.device.type == 'cuda':
            engine = self._get_engine()
            if engine is not None:
                return engine.forward(pts).reshape(-1, 1).cpu().numpy()
        with torch.no_grad():
            result = self.ctx.run(self.model, pts)
        return result.detach().cpu().numpy()

    # ------------------------------------------------------------------------------------------
    # engine-level helpers (parity tests, smoke, bench)
    # ------------------------------------------------------------------------------------------
    def flat_params(self):
        """ The flat fp32 parameter buffer in engine layout (W_0, b_0, …, log_scale, V…; padded). """
        return self._get_engine().flat.detach().clone()

    def load_flat_params(self, flat):
        eng = self._get_engine()
        with torch.no_grad():
            eng.flat[:len(flat)].copy_(torch.as_tensor(flat, dtype=torch.float32))

    def loss_and_grads(self, points):
        """ One fused evaluation on explicit points -> (loss, flat grads [n_params], residual [N]). """
        return self._get_engine().loss_and_grads(points)
