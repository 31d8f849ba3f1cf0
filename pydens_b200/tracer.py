""" Symbolic tracing of user `equation` / `initial_condition` callables.

The reference treats the equation as an opaque Python callable executed on autograd tensors every
iteration (pydens/model_torch.py:448), each `D` being a full reverse sweep (:174-178).  Here the
callable is run ONCE on symbolic proxies; `D` differentiates symbolically, so the residual becomes
a small expression DAG over

    x_k (point columns), u, du/dx_i, d2u/dx_i^2, V variables, constants,

from which we derive (a) the derivative jet the network kernel has to carry and (b) two register
programs (include/pinn_b200.h, PinnInstr): the residual with its partials w.r.t. every jet channel
and variable, and the jet of the initial condition.  Anything outside this vocabulary raises
`NotLowerable`; the Solver then uses its autograd path for that problem.
"""
import math
import numbers

import numpy as np
import torch


class NotLowerable(Exception):
    """ The callable uses something the fused path does not cover. """


# ------------------------------------------------------------------------------------------------
# expression DAG (hash-consed)
# ------------------------------------------------------------------------------------------------
UNARY = ('neg', 'sin', 'cos', 'tan', 'exp', 'log', 'sqrt', 'tanh', 'sigmoid', 'abs', 'sign')
BINARY = ('add', 'sub', 'mul', 'div', 'pow')


class Expr:
    __slots__ = ('kind', 'args', 'value', '_hash')
    _table = {}

    def __new__(cls, kind, args=(), value=None):
        key = (kind, tuple(id(a) for a in args), value)
        hit = cls._table.get(key)
        if hit is not None:
            return hit
        self = object.__new__(cls)
        self.kind, self.args, self.value = kind, tuple(args), value
        self._hash = hash(key)
        cls._table[key] = self
        return self

    def __hash__(self):
        return self._hash

    def __eq__(self, other):
        return self is other

    def __repr__(self):
        if self.kind == 'const':
            return repr(self.value)
        if self.kind == 'coord':
            return 'x%d' % self.value
        if self.kind == 'u':
            return 'u' + ''.join('_%d' % i for i in self.value)
        if self.kind == 'uc':
            return 'u[%d]' % self.value[0] + ''.join('_%d' % i for i in self.value[1])
        if self.kind == 'var':
            return 'V[%s]' % self.value
        if self.kind == 'ch':
            return 'U%d' % self.value
        if self.kind == 'powi':
            return '(%r)**%d' % (self.args[0], self.value)
        return '%s(%s)' % (self.kind, ', '.join(map(repr, self.args)))


def const(v):
    v = float(v)
    if v == 0.0:
        v = 0.0                      # fold -0.0
    return Expr('const', (), v)


ZERO, ONE = const(0.0), const(1.0)
MAX_ORDER = 4                               # D() nests up to four times on the fused path (u_xxx of KdV, u_xxxx of beams)


def is_const(e, v=None):
    return e.kind == 'const' and (v is None or e.value == v)


def coord(k):
    return Expr('coord', (), int(k))


def uleaf(multi_index=()):
    return Expr('u', (), tuple(sorted(multi_index)))


def ucleaf(j, multi_index=()):
    """ Component j of the output of a network with several outputs, differentiated along `multi_index`. """
    return Expr('uc', (), (int(j), tuple(sorted(multi_index))))


def var(name):
    return Expr('var', (), name)


def chleaf(c):
    """ Channel c of the jet of u as the kernel carries it (value, directional firsts, directional seconds). """
    return Expr('ch', (), int(c))


def add(a, b):
    if is_const(a) and is_const(b):
        return const(a.value + b.value)
    if is_const(a, 0.0):
        return b
    if is_const(b, 0.0):
        return a
    return Expr('add', (a, b))


def sub(a, b):
    if is_const(a) and is_const(b):
        return const(a.value - b.value)
    if is_const(b, 0.0):
        return a
    if is_const(a, 0.0):
        return neg(b)
    if a is b:
        return ZERO
    return Expr('sub', (a, b))


def neg(a):
    if is_const(a):
        return const(-a.value)
    if a.kind == 'neg':
        return a.args[0]
    return Expr('neg', (a,))


def mul(a, b):
    if is_const(a) and is_const(b):
        return const(a.value * b.value)
    if is_const(a, 0.0) or is_const(b, 0.0):
        return ZERO
    if is_const(a, 1.0):
        return b
    if is_const(b, 1.0):
        return a
    if is_const(a, -1.0):
        return neg(b)
    if is_const(b, -1.0):
        return neg(a)
    if is_const(b):                  # constants to the left: canonical form
        a, b = b, a
    return Expr('mul', (a, b))


def div(a, b):
    if is_const(b, 1.0):
        return a
    if is_const(a) and is_const(b):
        return const(a.value / b.value)
    if is_const(a, 0.0):
        return ZERO
    return Expr('div', (a, b))


def powi(a, n):
    n = int(n)
    if n == 0:
        return ONE
    if n == 1:
        return a
    if is_const(a):
        return const(a.value ** n)
    return Expr('powi', (a,), n)


def power(a, b):
    if is_const(b):
        e = b.value
        if float(e).is_integer() and abs(e) <= 64:
            return powi(a, int(e))
        if e == 0.5:
            return unary('sqrt', a)
        if is_const(a):
            return const(a.value ** e)
    return Expr('pow', (a, b))


_FOLD = {'neg': lambda v: -v, 'sin': math.sin, 'cos': math.cos, 'tan': math.tan, 'exp': math.exp,
         'log': math.log, 'sqrt': math.sqrt, 'tanh': math.tanh,
         'sigmoid': lambda v: 1.0 / (1.0 + math.exp(-v)), 'abs': abs,
         'sign': lambda v: (v > 0) - (v < 0)}


def unary(kind, a):
    if kind == 'neg':
        return neg(a)
    if is_const(a):
        try:
            return const(_FOLD[kind](a.value))
        except (ValueError, OverflowError):
            pass
    return Expr(kind, (a,))


# ------------------------------------------------------------------------------------------------
# differentiation
# ------------------------------------------------------------------------------------------------
def _chain(e, da_of):
    """ Shared derivative rules; `da_of(arg)` gives the derivative of an argument. """
    k = e.kind
    if k in ('add', 'sub'):
        a, b = e.args
        return (add if k == 'add' else sub)(da_of(a), da_of(b))
    if k == 'neg':
        return neg(da_of(e.args[0]))
    if k == 'mul':
        a, b = e.args
        return add(mul(da_of(a), b), mul(a, da_of(b)))
    if k == 'div':
        a, b = e.args
        da, db = da_of(a), da_of(b)
        if is_const(db, 0.0):
            return div(da, b)
        return sub(div(da, b), mul(div(e, b), db))
    if k == 'powi':
        a, n = e.args[0], e.value
        return mul(mul(const(n), powi(a, n - 1)), da_of(a))
    if k == 'pow':
        a, b = e.args
        da, db = da_of(a), da_of(b)
        t = ZERO
        if not is_const(da, 0.0):
            t = add(t, mul(mul(b, power(a, sub(b, ONE))), da))
        if not is_const(db, 0.0):
            t = add(t, mul(mul(e, unary('log', a)), db))
        return t
    a = e.args[0]
    da = da_of(a)
    if is_const(da, 0.0):
        return ZERO
    if k == 'sin':
        return mul(unary('cos', a), da)
    if k == 'cos':
        return neg(mul(unary('sin', a), da))
    if k == 'tan':
        return mul(add(ONE, powi(e, 2)), da)
    if k == 'exp':
        return mul(e, da)
    if k == 'log':
        return div(da, a)
    if k == 'sqrt':
        return div(da, mul(const(2.0), e))
    if k == 'tanh':
        return mul(sub(ONE, powi(e, 2)), da)
    if k == 'sigmoid':
        return mul(mul(e, sub(ONE, e)), da)
    if k == 'abs':
        return mul(unary('sign', a), da)
    if k == 'sign':
        return ZERO
    raise NotLowerable('cannot differentiate %r' % k)


def diff_coord(e, k, memo=None):
    """ Total derivative of `e` w.r.t. point column k (u depends on every column). """
    memo = {} if memo is None else memo
    hit = memo.get(e)
    if hit is not None:
        return hit
    if e.kind == 'const' or e.kind == 'var':
        r = ZERO
    elif e.kind == 'coord':
        r = ONE if e.value == k else ZERO
    elif e.kind == 'u':
        if len(e.value) >= MAX_ORDER:
            raise NotLowerable('derivatives of order > %d are not supported by the fused path' % MAX_ORDER)
        r = uleaf(e.value + (k,))
    elif e.kind == 'uc':
        if len(e.value[1]) >= MAX_ORDER:
            raise NotLowerable('derivatives of order > %d are not supported by the fused path' % MAX_ORDER)
        r = ucleaf(e.value[0], e.value[1] + (k,))
    else:
        r = _chain(e, lambda a: diff_coord(a, k, memo))
    memo[e] = r
    return r


def diff_leaf(e, leaf, memo=None):
    """ Partial derivative of `e` w.r.t. one leaf (a jet channel of u or a variable). """
    memo = {} if memo is None else memo
    hit = memo.get(e)
    if hit is not None:
        return hit
    if e is leaf:
        r = ONE
    elif e.kind in ('const', 'coord', 'u', 'uc', 'var', 'ch'):
        r = ZERO
    else:
        r = _chain(e, lambda a: diff_leaf(a, leaf, memo))
    memo[e] = r
    return r


def leaves(e, kinds, seen=None, out=None):
    seen = set() if seen is None else seen
    out = [] if out is None else out
    if e in seen:
        return out
    seen.add(e)
    if e.kind in kinds:
        out.append(e)
    for a in e.args:
        leaves(a, kinds, seen, out)
    return out


_REBUILD = {'add': lambda a: add(*a), 'sub': lambda a: sub(*a), 'mul': lambda a: mul(*a), 'div': lambda a: div(*a),
            'pow': lambda a: power(*a), 'neg': lambda a: neg(*a)}


def substitute(e, mapping, memo=None):
    """ Rebuild `e` with the leaves in `mapping` replaced by the mapped expressions. """
    memo = {} if memo is None else memo
    hit = memo.get(e)
    if hit is not None:
        return hit
    if e in mapping:
        r = mapping[e]
    elif not e.args:
        r = e
    else:
        args = [substitute(a, mapping, memo) for a in e.args]
        if e.kind == 'powi':
            r = powi(args[0], e.value)
        elif e.kind in _REBUILD:
            r = _REBUILD[e.kind](args)
        else:
            r = unary(e.kind, args[0])
    memo[e] = r
    return r


# ------------------------------------------------------------------------------------------------
# proxies handed to user callables
# ------------------------------------------------------------------------------------------------
def _as_expr(x):
    if isinstance(x, Sym):
        return x.expr
    if isinstance(x, (numbers.Real, np.floating, np.integer)):
        return const(float(x))
    if isinstance(x, np.ndarray) and x.size == 1:
        return const(float(x.reshape(-1)[0]))
    if isinstance(x, torch.Tensor):
        if x.numel() == 1 and not x.requires_grad:
            return const(float(x.reshape(-1)[0]))
        raise NotLowerable('tensor constants with more than one element (or requiring grad) in the equation')
    raise NotLowerable('unsupported operand of type %s' % type(x).__name__)


_TORCH_UNARY = {'sin': 'sin', 'cos': 'cos', 'tan': 'tan', 'exp': 'exp', 'log': 'log', 'sqrt': 'sqrt',
                'tanh': 'tanh', 'sigmoid': 'sigmoid', 'abs': 'abs', 'absolute': 'abs', 'neg': 'neg',
                'negative': 'neg', 'sign': 'sign', 'sgn': 'sign'}
_TORCH_BINARY = {'add': add, 'sub': sub, 'subtract': sub, 'mul': mul, 'multiply': mul, 'div': div,
                 'divide': div, 'true_divide': div, 'pow': power}
_NP_UNARY = {np.sin: 'sin', np.cos: 'cos', np.tan: 'tan', np.exp: 'exp', np.log: 'log', np.sqrt: 'sqrt',
             np.tanh: 'tanh', np.abs: 'abs', np.negative: 'neg', np.sign: 'sign'}
_NP_BINARY = {np.add: add, np.subtract: sub, np.multiply: mul, np.divide: div, np.true_divide: div,
              np.power: power}

# functions expressed through the opcodes above (no opcode of their own)
_REWRITES = {
    'square': lambda a: powi(a, 2),
    'reciprocal': lambda a: div(ONE, a),
    'rsqrt': lambda a: div(ONE, unary('sqrt', a)),
    'sinh': lambda a: mul(const(0.5), sub(unary('exp', a), unary('exp', neg(a)))),
    'cosh': lambda a: mul(const(0.5), add(unary('exp', a), unary('exp', neg(a)))),
    'exp2': lambda a: unary('exp', mul(const(math.log(2.0)), a)),
    'log2': lambda a: mul(const(1.0 / math.log(2.0)), unary('log', a)),
    'log10': lambda a: mul(const(1.0 / math.log(10.0)), unary('log', a)),
    # piecewise-linear functions through |.|: exact where they are linear, torch's values everywhere, torch's
    # derivatives except exactly at the kink (there: the mean of the one-sided ones)
    'expm1': lambda a: mul(unary('tanh', mul(const(0.5), a)), add(unary('exp', a), ONE)),   # e^a - 1 = tanh(a / 2) (e^a + 1): no cancellation near 0
    'log1p': lambda a: unary('log', add(ONE, a)),        # absolute error of one rounding of 1 + a (1e-7 in fp32), not a relative one
    'relu': lambda a: mul(const(0.5), add(a, unary('abs', a))),
    'silu': lambda a: mul(a, unary('sigmoid', a)),
    'softplus': lambda a: add(mul(const(0.5), add(a, unary('abs', a))),                     # max(a, 0) + log(1 + e^-|a|)
                              unary('log', add(ONE, unary('exp', neg(unary('abs', a)))))),
}


def _maximum(a, b):
    return mul(const(0.5), add(add(a, b), unary('abs', sub(a, b))))


def _minimum(a, b):
    return mul(const(0.5), sub(add(a, b), unary('abs', sub(a, b))))


def _clamp(a, lo=None, hi=None):
    if lo is not None:
        a = _maximum(a, _as_expr(lo))
    if hi is not None:
        a = _minimum(a, _as_expr(hi))
    return a


_FINITE_KINDS = ('const', 'coord', 'u', 'uc', 'var', 'ch', 'add', 'sub', 'mul', 'neg', 'sin', 'cos', 'tanh', 'sigmoid', 'abs', 'sign')


def _always_finite(e, seen=None):
    """ True when `e` cannot evaluate to inf / NaN on finite inputs short of overflow of a polynomial: sums, products,
    bounded functions, non-negative integer powers.  (exp, log, sqrt, /, ** and tan are not in that set.) """
    seen = set() if seen is None else seen
    if e in seen:
        return True
    seen.add(e)
    if e.kind == 'powi':
        return e.value >= 0 and _always_finite(e.args[0], seen)
    if e.kind not in _FINITE_KINDS:
        return False
    return all(_always_finite(a, seen) for a in e.args)


def _where(condition, a, b):
    """ torch.where(condition, a, b) as c a + (1 - c) b with the 0 / 1 indicator c of the condition: exact for c in {0, 1}
    provided the branch that is NOT selected is finite — torch.where is often the guard around a branch that is not
    (sqrt of a negative number, a division by zero), and 0 * NaN is NaN: such branches stay on autograd. """
    c = Sym._indicator_expr(condition)
    a, b = _as_expr(a), _as_expr(b)
    if not (_always_finite(a) and _always_finite(b)):
        raise NotLowerable('torch.where with a branch that may not be finite where it is not selected')
    return add(mul(c, a), mul(sub(ONE, c), b))


_REWRITES2 = {'maximum': _maximum, 'minimum': _minimum, 'max': _maximum, 'min': _minimum, 'fmax': _maximum, 'fmin': _minimum,
              'hypot': lambda a, b: unary('sqrt', add(powi(a, 2), powi(b, 2)))}


class Sym:
    """ Symbolic stand-in for an `[N, 1]` tensor inside a traced callable. """
    __array_priority__ = 1000

    def __init__(self, expr):
        self.expr = expr

    # arithmetic
    def __add__(self, o): return Sym(add(self.expr, _as_expr(o)))
    def __radd__(self, o): return Sym(add(_as_expr(o), self.expr))
    def __sub__(self, o): return Sym(sub(self.expr, _as_expr(o)))
    def __rsub__(self, o): return Sym(sub(_as_expr(o), self.expr))
    def __mul__(self, o): return Sym(mul(self.expr, _as_expr(o)))
    def __rmul__(self, o): return Sym(mul(_as_expr(o), self.expr))
    def __truediv__(self, o): return Sym(div(self.expr, _as_expr(o)))
    def __rtruediv__(self, o): return Sym(div(_as_expr(o), self.expr))
    def __pow__(self, o): return Sym(power(self.expr, _as_expr(o)))
    def __rpow__(self, o): return Sym(power(_as_expr(o), self.expr))
    def __neg__(self): return Sym(neg(self.expr))
    def __pos__(self): return self
    def __abs__(self): return Sym(unary('abs', self.expr))

    # tensor-ish methods users reach for
    def sin(self): return Sym(unary('sin', self.expr))
    def cos(self): return Sym(unary('cos', self.expr))
    def exp(self): return Sym(unary('exp', self.expr))
    def log(self): return Sym(unary('log', self.expr))
    def sqrt(self): return Sym(unary('sqrt', self.expr))
    def tanh(self): return Sym(unary('tanh', self.expr))
    def abs(self): return Sym(unary('abs', self.expr))
    def pow(self, o): return self.__pow__(o)
    def square(self): return Sym(powi(self.expr, 2))
    def tan(self): return Sym(unary('tan', self.expr))
    def sigmoid(self): return Sym(unary('sigmoid', self.expr))
    def sinh(self): return Sym(_REWRITES['sinh'](self.expr))
    def cosh(self): return Sym(_REWRITES['cosh'](self.expr))
    def reciprocal(self): return Sym(div(ONE, self.expr))
    def rsqrt(self): return Sym(_REWRITES['rsqrt'](self.expr))
    def neg(self): return Sym(neg(self.expr))
    def relu(self): return Sym(_REWRITES['relu'](self.expr))
    def clamp(self, min=None, max=None): return Sym(_clamp(self.expr, min, max))      # noqa: A002  (torch's own names)
    clip = clamp
    def clamp_min(self, min): return Sym(_clamp(self.expr, min, None))                 # noqa: A002
    def clamp_max(self, max): return Sym(_clamp(self.expr, None, max))                 # noqa: A002
    def maximum(self, o): return Sym(_maximum(self.expr, _as_expr(o)))
    def minimum(self, o): return Sym(_minimum(self.expr, _as_expr(o)))
    def view(self, *shape): return self
    def reshape(self, *shape): return self
    def float(self): return self
    def double(self): return self
    def to(self, *args, **kwargs): return self             # dtype / device casts of a symbolic column are no-ops
    def type(self, *args, **kwargs): return self
    def type_as(self, other): return self
    def clone(self): return self
    def contiguous(self): return self
    def squeeze(self, *args): return self
    def unsqueeze(self, *args): return self
    dtype = torch.float32

    def __bool__(self):
        raise NotLowerable('data-dependent control flow in a traced callable')

    # Order comparisons give the 0 / 1 indicator (1 + sign(a - b)) / 2 — what torch's bool tensor is once it meets
    # arithmetic or torch.where, except ON the threshold (1/2 instead of 0 or 1: a set of measure zero for sampled
    # points).  Its derivative is zero, as autograd's.  Indicators combine with & | ~ and select with torch.where;
    # using one in an `if` still leaves the fused path (__bool__), and so does == / !=.
    def _indicator(self, other, flip):
        a, b = self.expr, _as_expr(other)
        d = sub(b, a) if flip else sub(a, b)
        out = Sym(mul(const(0.5), add(ONE, unary('sign', d))))
        out.is_indicator = True
        return out

    def __gt__(self, o): return self._indicator(o, False)
    def __ge__(self, o): return self._indicator(o, False)
    def __lt__(self, o): return self._indicator(o, True)
    def __le__(self, o): return self._indicator(o, True)

    def _compare(self, other):
        raise NotLowerable('== / != (data-dependent control flow) in a traced callable')

    __eq__ = __ne__ = _compare
    __hash__ = object.__hash__                 # defining __eq__ would otherwise make Sym unhashable

    @staticmethod
    def _indicator_expr(x):
        if isinstance(x, Sym) and getattr(x, 'is_indicator', False):
            return x.expr
        if isinstance(x, (bool, np.bool_)):
            return ONE if x else ZERO
        if isinstance(x, torch.Tensor) and x.dtype == torch.bool and x.numel() == 1:
            return ONE if bool(x) else ZERO
        raise NotLowerable('boolean operation on something that is not a comparison of traced tensors')

    def _logical(self, other, kind):
        a, b = Sym._indicator_expr(self), Sym._indicator_expr(other)
        out = Sym(mul(a, b) if kind == 'and' else sub(add(a, b), mul(a, b)) if kind == 'or'
                  else sub(add(a, b), mul(const(2.0), mul(a, b))))
        out.is_indicator = True
        return out

    def __and__(self, o): return self._logical(o, 'and')
    def __or__(self, o): return self._logical(o, 'or')
    def __xor__(self, o): return self._logical(o, 'xor')
    __rand__, __ror__, __rxor__ = __and__, __or__, __xor__

    def __invert__(self):
        out = Sym(sub(ONE, Sym._indicator_expr(self)))
        out.is_indicator = True
        return out

    def where(self, condition, other):
        return Sym(_where(condition, self, other))

    # A traced value that depends on the points (u, its derivatives, the point columns) is one column, [N, 1].
    # Selecting that column keeps the shape and is the identity: f[:, 0:1], f[:, [0]], f[..., 0:1], and splitting into
    # one-column pieces.  f[:, 0] is [N] in torch (and then broadcasts to [N, N] against the [N, 1] columns), so it
    # stays on autograd, as does any other index — and any index of a variable or constant, which is not [N, 1].
    def __getitem__(self, key):
        _column_of_index(_as_column(self), key)
        return self

    def split(self, size, dim=None):
        return _split_columns(self, size, dim)

    def chunk(self, chunks, dim=None):
        return _chunk_columns(self, chunks, dim)

    # what a tensor would accept but a symbolic column cannot express: bail out of the fused path cleanly
    # (the reference runs such equations on autograd, model_torch.py:448) instead of raising a TypeError
    def _unsupported(self, *args, **kwargs):
        raise NotLowerable('indexing / integer arithmetic / len() on a traced tensor')

    __setitem__ = __mod__ = __rmod__ = __floordiv__ = __rfloordiv__ = _unsupported
    __len__ = __iter__ = __matmul__ = __rmatmul__ = _unsupported
    __int__ = __float__ = __index__ = _unsupported

    def __getattr__(self, name):
        if name.startswith('__'):
            raise AttributeError(name)
        raise NotLowerable('tensor attribute %r is not available while tracing' % name)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        name = getattr(func, '__name__', None)
        if name in _COLUMN_FUNCS:
            return _COLUMN_FUNCS[name](*args, **(kwargs or {}))
        if name in ('clamp', 'clip', 'clamp_min', 'clamp_max') and args and set(kwargs or ()) <= {'min', 'max'}:
            rest = list(args[1:])
            if name == 'clamp_max':
                rest = [None] + rest
            lo = (kwargs or {}).get('min', rest[0] if len(rest) > 0 else None)
            hi = (kwargs or {}).get('max', rest[1] if len(rest) > 1 else None)
            if len(rest) <= 2 and (lo is not None or hi is not None):
                return Sym(_clamp(_as_expr(args[0]), lo, hi))
        if kwargs and name in ('relu', 'silu', 'softplus', 'sigmoid', 'tanh'):
            # torch.nn.functional passes its defaults on as keywords: those (and only those) are fine
            defaults = {'inplace': False, 'beta': 1, 'threshold': 20}
            if all(k in defaults and v == defaults[k] for k, v in kwargs.items()):
                kwargs = None
        if kwargs:
            raise NotLowerable('keyword arguments to torch.%s while tracing' % name)
        if name in ('__add__', '__radd__'): name = 'add'
        if name in ('__mul__', '__rmul__'): name = 'mul'
        if name in ('__sub__',): name = 'sub'
        if name in ('__truediv__',): name = 'div'
        if name in ('__pow__',): name = 'pow'
        if name == '__rsub__':
            return Sym(sub(_as_expr(args[1]), _as_expr(args[0])))
        if name == '__rtruediv__':
            return Sym(div(_as_expr(args[1]), _as_expr(args[0])))
        if name == '__rpow__':
            return Sym(power(_as_expr(args[1]), _as_expr(args[0])))
        if name in _TORCH_UNARY and len(args) == 1:
            return Sym(unary(_TORCH_UNARY[name], _as_expr(args[0])))
        if name in _TORCH_BINARY and len(args) == 2:
            return Sym(_TORCH_BINARY[name](_as_expr(args[0]), _as_expr(args[1])))
        if name in _REWRITES and len(args) == 1:
            return Sym(_REWRITES[name](_as_expr(args[0])))
        if name in _REWRITES2 and len(args) == 2:
            return Sym(_REWRITES2[name](_as_expr(args[0]), _as_expr(args[1])))
        if name == 'where' and len(args) == 3:
            return Sym(_where(args[0], args[1], args[2]))
        if name == 'heaviside' and len(args) == 2:
            # 0 below, `values` at, 1 above zero:  (1 + s) / 2 + (values - 1/2) (1 - s^2)  with s = sign(input)
            sg, v = unary('sign', _as_expr(args[0])), _as_expr(args[1])
            return Sym(add(mul(const(0.5), add(ONE, sg)), mul(sub(v, const(0.5)), sub(ONE, mul(sg, sg)))))
        if name in ('gt', 'ge', 'lt', 'le', 'greater', 'greater_equal', 'less', 'less_equal') and len(args) == 2:
            flip = name in ('lt', 'le', 'less', 'less_equal')
            if isinstance(args[0], Sym):
                return args[0]._indicator(args[1], flip)
            return args[1]._indicator(args[0], not flip)
        if name in ('logical_and', 'logical_or', 'logical_xor', '__and__', '__or__', '__xor__', '__rand__', '__ror__', '__rxor__') and len(args) == 2:
            lhs = args[0] if isinstance(args[0], Sym) else args[1]
            rhs = args[1] if isinstance(args[0], Sym) else args[0]
            return lhs._logical(rhs, 'and' if 'and' in name else ('xor' if 'xor' in name else 'or'))
        if name in ('logical_not', '__invert__') and len(args) == 1:
            return args[0].__invert__()
        if name in ('__gt__', '__ge__') and len(args) == 2:
            return args[0]._indicator(args[1], False) if isinstance(args[0], Sym) else args[1]._indicator(args[0], True)
        if name in ('__lt__', '__le__') and len(args) == 2:
            return args[0]._indicator(args[1], True) if isinstance(args[0], Sym) else args[1]._indicator(args[0], False)
        if name in ('zeros_like', 'ones_like') and len(args) == 1:
            return Sym(ZERO if name == 'zeros_like' else ONE)
        if name == 'full_like' and len(args) == 2 and isinstance(args[1], numbers.Real):
            return Sym(const(float(args[1])))
        raise NotLowerable('torch.%s is not supported by the fused path' % name)

    def __array_ufunc__(self, ufunc, method, *inputs, **kwargs):
        if method != '__call__' or kwargs:
            raise NotLowerable('numpy ufunc %s.%s while tracing' % (ufunc.__name__, method))
        if ufunc in _NP_UNARY and len(inputs) == 1:
            return Sym(unary(_NP_UNARY[ufunc], _as_expr(inputs[0])))
        if ufunc in _NP_BINARY and len(inputs) == 2:
            return Sym(_NP_BINARY[ufunc](_as_expr(inputs[0]), _as_expr(inputs[1])))
        if ufunc.__name__ in _REWRITES and len(inputs) == 1:
            return Sym(_REWRITES[ufunc.__name__](_as_expr(inputs[0])))
        if ufunc.__name__ in _REWRITES2 and len(inputs) == 2:
            return Sym(_REWRITES2[ufunc.__name__](_as_expr(inputs[0]), _as_expr(inputs[1])))
        raise NotLowerable('numpy.%s is not supported by the fused path' % ufunc.__name__)


def _as_column(s):
    """ `s` when it stands for an [N, 1] column of the batch: an expression of u or of the point columns.  A V(...)
    variable is a one-element tensor and a constant a number in the reference; indexing, splitting or concatenating
    those fails there (or means something else), so it is not lowered here either. """
    if not leaves(s.expr, ('u', 'uc', 'coord')):
        raise NotLowerable('indexing / split / concatenation of a traced value that is not a column of the batch')
    return s


def _column_of_index(s, key):
    """ Column selected by `key` when it keeps the [N, 1] shape (f[:, j:j+1], f[:, [j]], f[..., j:j+1]); a traced column
    has one column, so only j = 0 exists. """
    if not isinstance(key, tuple) or len(key) != 2 or not (key[0] is Ellipsis or key[0] == slice(None)):
        raise NotLowerable('indexing a traced tensor other than f[:, j:j+1] / f[:, [j]]')
    sel = key[1]
    if isinstance(sel, slice) and sel.step in (None, 1) and isinstance(sel.start, int) and isinstance(sel.stop, int) \
            and sel.start >= 0 and sel.stop == sel.start + 1:
        j = sel.start
    elif isinstance(sel, list) and len(sel) == 1 and isinstance(sel[0], int):
        j = sel[0]
    else:
        raise NotLowerable('indexing a traced tensor other than f[:, j:j+1] / f[:, [j]] (f[:, j] is one-dimensional)')
    if j not in (0, -1):
        raise NotLowerable('column %d of a one-column traced tensor' % j)
    return 0


def _column_dim(dim):
    if dim not in (1, -1):
        raise NotLowerable('split / concatenation of traced tensors along dimension %r (only the column one)' % (dim,))


def _split_columns(s, size, dim=None):
    """ torch.split(f, 1, dim=1) / f.split(1, 1) of a one-column value: that column. """
    _as_column(s)
    _column_dim(dim)
    if not (size >= 1 if isinstance(size, int) else isinstance(size, (list, tuple)) and list(size) == [1]):
        raise NotLowerable('torch.split of a traced tensor with sizes %r' % (size,))
    return (s,)


def _chunk_columns(s, chunks, dim=None):
    _as_column(s)
    _column_dim(dim)
    if not (isinstance(chunks, int) and chunks >= 1):
        raise NotLowerable('torch.chunk of a traced tensor into %r chunks' % (chunks,))
    return (s,)


def _concat_columns(tensors, dim=None, axis=None, hstack=False):
    """ torch.cat([r_1, …, r_m], dim=1) and its spellings: a residual of m columns (VecSym). """
    if not hstack:
        _column_dim(dim if axis is None else axis)
    cols = []
    for t in tensors:
        if isinstance(t, VecSym):
            cols += t.exprs
        elif isinstance(t, Sym):
            cols.append(_as_column(t).expr)
        else:
            raise NotLowerable('concatenation of a traced value with a %s' % type(t).__name__)
    if not cols:
        raise NotLowerable('empty concatenation')
    return Sym(cols[0]) if len(cols) == 1 else VecSym(cols)


_COLUMN_FUNCS = {
    'cat': lambda tensors, dim=0: _concat_columns(tensors, dim),
    'concat': lambda tensors, dim=0: _concat_columns(tensors, dim),
    'concatenate': lambda tensors, axis=0: _concat_columns(tensors, axis),
    'hstack': lambda tensors: _concat_columns(tensors, hstack=True),
    'column_stack': lambda tensors: _concat_columns(tensors, hstack=True),
    'split': lambda s, size, dim=0: _split_columns(s, size, dim),
    'chunk': lambda s, chunks, dim=0: _chunk_columns(s, chunks, dim),
}


class VecSym:
    """ Symbolic stand-in for an `[N, m]` residual, m > 1: the columns r_1 … r_m, as `torch.cat` of one-column values
    returns it.  It can only be returned by the equation (or concatenated further); the loss of the reference,
    `criterion(residual, zeros[N, 1])`, broadcasts over the m columns (model_torch.py:448). """

    def __init__(self, exprs):
        self.exprs = list(exprs)

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        name = getattr(func, '__name__', None)
        if name in ('cat', 'concat', 'concatenate', 'hstack', 'column_stack'):
            return _COLUMN_FUNCS[name](*args, **(kwargs or {}))
        raise NotLowerable('torch.%s of a residual with several columns' % name)

    def __getattr__(self, name):
        if name.startswith('__'):
            raise AttributeError(name)
        raise NotLowerable('%r of a residual with several columns' % name)

    def _unsupported(self, *args, **kwargs):
        raise NotLowerable('arithmetic / indexing on a residual with several columns')

    __add__ = __radd__ = __sub__ = __rsub__ = __mul__ = __rmul__ = __truediv__ = __rtruediv__ = _unsupported
    __pow__ = __rpow__ = __neg__ = __abs__ = __getitem__ = __len__ = __iter__ = __bool__ = _unsupported
    __array_ufunc__ = None


class Components:
    """ Symbolic stand-in for the `[N, k]` output of a network with k = 2..4 outputs (coupled systems).  The equation
    picks component j as a column, with the forms that keep the [N, 1] shape: f[:, j:j+1], f[:, [j]], f[..., j:j+1],
    torch.split(f, 1, dim=1), torch.chunk(f, k, dim=1) and their tensor-method spellings.  Anything else done to the whole
    value — arithmetic, D(), f[:, j] (one-dimensional in torch) — stays on autograd. """

    def __init__(self, k):
        self.k = k

    def column(self, j):
        if not 0 <= j < self.k:
            raise NotLowerable('component %d of a network with %d outputs' % (j, self.k))
        return Sym(ucleaf(j))

    def __getitem__(self, key):
        if not isinstance(key, tuple) or len(key) != 2 or not (key[0] is Ellipsis or key[0] == slice(None)):
            raise NotLowerable('indexing the network output other than f[:, j:j+1] / f[:, [j]]')
        sel = key[1]
        if isinstance(sel, slice) and sel.step in (None, 1) and isinstance(sel.start, int) and isinstance(sel.stop, int) \
                and sel.start >= 0 and sel.stop == sel.start + 1:
            return self.column(sel.start)
        if isinstance(sel, list) and len(sel) == 1 and isinstance(sel[0], int) and sel[0] >= 0:
            return self.column(sel[0])
        raise NotLowerable('indexing the network output other than f[:, j:j+1] / f[:, [j]] (f[:, j] is one-dimensional)')

    def split(self, size, dim=None):
        _column_dim(dim)
        if not (size == 1 or isinstance(size, (list, tuple)) and list(size) == [1] * self.k):
            raise NotLowerable('torch.split of the network output with sizes %r (one column per piece only)' % (size,))
        return tuple(self.column(j) for j in range(self.k))

    def chunk(self, chunks, dim=None):
        _column_dim(dim)
        if not (isinstance(chunks, int) and chunks >= self.k):
            raise NotLowerable('torch.chunk of the network output into %r chunks (one column per chunk only)' % (chunks,))
        return tuple(self.column(j) for j in range(self.k))

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        name = getattr(func, '__name__', None)
        if name in ('split', 'chunk') and args and isinstance(args[0], Components):
            return getattr(args[0], name)(*args[1:], **(kwargs or {}))
        raise NotLowerable('torch.%s of the whole output of a network with several outputs' % name)

    def __getattr__(self, name):
        if name.startswith('__'):
            raise AttributeError(name)
        raise NotLowerable('%r of the whole output of a network with several outputs' % name)

    def _unsupported(self, *args, **kwargs):
        raise NotLowerable('arithmetic on the whole output of a network with several outputs (select a component first)')

    __add__ = __radd__ = __sub__ = __rsub__ = __mul__ = __rmul__ = __truediv__ = __rtruediv__ = _unsupported
    __pow__ = __rpow__ = __neg__ = __pos__ = __abs__ = __len__ = __iter__ = __bool__ = _unsupported
    __array_ufunc__ = None


def sym_D(y, x):
    """ Symbolic counterpart of the D token. """
    if isinstance(y, VecSym):
        raise NotLowerable('D() of a residual with several columns')
    if isinstance(y, Components):
        raise NotLowerable('D() of the whole output of a network with several outputs (select a component first)')
    if _constraint_calls:                          # inside trace_constraint: x is a point tensor of the model call
        return Sym(diff_coord(_as_expr(y), _constraint_column(x)))
    if not isinstance(x, Sym) or x.expr.kind != 'coord':
        raise NotLowerable('D(y, x): x must be one of the equation arguments')
    return Sym(diff_coord(_as_expr(y), x.expr.value))


# the model calls of the constraint being traced (trace_constraint); a list rather than a ContextVar because the Solver
# runs user callables in its own contextvars.Context
_constraint_calls = []


def _constraint_column(x):
    """ The point column of the constraint's one model call that `x` was passed as (matched by identity): D(u(x0), x0)
    is the derivative of u along that column. """
    if isinstance(x, Sym):
        raise NotLowerable('D with respect to the batch points inside a constraint')
    calls = _constraint_calls[-1]
    if not calls:
        raise NotLowerable('D inside a constraint before it evaluates the model')
    cols = [k for k, p in enumerate(calls[0]) if p is x]
    if not cols:
        raise NotLowerable('D(y, p) inside a constraint: p is not one of the tensors the model is evaluated at')
    if len(cols) > 1:
        raise NotLowerable('D(y, p) inside a constraint: p is passed as %d point columns' % len(cols))
    if not isinstance(x, torch.Tensor) or not x.requires_grad:
        raise NotLowerable('D(y, p) inside a constraint: p does not require grad')
    return cols[0]


# ------------------------------------------------------------------------------------------------
# lowering: expression DAGs -> register programs
# ------------------------------------------------------------------------------------------------
OP = dict(CONST=0, COORD=1, VAR=2, ADD=3, SUB=4, MUL=5, DIV=6, NEG=7, MULI=8, ADDI=9, SIN=10, COS=11,
          EXP=12, LOG=13, SQRT=14, TANH=15, POWI=16, POW=17, ABS=18, SIGN=19, SIGMOID=20, RECIP=21, TAN=22)
_UNARY_OP = {'neg': 'NEG', 'sin': 'SIN', 'cos': 'COS', 'tan': 'TAN', 'exp': 'EXP', 'log': 'LOG',
             'sqrt': 'SQRT', 'tanh': 'TANH', 'sigmoid': 'SIGMOID', 'abs': 'ABS', 'sign': 'SIGN'}
MAX_PROG, MAX_SLOTS = 192, 96
MAX_DIRS = 6                                # derivative directions the kernels carry (include/pinn_b200.h: PINN_MAX_DIRS)


class Program:
    """ instrs: list of (op, dst, a, b, imm); outs: slot of every requested output. """

    def __init__(self, instrs, outs, n_slots):
        self.instrs, self.outs, self.n_slots = instrs, outs, n_slots

    def __len__(self):
        return len(self.instrs)


def lower(outputs, channel_of_u, var_index, n_reserved, pinned=None):
    """ Linearise `outputs` (list of Expr) into one program.

    Slots [0, n_reserved) hold the jet of u on entry and are never written ('ch' leaves read them;
    `channel_of_u` is kept for the signature only); `var_index` maps a variable name to its VAR operand.
    `pinned`: expressions to compute straight into a given reserved slot instead of a scratch one.
    """
    order, seen = [], set()

    def visit(e):
        if e in seen:
            return
        seen.add(e)
        for a in e.args:
            visit(a)
        order.append(e)

    for o in outputs:
        visit(o)

    def immediate_form(e):
        """ (op, operand, imm) when a binary node has a constant side that fits an immediate. """
        if e.kind == 'add':
            a, b = e.args
            if is_const(b): return 'ADDI', a, b.value
            if is_const(a): return 'ADDI', b, a.value
        if e.kind == 'sub' and is_const(e.args[1]):
            return 'ADDI', e.args[0], -e.args[1].value
        if e.kind == 'mul':
            a, b = e.args
            if is_const(a): return 'MULI', b, a.value
            if is_const(b): return 'MULI', a, b.value
        return None

    # which nodes need a materialised value (constants folded into immediates do not)
    needed = set()
    for e in order:
        imm = immediate_form(e)
        if imm:
            needed.add(imm[1])
        else:
            needed.update(e.args)
    needed.update(outputs)

    last_use = {}
    for i, e in enumerate(order):
        imm = immediate_form(e)
        for a in ([imm[1]] if imm else e.args):
            last_use[a] = i
    for o in outputs:
        last_use[o] = len(order) + 1          # outputs stay live

    slot_of, free, next_slot = {}, [], [n_reserved]
    instrs = []

    def alloc():
        if free:
            free.sort()
            return free.pop(0)
        s = next_slot[0]
        next_slot[0] += 1
        if s >= MAX_SLOTS:
            raise NotLowerable('expression needs more than %d scratch slots' % MAX_SLOTS)
        return s

    for i, e in enumerate(order):
        if e not in needed:
            continue
        if e.kind == 'ch':
            slot_of[e] = e.value
            continue
        if e.kind in ('u', 'uc'):
            raise NotLowerable('unexpected derivative leaf %r' % e)
        imm = immediate_form(e)
        operands = [imm[1]] if imm else list(e.args)
        srcs = [slot_of[a] for a in operands]
        # operands whose last use is this instruction free their slot (never a reserved/output one)
        for a in operands:
            if last_use.get(a) == i and a.kind != 'ch' and slot_of[a] >= n_reserved and slot_of[a] not in free:
                free.append(slot_of[a])
        dst = pinned[e] if pinned and e in pinned else alloc()
        slot_of[e] = dst
        if e.kind == 'const':
            instrs.append((OP['CONST'], dst, 0, 0, e.value))
        elif e.kind == 'coord':
            instrs.append((OP['COORD'], dst, e.value, 0, 0.0))
        elif e.kind == 'var':
            if e.value not in var_index:
                raise NotLowerable('variable %r is not available here' % e.value)
            instrs.append((OP['VAR'], dst, var_index[e.value], 0, 0.0))
        elif imm:
            instrs.append((OP[imm[0]], dst, srcs[0], 0, imm[2]))
        elif e.kind in ('add', 'sub', 'mul', 'div', 'pow'):
            instrs.append((OP[e.kind.upper()], dst, srcs[0], srcs[1], 0.0))
        elif e.kind == 'powi':
            instrs.append((OP['POWI'], dst, srcs[0], 0, float(e.value)))
        elif e.kind in _UNARY_OP:
            instrs.append((OP[_UNARY_OP[e.kind]], dst, srcs[0], 0, 0.0))
        else:
            raise NotLowerable('cannot lower %r' % e.kind)
    if len(instrs) > MAX_PROG:
        raise NotLowerable('expression needs %d instructions (max %d)' % (len(instrs), MAX_PROG))
    return Program(instrs, [slot_of[o] for o in outputs], max(next_slot[0], n_reserved))


def run_program(prog, ujet, coords, var_values):
    """ Reference interpreter of a Program on numpy arrays (host-side check of the lowering).
    ujet: [C, N] values of the reserved slots; coords: [total, N]; returns the list of outputs. """
    n = coords.shape[1]
    slots = np.zeros((max(prog.n_slots, 1), n), dtype=coords.dtype)
    slots[:ujet.shape[0]] = ujet
    inv = {v: k for k, v in OP.items()}
    for op, dst, a, b, imm in prog.instrs:
        name = inv[op]
        if name == 'CONST': r = np.full(n, imm, dtype=coords.dtype)
        elif name == 'COORD': r = coords[a]
        elif name == 'VAR': r = np.full(n, var_values[a], dtype=coords.dtype)
        elif name == 'ADD': r = slots[a] + slots[b]
        elif name == 'SUB': r = slots[a] - slots[b]
        elif name == 'MUL': r = slots[a] * slots[b]
        elif name == 'DIV': r = slots[a] / slots[b]
        elif name == 'POW': r = np.power(slots[a], slots[b])
        elif name == 'NEG': r = -slots[a]
        elif name == 'MULI': r = slots[a] * coords.dtype.type(imm)
        elif name == 'ADDI': r = slots[a] + coords.dtype.type(imm)
        elif name == 'POWI': r = slots[a] ** int(imm)
        elif name == 'SIGMOID': r = 1.0 / (1.0 + np.exp(-slots[a]))
        elif name == 'RECIP': r = 1.0 / slots[a]
        else: r = getattr(np, {'ABS': 'abs'}.get(name, name.lower()))(slots[a])
        slots[dst] = r
    return [slots[s].copy() for s in prog.outs]


# ------------------------------------------------------------------------------------------------
# tracing entry points
# ------------------------------------------------------------------------------------------------
class TracedEquation:
    """ Result of tracing: jet set + residual program (+ IC program). """

    def __init__(self):
        self.residual = None        # Expr
        self.dirs = []              # per direction: its point column when it is a unit vector, else -1
        self.dir_vecs = []          # per direction: the vector in point-column space (second-order directions first)
        self.ns = 0                 # how many of them also carry a second derivative
        self.var_names = []         # variables used by the equation, in VAR-operand order
        self.eq_prog = None         # outputs: [r, dr/dchannel_0 .. dr/dchannel_{C-1}, dr/dV_0 ..]
        self.ic_prog = None         # outputs: jet of ic (C entries) [+ C partials per variable] or None
        self.ic_has_vars = False
        self.n_slots = 0
        self.n_out = 1              # outputs of the network (k); k > 1: see trace
        self.order = 2              # 3 / 4: every direction carries its whole Taylor jet up to this order (ns = 0):
                                    # channel 1 + d*order + (k-1) = k-th derivative along direction d

    @property
    def nf(self):
        return len(self.dirs)

    @property
    def channels(self):
        return 1 + self.nf * self.order if self.order > 2 else 1 + self.nf + self.ns


CRITERION_EPS = 1e-30       # keeps sqrt(rho) differentiable at rho = 0 (a normal fp32 number; adds 1e-30 to the loss)


def apply_criterion(res, criterion):
    """ The kernels implement `MSELoss(residual, 0)` (reference model_torch.py:448 with its default criterion).  Any
    other pointwise criterion rho >= 0 with mean reduction is brought to that form by training on the residual
    r~ = sqrt(rho(r) + eps):  mean(r~^2) = mean(rho(r)) + eps, and the adjoint seed 2 r~ . dr~ = rho'(r) dr exactly —
    the square root cancels, also in floating point up to rounding, and sign(0) = 0 gives torch's subgradient at r = 0.

    criterion: None / ('mse',) | ('l1',) | ('huber', delta) | ('smooth_l1', beta)     (nn.L1Loss, nn.HuberLoss, nn.SmoothL1Loss)
    min(|r|, delta) is written |r| - relu(|r| - delta) with relu(x) = (x + |x|) / 2, which is exact for |r| <= delta: small
    residuals — where a fit ends up — do not lose digits against delta. """
    if criterion is None or criterion[0] == 'mse':
        return res
    return unary('sqrt', add(criterion_rho(res, criterion), const(CRITERION_EPS)))


def criterion_rho(res, criterion):
    """ The criterion's pointwise function rho(r): r^2 for MSELoss, |r| for L1Loss, Huber's / SmoothL1's piecewise form. """
    if criterion is None or criterion[0] == 'mse':
        return powi(res, 2)
    kind = criterion[0]
    a = unary('abs', res)
    if kind == 'l1' or (kind == 'smooth_l1' and float(criterion[1]) == 0.0):
        rho = a
    elif kind in ('huber', 'smooth_l1'):
        delta = float(criterion[1])
        if not delta > 0.0 or not math.isfinite(delta):
            raise NotLowerable('criterion threshold %r' % (criterion[1],))
        x = sub(a, const(delta))
        m = sub(a, mul(const(0.5), add(x, unary('abs', x))))              # min(|r|, delta)
        rho = mul(m, sub(a, mul(const(0.5), m)))                          # r^2 / 2 below delta, delta (|r| - delta / 2) above
        if kind == 'smooth_l1':
            rho = mul(const(1.0 / delta), rho)
    else:
        raise NotLowerable('criterion %r' % (kind,))
    return rho


def criterion_outputs(res, partials, criterion):
    """ Outputs of a residual program under a criterion: [r~] + [dr~/dr * p for p in partials], `partials` being the
    partials of the untransformed residual `res`.  dr~/dr is differentiated ONCE, on a placeholder leaf, and shared by
    all partials (instead of pushing every partial through the transform's product and quotient rules). """
    if criterion is None or criterion[0] == 'mse':
        return [res] + list(partials)
    z = var('__residual__')
    g = apply_criterion(z, criterion)
    gp = substitute(diff_leaf(g, z), {z: res})
    return [substitute(g, {z: res})] + [mul(gp, p) for p in partials]


def residual_outputs(rs, wrt, criterion):
    """ Outputs of the residual program of an equation with residual columns `rs` (m of them): the residual the kernels
    train on, then its partial w.r.t. every leaf of `wrt` (jet channels, then variables).

    One column: `criterion_outputs`, the program of a scalar equation.  Several: the reference's loss
    `criterion(residual[N, m], zeros[N, 1])` broadcasts, so it is the mean (reduction='sum': the sum) of rho(r_j) over
    all N m entries.  The kernels train on ONE residual per point, so the columns are folded into
        r~ = sqrt(s sum_j rho(r_j) + eps),   s = 1 / m (mean) or 1 (sum),
    whose per-point weight 1 / N (or 1) gives exactly that loss plus eps, and whose adjoint seed
    2 r~ dr~ = s sum_j rho'(r_j) dr_j is exact (the square root cancels, as in apply_criterion).  The derivative of r~
    w.r.t. every r_j is taken once, on placeholder leaves, and shared by all partials. """
    if len(rs) == 1:
        return criterion_outputs(rs[0], [diff_leaf(rs[0], l) for l in wrt], criterion)
    zs = [var('__residual_%d__' % j) for j in range(len(rs))]
    total = ZERO
    for z in zs:
        total = add(total, criterion_rho(z, criterion))
    scale = 1.0 if (criterion is not None and criterion[-1] == 'sum') else 1.0 / len(rs)
    g = unary('sqrt', add(mul(const(scale), total), const(CRITERION_EPS)))
    to_res = dict(zip(zs, rs))
    gps = [substitute(diff_leaf(g, z), to_res) for z in zs]
    outs = [substitute(g, to_res)]
    for leaf in wrt:
        acc = ZERO
        for gp, r in zip(gps, rs):
            p = diff_leaf(r, leaf)
            if not is_const(p, 0.0):
                acc = add(acc, mul(gp, p))
        outs.append(acc)
    return outs


def _residual_columns(out):
    """ The equation's return value as a list of per-point expressions (one per residual column). """
    if isinstance(out, VecSym):
        return list(out.exprs)
    return [out.expr if isinstance(out, Sym) else _as_expr(out)]


def _leaves_of(exprs, kinds):
    seen, found = set(), []
    for e in exprs:
        leaves(e, kinds, seen, found)
    return found


def trace(equation, total, var_factory, initial_condition=None, ndims_spatial=0, run=None, criterion=None, n_out=1,
          layout=None):
    """ Trace `equation(u, *xs)` (and `initial_condition(*x_spatial)` if callable).

    `var_factory(name)` is installed by the caller so that V(name, ...) returns `Sym(var(name))`
    during the trace.  `run` wraps the call (the Solver passes its contextvars ctx.run).
    `criterion`: see apply_criterion (default: the residual itself, MSE).
    The equation may return one column or several (`torch.cat([...], dim=1)`): see residual_outputs.
    `n_out` = k in 2..4: the network has k outputs; the equation selects component j (Components), every component
    carries the same jet set, and the residual program follows the k-output convention of include/pinn_b200.h: slot
    j*C + c holds channel c of component j on entry, and dr/d(that channel) is left in slot eq_out[1] + j*C + c.
    `layout`: a TracedEquation of order 2 whose jet set (dirs, dir_vecs, ns) is taken instead of the one the derivatives
    call for — channels nothing uses get zero partials; raises NotLowerable if a derivative has no channel there.
    """
    run = run or (lambda f, *a: f(*a))
    xs = [Sym(coord(k)) for k in range(total)]
    rs = _residual_columns(run(equation, Sym(uleaf()) if n_out == 1 else Components(n_out), *xs))
    res = rs[0]
    T = TracedEquation()
    T.residual = res
    T.n_out = n_out

    u_leaves = _leaves_of(rs, ('u',) if n_out == 1 else ('uc',))
    mis = [l.value for l in u_leaves] if n_out == 1 else [l.value[1] for l in u_leaves]
    if any(len(mi) > 2 for mi in mis):
        if n_out > 1:
            raise NotLowerable('derivatives of order > 2 of a network with several outputs')
        if layout is not None:
            raise NotLowerable('derivatives of order > 2 in a second-order jet set')
        return _trace_high_order(T, rs, u_leaves, xs, total, initial_condition, ndims_spatial, run, criterion)
    if layout is not None:
        T.dirs, T.dir_vecs, T.ns = list(layout.dirs), [list(v) for v in layout.dir_vecs], layout.ns
        nf, ns = len(T.dirs), T.ns
        # the mixed directions e_i + e_j of the layout; D nests in either order, so both multi-indices map to it
        mixed = [(d, tuple(k for k, v in enumerate(T.dir_vecs[d]) if v != 0.0)) for d in range(ns) if T.dirs[d] < 0]
        mixed += [(d, (j, i)) for d, (i, j) in mixed]
    else:
        first, second, mixed = set(), set(), set()
        for mi in mis:
            if len(mi) == 1:
                first.add(mi[0])
            elif len(mi) == 2:
                if mi[0] != mi[1]:
                    mixed.add(mi)                      # polarisation: u_ij = (u_vv - u_ii - u_jj) / 2, v = e_i + e_j
                    second.update(mi)
                else:
                    second.add(mi[0])
        first |= second
        axes2, mixed, axes1 = sorted(second), sorted(mixed), sorted(first - second)

        def unit(k, *more):
            return [1.0 if i in (k,) + more else 0.0 for i in range(total)]
        T.dir_vecs = [unit(k) for k in axes2] + [unit(i, j) for i, j in mixed] + [unit(k) for k in axes1]
        T.dirs = list(axes2) + [-1] * len(mixed) + list(axes1)
        T.ns = len(axes2) + len(mixed)
        mixed = [(len(axes2) + n, ij) for n, ij in enumerate(mixed)]
        nf, ns = len(T.dirs), T.ns
        if nf > MAX_DIRS:
            raise NotLowerable('more than %d derivative directions' % MAX_DIRS)
        if n_out > 1 and nf > 4:
            raise NotLowerable('more than 4 derivative directions in a network with several outputs')
        if nf > 4:
            # five / six directions (full Hessians in 3-D, Laplacians in 5-D / 6-D): the library holds ONE kernel per
            # direction count there, the one in which every direction carries its second derivative — first-order-only
            # directions are promoted (their second-order channel is computed and meets a zero adjoint seed)
            T.ns = ns = nf
    C = 1 + nf + ns
    mapping = {}
    for q in range(n_out):                         # component q's jet: slots q*C .. q*C + C-1
        def leaf(mi=(), q=q):
            return uleaf(mi) if n_out == 1 else ucleaf(q, mi)
        base = q * C
        mapping[leaf()] = chleaf(base)
        for d, col in enumerate(T.dirs):
            if col >= 0:
                mapping[leaf((col,))] = chleaf(base + 1 + d)
                if d < ns:
                    mapping[leaf((col, col))] = chleaf(base + 1 + nf + d)
        for d, (i, j) in mixed:
            mapping[leaf((i, j))] = mul(const(0.5), sub(sub(chleaf(base + 1 + nf + d), mapping[leaf((i, i))]),
                                                        mapping[leaf((j, j))]))
    memo = {}
    rs = [substitute(r, mapping, memo) for r in rs]
    if layout is not None and _leaves_of(rs, ('u',)):
        raise NotLowerable('a derivative has no channel in the jet set')
    res = rs[0]
    chan = {}
    by_channel = {c: chleaf(c) for c in range(n_out * C)}

    # the initial condition is traced first: its variables join the equation's (README.md:112-118)
    ic = None
    if initial_condition is not None:
        if callable(initial_condition):
            ic_out = run(initial_condition, *xs[:ndims_spatial])
            ic = ic_out.expr if isinstance(ic_out, Sym) else _as_expr(ic_out)
        else:
            ic = const(float(np.float32(initial_condition)))
        if leaves(ic, ('u',)):
            raise NotLowerable('initial_condition must not depend on the solution')
    ic_vars = {l.value for l in leaves(ic, ('var',))} if ic is not None else set()
    T.var_names = sorted({l.value for l in _leaves_of(rs, ('var',))} | ic_vars)
    if len(T.var_names) > 4:
        raise NotLowerable('more than 4 trainable variables')
    var_index = {n: i for i, n in enumerate(T.var_names)}

    outputs = residual_outputs(rs, [by_channel[c] for c in range(n_out * C)] + [var(n) for n in T.var_names], criterion)
    T.residual = apply_criterion(res, criterion) if len(rs) == 1 else outputs[0]
    T.eq_prog = lower(outputs, chan, var_index, C) if n_out == 1 else _lower_partial_block(outputs, var_index, C, n_out)
    T.n_slots = T.eq_prog.n_slots

    if ic is not None:
        def along(e, vec):                         # directional derivative sum_k v_k d/dx_k
            out = ZERO
            for k, v in enumerate(vec):
                if v != 0.0:
                    out = add(out, mul(const(v), diff_coord(e, k)))
            return out
        jet = [ic]
        firsts = [along(ic, vec) for vec in T.dir_vecs]
        jet += firsts
        jet += [along(firsts[d], T.dir_vecs[d]) for d in range(ns)]
        T.ic_has_vars = bool(ic_vars)
        base = C
        if T.ic_has_vars:               # partials w.r.t. every variable; slots above the equation's
            jet = jet + [diff_leaf(j, var(n)) for n in T.var_names for j in jet]
            base = T.eq_prog.n_slots
        T.ic_prog = lower(jet, {}, var_index, base)
        T.n_slots = max(T.n_slots, T.ic_prog.n_slots)
    return T


def _lower_partial_block(outputs, var_index, C, n_out):
    """ The residual program of a network with k = n_out outputs: `outputs` = [r, dr/d(slot s) for s < k C, dr/dV ..].
    The k C partials must form one contiguous block: slots [k C, 2 k C) are kept out of the lowering and filled by copies
    (x * 1, exact) at the end where a partial is not computed in its block slot in the first place.  Program outputs as in a one-output program: [r, the block's first C slots, dr/dV ..]. """
    kc = n_out * C
    pinned = {}
    for s in range(kc):                            # a partial met for the first time is computed in its block slot
        e = outputs[1 + s]
        if e.kind != 'ch' and e not in pinned and e is not outputs[0] and all(e is not o for o in outputs[1 + kc:]):
            pinned[e] = kc + s
    prog = lower(outputs, {}, var_index, 2 * kc, pinned)
    instrs = prog.instrs + [(OP['MULI'], kc + s, prog.outs[1 + s], 0, 1.0) for s in range(kc) if prog.outs[1 + s] != kc + s]
    if len(instrs) > MAX_PROG:
        raise NotLowerable('expression needs %d instructions (max %d)' % (len(instrs), MAX_PROG))
    return Program(instrs, [prog.outs[0]] + [kc + c for c in range(C)] + prog.outs[1 + kc:], prog.n_slots)


def _trace_high_order(T, rs, u_leaves, xs, total, initial_condition, ndims_spatial, run, criterion=None):
    """ Equations with derivatives of order 3 / 4 (D nested three / four times: u_xxx, u_xxxx): every direction carries
    its whole Taylor jet up to the highest order met (pinn_device_hi.cuh).  Directions are the differentiated
    arguments and, for every pair (i, j) with a mixed derivative, the two diagonals p = e_i + e_j and m = e_i - e_j,
    which carry it by polarisation (P_n, M_n = n-th derivative along p, m):
        u_ij = (P_2 - M_2) / 4,  u_iij = (P_3 - M_3 - 2 u_jjj) / 6,  u_ijj = (P_3 + M_3 - 2 u_iii) / 6,
        u_iijj = (P_4 + M_4 - 2 u_iiii - 2 u_jjjj) / 12      (what the biharmonic operator needs). """
    order = max(len(l.value) for l in u_leaves)
    axes, pairs = set(), set()
    for l in u_leaves:
        distinct = sorted(set(l.value))
        axes.update(distinct)
        if len(distinct) > 2:
            raise NotLowerable('mixed derivatives along three arguments next to derivatives of order > 2')
        if len(distinct) == 2:
            counts = (l.value.count(distinct[0]), l.value.count(distinct[1]))
            if max(counts) > 2:
                raise NotLowerable('mixed derivative %r is not carried by the diagonals e_i +- e_j' % (l.value,))
            pairs.add((distinct[0], distinct[1]))
    axes, pairs = sorted(axes), sorted(pairs)
    nf = len(axes) + 2 * len(pairs)
    if nf > 4:
        raise NotLowerable('derivatives of order > 2 along more than 4 directions (arguments and diagonals)')

    def vec(entries):
        return [float(entries.get(i, 0.0)) for i in range(total)]
    T.order, T.ns = order, 0
    T.dirs = list(axes) + [-1] * (2 * len(pairs))
    T.dir_vecs = [vec({k: 1.0}) for k in axes]
    for i, j in pairs:
        T.dir_vecs += [vec({i: 1.0, j: 1.0}), vec({i: 1.0, j: -1.0})]
    C = 1 + nf * order

    def ch(d, n):
        return chleaf(1 + d * order + (n - 1))
    mapping = {uleaf(): chleaf(0)}
    d_of = {col: d for d, col in enumerate(axes)}
    for col, d in d_of.items():
        for n in range(1, order + 1):
            mapping[uleaf((col,) * n)] = ch(d, n)
    for q, (i, j) in enumerate(pairs):
        dp, dm = len(axes) + 2 * q, len(axes) + 2 * q + 1
        di, dj = d_of[i], d_of[j]
        mapping[uleaf((i, j))] = mul(const(0.25), sub(ch(dp, 2), ch(dm, 2)))
        if order >= 3:
            mapping[uleaf((i, i, j))] = mul(const(1.0 / 6.0), sub(sub(ch(dp, 3), ch(dm, 3)), mul(const(2.0), ch(dj, 3))))
            mapping[uleaf((i, j, j))] = mul(const(1.0 / 6.0), sub(add(ch(dp, 3), ch(dm, 3)), mul(const(2.0), ch(di, 3))))
        if order >= 4:
            mapping[uleaf((i, i, j, j))] = mul(const(1.0 / 12.0), sub(sub(add(ch(dp, 4), ch(dm, 4)), mul(const(2.0), ch(di, 4))),
                                                                    mul(const(2.0), ch(dj, 4))))
    memo = {}
    rs = [substitute(r, mapping, memo) for r in rs]
    res = rs[0]
    if _leaves_of(rs, ('u',)):
        raise NotLowerable('a derivative of the equation has no jet channel')

    ic = None
    if initial_condition is not None:
        if callable(initial_condition):
            ic_out = run(initial_condition, *xs[:ndims_spatial])
            ic = ic_out.expr if isinstance(ic_out, Sym) else _as_expr(ic_out)
        else:
            ic = const(float(np.float32(initial_condition)))
        if leaves(ic, ('u',)):
            raise NotLowerable('initial_condition must not depend on the solution')
    ic_vars = {l.value for l in leaves(ic, ('var',))} if ic is not None else set()
    T.var_names = sorted({l.value for l in _leaves_of(rs, ('var',))} | ic_vars)
    if len(T.var_names) > 4:
        raise NotLowerable('more than 4 trainable variables')
    if 1 + C + len(T.var_names) > 2 + 2 * MAX_DIRS + 4 or (ic_vars and C * (1 + len(T.var_names)) > (1 + 2 * MAX_DIRS) * 5):
        raise NotLowerable('%d jet channels and %d variables exceed the outputs of a residual program' % (C, len(T.var_names)))
    var_index = {n: i for i, n in enumerate(T.var_names)}
    outputs = residual_outputs(rs, [chleaf(c) for c in range(C)] + [var(n) for n in T.var_names], criterion)
    T.residual = apply_criterion(res, criterion) if len(rs) == 1 else outputs[0]
    T.eq_prog = lower(outputs, {}, var_index, C)
    T.n_slots = T.eq_prog.n_slots
    if ic is not None:
        jet = [ic]
        for dvec in T.dir_vecs:
            e = ic
            for _ in range(order):
                out = ZERO
                for k, v in enumerate(dvec):
                    if v != 0.0:
                        out = add(out, mul(const(v), diff_coord(e, k)))
                e = out
                jet.append(e)
        T.ic_has_vars = bool(ic_vars)
        base = C
        if T.ic_has_vars:               # partials w.r.t. every variable; slots above the equation's (they outlive it)
            jet = jet + [diff_leaf(j, var(n)) for n in T.var_names for j in jet]
            base = T.eq_prog.n_slots
        T.ic_prog = lower(jet, {}, var_index, base)
        T.n_slots = max(T.n_slots, T.ic_prog.n_slots)
    return T


def trace_constraint(constraint, total, initial_condition=None, ndims_spatial=0, run=None, criterion=None, layout=None):
    """ Trace a constraint `constraint(u, *xs)` (reference model_torch.py:451-457: `u` is a callable that
    evaluates the model at user points, the value is driven to zero by MSE) into the same program form as an
    equation.  Lowerable when the constraint evaluates the model ONCE, at concrete points, and combines that
    value pointwise with constants / variables: `lambda u, t: u(torch.tensor([0.5]))`, `… - 2.0`, `… ** 2`.
    The value may be differentiated along a point tensor of that call, `D(u(t0), t0)` with t0 requiring grad: the
    derivative along t0's column, nested as in an equation.

    A constraint without derivatives has no derivative directions (C = 1).  One with derivatives takes the jet set of
    `layout` (the equation's TracedEquation) when that is of order 2 and carries every derivative it needs — the
    persistent kernels run such a constraint next to the equation — else its own.

    Returns (TracedEquation, the tuple of point arguments of the one call).
    """
    traced, pts = _trace_constraint(constraint, total, initial_condition, ndims_spatial, run, criterion, None)
    if traced.nf and layout is not None and layout.order == 2 and layout.n_out == 1:
        try:
            traced, pts = _trace_constraint(constraint, total, initial_condition, ndims_spatial, run, criterion, layout)
        except NotLowerable:
            pass
    return traced, pts


def _trace_constraint(constraint, total, initial_condition, ndims_spatial, run, criterion, layout):
    calls = []

    def u_at(*pts):
        if any(isinstance(p, Sym) for p in pts):
            raise NotLowerable('constraint evaluates the model at the batch points')
        if calls:
            raise NotLowerable('constraint evaluates the model more than once')
        calls.append(pts)
        return Sym(uleaf())

    _constraint_calls.append(calls)
    try:
        traced = trace(lambda _u, *xs: constraint(u_at, *xs), total, None, initial_condition=initial_condition,
                       ndims_spatial=ndims_spatial, run=run, criterion=criterion, layout=layout)
    finally:
        _constraint_calls.pop()
    if not calls:
        raise NotLowerable('constraint does not evaluate the model')
    if leaves(traced.residual, ('coord',)):
        raise NotLowerable('constraint depends on the batch points')
    return traced, calls[0]
