""" The L-BFGS state machine of pinn_lbfgs.cuh, built for the host in fp64 (tests/emul/lbfgs_host.cpp), against
torch.optim.LBFGS in float64: the same evaluations per step, the same iterations, the same iterates. """
import ctypes as C
import numpy as np
import pytest
import torch

from pydens_b200 import _native as N

_lib = None


def lib():
    global _lib
    if _lib is None:
        import __graft_entry__                      # the one recipe of the host build
        _lib = C.CDLL(__graft_entry__.build_lbfgs_host())
        _lib.lbfgs_host_state_bytes.restype = C.c_size_t
        _lib.lbfgs_host_state_bytes.argtypes = [C.c_int64, C.c_int]
        _lib.lbfgs_host_vector_offset.restype = C.c_size_t
        _lib.lbfgs_host_vector_offset.argtypes = [C.c_int]
        _lib.lbfgs_host_advance.argtypes = [C.POINTER(N.PinnLbfgs), C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
    return _lib


def settings(lr=1.0, max_iter=20, max_eval=None, tolerance_grad=1e-7, tolerance_change=1e-9, history_size=100,
             line_search_fn=None):
    return dict(lr=lr, max_iter=max_iter, max_eval=max_eval, tolerance_grad=tolerance_grad,
                tolerance_change=tolerance_change, history_size=history_size, line_search_fn=line_search_fn)


class HostLbfgs:
    """ pinn_lbfgs_advance on the host: the caller's objective evaluated at `params` between two advances. """
    def __init__(self, n, mask, s, ring_len=64):
        self.n, self.mask = n, np.ascontiguousarray(mask, dtype=np.float64)
        self.state = np.zeros(lib().lbfgs_host_state_bytes(n, s['history_size']) // 8 + 1, dtype=np.float64)
        self.ring = np.zeros(ring_len, dtype=np.float32)
        self.counter = np.zeros(1, dtype=np.uint64)
        self.cfg = N.PinnLbfgs(lr=s['lr'], tolerance_grad=s['tolerance_grad'], tolerance_change=s['tolerance_change'],
                               max_iter=s['max_iter'],
                               max_eval=s['max_eval'] if s['max_eval'] is not None else s['max_iter'] * 5 // 4,
                               history_size=s['history_size'], line_search=int(s['line_search_fn'] == 'strong_wolfe'),
                               mask=self.mask.ctypes.data, losses_ring=self.ring.ctypes.data, ring_len=ring_len,
                               step_counter=self.counter.ctypes.data)

    def header(self):
        return N.PinnLbfgsState.from_buffer(self.state)

    def step(self, x, fun):
        """ One optimizer step from x (in place) -> (first loss, evaluations) """
        gl = np.zeros(self.n + 1, dtype=np.float64)
        evals, first = 0, None
        while True:
            f, g = fun(x)
            evals += 1
            first = f if first is None else first
            gl[:self.n], gl[self.n] = g, f
            st = lib().lbfgs_host_advance(C.byref(self.cfg), self.n, x.ctypes.data, gl.ctypes.data,
                                          self.state.ctypes.data, self.mask.ctypes.data)
            if st == N.LBFGS_DONE:
                return first, evals


def torch_run(x0, fun, s, steps, mask):
    """ torch.optim.LBFGS in float64 over the masked entries -> per step (loss, evaluations, n_iter), iterates """
    x = torch.tensor(x0, dtype=torch.float64)
    idx = np.flatnonzero(mask)
    p = torch.nn.Parameter(x[idx].clone())
    opt = torch.optim.LBFGS([p], **s)
    evals = [0]

    def closure():
        opt.zero_grad()
        full = x.clone()
        full[idx] = p.detach()
        f, g = fun(full.numpy())
        evals[0] += 1
        p.grad = torch.tensor(g[idx], dtype=torch.float64)
        return torch.tensor(f, dtype=torch.float64)
    out, its = [], []
    for _ in range(steps):
        evals[0] = 0
        loss = opt.step(closure)
        st = opt.state[p]
        out.append((float(loss), evals[0], int(st.get('n_iter', 0)), int(st.get('func_evals', 0))))
        full = x.clone()
        full[idx] = p.detach()
        its.append(full.numpy().copy())
    return out, its


def host_run(x0, fun, s, steps, mask):
    x = np.array(x0, dtype=np.float64)
    h = HostLbfgs(len(x), mask, s)
    out, its = [], []
    for _ in range(steps):
        loss, ev = h.step(x, fun)
        hd = h.header()
        out.append((loss, ev, int(hd.n_iter), int(hd.func_evals)))
        its.append(x.copy())
    return out, its, h


def quadratic(cond, n=12, seed=0):
    rng = np.random.default_rng(seed)
    q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = q @ np.diag(np.logspace(0, np.log10(cond), n)) @ q.T
    b = rng.standard_normal(n)
    return (lambda x: (0.5 * x @ A @ x - b @ x, A @ x - b)), rng.standard_normal(n)


def rosenbrock(x):
    f = np.sum(100.0 * (x[1:] - x[:-1] ** 2) ** 2 + (1 - x[:-1]) ** 2)
    g = np.zeros_like(x)
    g[:-1] = -400.0 * x[:-1] * (x[1:] - x[:-1] ** 2) - 2 * (1 - x[:-1])
    g[1:] += 200.0 * (x[1:] - x[:-1] ** 2)
    return f, g


def linear(x):                                   # y = 0 for every pair: ys <= 1e-10, every pair is rejected
    c = np.linspace(-1, 1, len(x))
    return float(c @ x), c.copy()


def compare(x0, fun, s, steps, mask=None, rtol=1e-8):
    mask = np.ones(len(x0)) if mask is None else mask
    ref, ref_its = torch_run(x0, fun, s, steps, mask)
    got, got_its, h = host_run(x0, fun, s, steps, mask)
    for k, (r, g) in enumerate(zip(ref, got)):
        assert g[1:] == r[1:], (k, 'evaluations / n_iter / func_evals', g, r)
        assert abs(g[0] - r[0]) <= rtol * max(1.0, abs(r[0])), (k, g[0], r[0])
    for k, (a, b) in enumerate(zip(got_its, ref_its)):
        err = np.linalg.norm(a - b) / max(1.0, np.linalg.norm(b))
        assert err <= rtol, (k, err)
    return got, h


LS = [None, 'strong_wolfe']


@pytest.mark.parametrize('ls', LS)
@pytest.mark.parametrize('history', [1, 3, 100])
@pytest.mark.parametrize('cond', [1e1, 1e4])
def test_quadratic(ls, history, cond):
    fun, x0 = quadratic(cond, seed=int(cond))
    compare(x0, fun, settings(lr=1.0 if ls else 0.1, max_iter=8, history_size=history, line_search_fn=ls), 4)


@pytest.mark.parametrize('ls', LS)
@pytest.mark.parametrize('history', [1, 3, 100])
def test_rosenbrock(ls, history):
    x0 = np.array([-1.2, 1.0, -0.5, 0.8, 1.1, 0.3])
    s = settings(lr=1.0 if ls else 1e-3, max_iter=20, history_size=history, line_search_fn=ls)
    # history 1 with the line search sits on the edge of the Rosenbrock valley: the iterates drift to 2.3e-6 by step 5
    got, _ = compare(x0, rosenbrock, s, 6, rtol=1e-6 if history > 1 or ls is None else 1e-5)


@pytest.mark.parametrize('ls', LS)
def test_ring_wraps(ls):
    """ history 3 over 40 iterations: the ring of pairs wraps many times """
    fun, x0 = quadratic(1e3, n=20, seed=3)
    _, h = compare(x0, fun, settings(lr=1.0 if ls else 0.05, max_iter=40, history_size=3, line_search_fn=ls,
                                     tolerance_grad=1e-12, tolerance_change=1e-14), 1)
    assert h.header().ring_count == 3


def test_rejected_pairs_linear():
    """ a linear objective: y = 0, so every pair is rejected and d stays -g """
    x0 = np.linspace(0, 1, 8)
    _, h = compare(x0, linear, settings(lr=0.1, max_iter=5, history_size=3), 3)
    assert h.header().ring_count == 0 and h.header().n_iter == 15


def sines(x):                                    # concave around pi/2: pairs with ys < 0 there
    return float(np.sum(np.sin(x))), np.cos(x)


@pytest.mark.parametrize('ls', LS)
def test_rejected_pairs(ls):
    x0 = np.linspace(1.3, 1.8, 6)
    # pairs of small ys next to rejected ones amplify the reassociated two-loop's rounding: the Rosenbrock bar
    compare(x0, sines, settings(lr=0.5, max_iter=12, history_size=3, line_search_fn=ls), 3, rtol=1e-6)


@pytest.mark.parametrize('ls', LS)
def test_frozen_entries(ls):
    """ masked-out entries take no part and stay where they are """
    fun, x0 = quadratic(1e2, n=10, seed=5)
    mask = np.array([1, 1, 0, 1, 1, 1, 0, 1, 1, 0], dtype=np.float64)
    compare(x0, fun, settings(lr=1.0 if ls else 0.1, max_iter=10, history_size=4, line_search_fn=ls), 3, mask=mask)


EXITS = {                                        # settings that end the step by each of torch's exits
    'opt_cond_at_entry': (lambda: (quadratic(10)[0], np.linalg.solve(*_qab(10))), settings(tolerance_grad=1e-6)),
    'max_iter': (lambda: quadratic(1e3), settings(lr=0.1, max_iter=3)),
    'max_eval': (lambda: quadratic(1e3), settings(lr=1.0, max_iter=50, max_eval=7, line_search_fn='strong_wolfe')),
    'opt_cond': (lambda: quadratic(10), settings(lr=1.0, max_iter=100, tolerance_grad=1e-5, line_search_fn='strong_wolfe')),
    'small_step': (lambda: quadratic(10), settings(lr=1e-4, max_iter=50, tolerance_change=1e-2)),
    'small_change': (lambda: quadratic(10), settings(lr=0.01, max_iter=50, tolerance_change=1e-3)),
    'gtd': (lambda: quadratic(10), settings(lr=0.1, max_iter=50, tolerance_change=1e3)),
}


def _qab(cond):
    rng = np.random.default_rng(0)
    n = 12
    q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = q @ np.diag(np.logspace(0, np.log10(cond), n)) @ q.T
    return A, rng.standard_normal(n)


@pytest.mark.parametrize('name', sorted(EXITS))
def test_exits(name):
    make, s = EXITS[name]
    fun, x0 = make()
    got, h = compare(x0, fun, s, 2)
    hd = h.header()
    if name == 'opt_cond_at_entry':
        assert hd.n_iter == 0 and got[0][1] == 1
    if name == 'max_eval':
        assert got[0][1] == 7


def test_header_layout():
    """ PinnLbfgsState / PinnLbfgs in ctypes as gcc lays them out """
    out = (C.c_int64 * 64)()
    k = lib().lbfgs_host_header_layout(out)
    names = [f[0] for f in N.PinnLbfgsState._fields_]
    assert out[0] == C.sizeof(N.PinnLbfgsState) <= N.LBFGS_HEADER_BYTES
    assert k - 1 == len(names)
    for i, name in enumerate(names):
        assert out[i + 1] == getattr(N.PinnLbfgsState, name).offset, name
    k = lib().lbfgs_host_cfg_layout(out)
    names = [f[0] for f in N.PinnLbfgs._fields_]
    assert out[0] == C.sizeof(N.PinnLbfgs) and k - 1 == len(names)
    for i, name in enumerate(names):
        assert out[i + 1] == getattr(N.PinnLbfgs, name).offset, name


@pytest.mark.parametrize('n,m', [(1, 1), (403, 10), (13000, 100)])
def test_state_layout(n, m):
    lay = N.lbfgs_layout(n, m, itemsize=8)
    assert lay['vectors'] == lib().lbfgs_host_vector_offset(m)
    assert lay['total'] == lib().lbfgs_host_state_bytes(n, m)


def test_torch_state_round_trip():
    """ a torch.optim.LBFGS state after a few steps, imported into a state buffer and exported into a fresh optimizer
    (engine.lbfgs_import / lbfgs_export), comes back in torch's layout: vectors in the optimizer's parameter order,
    the history oldest first, ro = 1 / (s . y) """
    from pydens_b200 import engine as E
    fun, x0 = quadratic(1e2, n=10, seed=7)
    x = torch.nn.Parameter(torch.tensor(x0[:6], dtype=torch.float32))
    y_ = torch.nn.Parameter(torch.tensor(x0[6:], dtype=torch.float32))
    opt = torch.optim.LBFGS([y_, x], lr=0.5, max_iter=3, history_size=3)

    def closure():
        opt.zero_grad()
        v = torch.cat([x, y_]).double().detach().numpy()
        f, g = fun(v)
        x.grad, y_.grad = torch.tensor(g[:6], dtype=torch.float32), torch.tensor(g[6:], dtype=torch.float32)
        return torch.tensor(f)
    for _ in range(3):
        opt.step(closure)
    st = opt.state[y_]
    n = 12                                           # engine layout: x at 0..5, y_ at 6..9, two entries of padding
    idx = torch.cat([torch.arange(6, 10), torch.arange(0, 6)])       # the optimizer's order: y_ first
    state = torch.zeros(N.lbfgs_layout(n, 3)['total'], dtype=torch.uint8)
    E.lbfgs_import(state, st, idx, n, 3)
    back = torch.optim.LBFGS([torch.nn.Parameter(torch.zeros(4)), torch.nn.Parameter(torch.zeros(6))], history_size=3)
    E.lbfgs_export(state, back, idx, n, 3)
    got = back.state[back.param_groups[0]['params'][0]]
    for k in ('n_iter', 'func_evals', 'prev_loss'):
        assert got[k] == st[k], k
    assert got['t'] == pytest.approx(float(st['t']), rel=1e-7)
    assert float(got['H_diag']) == pytest.approx(float(st['H_diag']), rel=1e-6)
    for k in ('d', 'prev_flat_grad'):
        assert torch.equal(got[k], st[k]), k
    assert len(got['old_dirs']) == len(st['old_dirs']) == 3
    for u, v in zip(got['old_dirs'] + got['old_stps'], st['old_dirs'] + st['old_stps']):
        assert torch.equal(u, v)
    for u, v in zip(got['ro'], st['ro']):
        assert float(u) == pytest.approx(float(v), rel=1e-5)
