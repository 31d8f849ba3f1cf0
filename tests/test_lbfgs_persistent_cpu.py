""" L-BFGS in the persistent cluster kernel, without a GPU: the ABI of pinn_lbfgs_multi / pinn_lbfgs_multi_ensemble, the
routing of fit_ensemble(optimizer='LBFGS'), and a host twin of the kernel's step loop (one batch per step, evaluations
and advances until the step is done) in fp64 against torch's float64 LBFGS. """
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from pydens_b200 import D, V, Solver, ensemble
from pydens_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJECTIVE = C.CFUNCTYPE(None, C.c_uint64, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_void_p)

_lib = None


def host_lib():
    global _lib
    if _lib is None:
        import __graft_entry__                      # the one recipe of the host build
        _lib = C.CDLL(__graft_entry__.build_lbfgs_steps_host())
        _lib.lbfgs_steps_state_bytes.restype = C.c_size_t
        _lib.lbfgs_steps_state_bytes.argtypes = [C.c_int64, C.c_int]
        _lib.lbfgs_steps_run.argtypes = [C.POINTER(N.PinnLbfgs), C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                          OBJECTIVE, C.c_void_p, C.c_void_p]
    return _lib


# ---- ABI -----------------------------------------------------------------------------------------------------------------
def test_the_entry_points_are_exported_and_bound():
    assert {'pinn_lbfgs_multi', 'pinn_lbfgs_multi_ensemble'} <= set(N.EXPORTS)
    header = open(os.path.join(ROOT, 'include', 'pinn_b200.h')).read()
    assert 'int pinn_lbfgs_multi(' in header and 'int pinn_lbfgs_multi_ensemble(' in header
    assert N.ABI_VERSION == 11


def test_member_layout_matches_gcc(tmp_path):
    out = (C.c_int64 * 16)()
    k = host_lib().lbfgs_steps_member_layout(out)
    M = N.PinnLbfgsMember
    assert list(out[:k]) == [C.sizeof(M)] + [getattr(M, f).offset for f, _ in M._fields_]
    src = tmp_path / 'm.c'                         # and as the C compiler sees the header
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pinn_b200.h"\n'
                   'int main(){printf("%zu %zu %zu\\n", sizeof(PinnLbfgsMember), offsetof(PinnLbfgsMember, seed),'
                   ' offsetof(PinnLbfgsMember, lr));return 0;}\n')
    exe = tmp_path / 'm'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    assert list(map(int, subprocess.check_output([str(exe)]).split())) == [C.sizeof(M), M.seed.offset, M.lr.offset]


# ---- the kernel's step loop on the host, against torch's float64 LBFGS ------------------------------------------------------
N_PARAMS, BATCH = 6, 8


def batch(step):
    rng = np.random.default_rng(1000 + int(step))
    return rng.normal(size=(BATCH, N_PARAMS)), rng.normal(size=BATCH)


def objective(x, step):
    """ mean_i (tanh(a_i . x) - y_i)^2 + 0.01 |x|^2 on the batch of `step`, float64 torch -> (loss, grad) """
    a, y = (torch.as_tensor(v) for v in batch(step))
    x = x.detach().clone().requires_grad_()
    f = ((torch.tanh(a @ x) - y) ** 2).mean() + 0.01 * (x ** 2).sum()
    f.backward()
    return f.detach(), x.grad


@pytest.mark.parametrize('ls', [None, 'strong_wolfe'])
@pytest.mark.parametrize('history', [2, 10])
def test_step_loop_matches_torch_lbfgs(ls, history):
    kw = dict(lr=1.0 if ls else 0.3, max_iter=6, history_size=history, line_search_fn=ls)
    x0 = torch.linspace(-0.5, 0.7, N_PARAMS, dtype=torch.float64)
    # torch: one opt.step(closure) per step, on that step's batch
    xt = torch.nn.Parameter(x0.clone())
    opt = torch.optim.LBFGS([xt], **kw)
    first = []
    n_steps = 5
    for s in range(3, 3 + n_steps):
        def closure(s=s):
            opt.zero_grad()
            f, g = objective(xt, s)
            xt.grad = g
            return f
        first.append(float(opt.step(closure)))
    st = opt.state[xt]
    # the twin: one call runs every step, the batch fixed by the step number, the counter starting at 3
    lib = host_lib()
    x = x0.numpy().copy()
    mask = np.ones(N_PARAMS)
    state = np.zeros(lib.lbfgs_steps_state_bytes(N_PARAMS, history) // 8 + 1)
    ring, counter = np.zeros(16, dtype=np.float32), np.array([3], dtype=np.uint64)
    cfg = N.PinnLbfgs(lr=kw['lr'], tolerance_grad=1e-7, tolerance_change=1e-9, max_iter=6, max_eval=6 * 5 // 4,
                      history_size=history, line_search=int(ls == 'strong_wolfe'), mask=mask.ctypes.data,
                      losses_ring=ring.ctypes.data, ring_len=16, step_counter=counter.ctypes.data)
    gl = np.zeros(N_PARAMS + 1)
    steps_seen = []

    def fun(step, params, out, ctx):
        p = torch.as_tensor(np.ctypeslib.as_array(params, shape=(N_PARAMS,)).copy())
        f, g = objective(p, step)
        o = np.ctypeslib.as_array(out, shape=(N_PARAMS + 1,))
        o[:N_PARAMS], o[N_PARAMS] = g.numpy(), float(f)
        steps_seen.append(int(step))
    cb = OBJECTIVE(fun)
    evals = lib.lbfgs_steps_run(C.byref(cfg), N_PARAMS, x.ctypes.data, state.ctypes.data, mask.ctypes.data, n_steps, cb,
                                 None, gl.ctypes.data)
    hdr = N.PinnLbfgsState.from_buffer(state)
    assert int(counter[0]) == 3 + n_steps
    assert evals == int(st['func_evals']) == hdr.func_evals and hdr.n_iter == int(st['n_iter'])
    assert sorted(set(steps_seen)) == list(range(3, 3 + n_steps)) and steps_seen == sorted(steps_seen)
    np.testing.assert_allclose(ring[3:3 + n_steps], np.array(first, dtype=np.float32), rtol=1e-6)
    # the same iterates to fp64 rounding: the Gram-entry two-loop sums in another order than torch's
    assert np.linalg.norm(x - xt.detach().numpy()) <= 1e-6 * np.linalg.norm(xt.detach().numpy())


# ---- fit_ensemble routing ------------------------------------------------------------------------------------------------
def _solver(seed):
    torch.manual_seed(seed)
    return Solver(lambda u, t: D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t) + V('c', data=torch.Tensor([1.0])),
                  ndims=1, initial_condition=1.0, layout='fafaf', features=[12, 10, 1], activation='Tanh',
                  device='cpu', seed=seed)


def stand_ins(monkeypatch, solvers, takes=lambda j: True):
    """ engines that stand in for the fused ones on a CPU device: every check before the optimizer's passes, and
    member j's L-BFGS fit runs in the cluster kernel when takes(j) """
    spec = N.PinnSpec()
    for j, s in enumerate(solvers):
        def optimizer_for(optimizer, lr, kwargs, s=s):
            if optimizer is not None:
                s._make_optimizer(optimizer, lr, **kwargs)
            return s.optimizer, False
        eng = types.SimpleNamespace(spec=spec, info=types.SimpleNamespace(small_batch_points=1024),
                                    _persistent_terms=lambda loss_terms, batch_size: [],
                                    _optimizer_for=optimizer_for,
                                    _lbfgs_persistent_terms=lambda *a, j=j: [] if takes(j) else None)
        monkeypatch.setattr(s, '_get_engine', lambda eng=eng: eng)
    monkeypatch.setattr(Solver, '_fused_possible', lambda self, criterion, loss_terms: (True, ''))
    calls = []
    monkeypatch.setattr(ensemble, 'run_lbfgs_persistent', lambda *a, **k: calls.append((a, k)))
    return calls


def together(solvers, optimizer='LBFGS', lr=1.0, k=None, **kw):
    return ensemble._fit_together(solvers, 20, 16, [None] * len(solvers), ('equation',), optimizer, torch.nn.MSELoss(),
                                  lr, k, dict(max_iter=5, **kw))


def test_lbfgs_ensemble_takes_one_launch_per_chunk(monkeypatch):
    ens = [_solver(j) for j in range(3)]
    calls = stand_ins(monkeypatch, ens)
    assert together(ens, lr=[0.1, 0.2, 0.3], line_search_fn='strong_wolfe') is None
    (args, kw), = calls
    engines, opts, _, terms, niters, batch_size, k = args
    assert kw == dict(table=True) and (niters, batch_size, k) == (20, 16, 50) and terms == []
    assert [o.param_groups[0]['lr'] for o in opts] == [0.1, 0.2, 0.3]
    assert all(type(o) is torch.optim.LBFGS and o.param_groups[0]['max_iter'] == 5 for o in opts)
    calls.clear()
    assert together(ens, k=7) is None and calls[0][0][6] == 7


def test_lbfgs_ensemble_falls_back_with_a_reason(monkeypatch):
    ens = [_solver(j) for j in range(3)]
    calls = stand_ins(monkeypatch, ens, takes=lambda j: j != 1)
    why = together(ens)
    assert why is not None and 'solver 1' in why and 'cluster kernel' in why
    monkeypatch.undo()
    calls = stand_ins(monkeypatch, ens)
    for j, s in enumerate(ens):                     # optimizer=None: each keeps its own, and they differ in max_iter
        s._make_optimizer('LBFGS', 1.0, max_iter=5 + (j == 2))
    why = together(ens, optimizer=None)
    assert why is not None and 'solver 2' in why and 'max_iter' in why and not calls
    for s in ens:
        s._make_optimizer('LBFGS', 1.0, max_iter=5)
    s0 = ens[0]
    s0._make_optimizer('LBFGS', 0.5, max_iter=5)    # lr may differ
    assert together(ens, optimizer=None) is None and len(calls) == 1


def test_mixed_optimizers_stay_on_the_adam_checks(monkeypatch):
    ens = [_solver(j) for j in range(2)]
    calls = stand_ins(monkeypatch, ens)
    why = ensemble._fit_together(ens, 20, 16, [None] * 2, ('equation',), 'SGD', torch.nn.MSELoss(), 0.1, None, {})
    assert why is not None and 'Adam' in why and not calls
