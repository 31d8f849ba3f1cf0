""" Per-member Adam hyper-parameters of fit_ensemble without a GPU: the ctypes mirror of PinnAdamHyper matches the C
layout, pinn_multi_step_ensemble_adam is declared and exported, a per-member sequence of the wrong length is refused
before anything trains, and on a CPU device an lr sweep is the sequential `fit` of every solver with its own lr. """
import ctypes as C
import os
import re
import subprocess
import warnings

import numpy as np
import pytest
import torch

from pydens_b200 import _native, fit_ensemble
from pydens_b200.ensemble import member_hyper
from test_ensemble_cpu import HEADER, ROOT, _solver

FIELDS = ('lr', 'beta1', 'beta2', 'eps', 'weight_decay')


def test_pinn_adam_hyper_layout_matches_c(tmp_path):
    src = tmp_path / 'hyper.c'
    offs = ''.join(', offsetof(PinnAdamHyper, %s)' % f for f in FIELDS)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pinn_b200.h"\n'
                   'int main(){printf("%zu' + ' %zu' * len(FIELDS) + '\\n", sizeof(PinnAdamHyper)' + offs + ');'
                   'return 0;}\n')
    exe = tmp_path / 'hyper'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = list(map(int, subprocess.check_output([str(exe)]).split()))
    H = _native.PinnAdamHyper
    assert got == [C.sizeof(H)] + [getattr(H, f).offset for f in FIELDS]


def test_entry_point_is_declared_and_exported():
    text = open(HEADER).read()
    assert re.search(r'int\s+pinn_multi_step_ensemble_adam\s*\(', text)
    assert 'pinn_multi_step_ensemble_adam' in _native.EXPORTS
    lib = C.CDLL(_native.LIB_PATH)                       # built by build(); loading it needs no device
    assert hasattr(lib, 'pinn_multi_step_ensemble_adam')


def test_member_hyper_spreads_values():
    lrs, kws = member_hyper(2, 0.01, dict(betas=(0.9, 0.99), eps=1e-7))
    assert lrs == [0.01, 0.01] and kws == [dict(betas=(0.9, 0.99), eps=1e-7)] * 2
    lrs, kws = member_hyper(2, np.array([0.1, 0.2]), dict(betas=[(0.9, 0.99), (0.0, 0.9)], weight_decay=[0.0, 1e-3],
                                                          amsgrad=False))
    assert lrs == [0.1, 0.2]
    assert kws == [dict(betas=(0.9, 0.99), weight_decay=0.0, amsgrad=False),
                   dict(betas=(0.0, 0.9), weight_decay=1e-3, amsgrad=False)]


@pytest.mark.parametrize('kw', [dict(lr=[0.1, 0.2]), dict(eps=[1e-8] * 4), dict(weight_decay=[0.0]),
                                dict(betas=[(0.9, 0.999)] * 2)])
def test_wrong_length_raises_before_training(kw):
    ens = [_solver(seed=j) for j in range(3)]
    name = next(iter(kw))
    with pytest.raises(ValueError, match='values of %s for 3 solvers' % name):
        fit_ensemble(ens, niters=5, batch_size=16, **kw)
    assert all(s.losses == [] and s.optimizer is None for s in ens)


def test_cpu_lr_sweep_fits_one_after_another():
    lrs = [0.001, 0.005, 0.02]
    betas = [(0.9, 0.999), (0.0, 0.99), (0.8, 0.9)]
    ens = [_solver(seed=j) for j in range(3)]
    solo = [_solver(seed=j) for j in range(3)]
    torch.manual_seed(7)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        fit_ensemble(ens, niters=5, batch_size=16, lr=lrs, betas=betas)
    ours = [w for w in caught if 'fit_ensemble' in str(w.message)]
    assert len(ours) == 1 and 'cpu' in str(ours[0].message)
    torch.manual_seed(7)
    for s, lr, b in zip(solo, lrs, betas):
        s.fit(niters=5, batch_size=16, lr=lr, betas=b)
    for a, b, lr, bt in zip(ens, solo, lrs, betas):
        g = a.optimizer.param_groups[0]
        assert g['lr'] == lr and tuple(g['betas']) == bt
        np.testing.assert_array_equal(np.array(a.losses, dtype=np.float32), np.array(b.losses, dtype=np.float32))
        for p, q in zip(a.model.parameters(), b.model.parameters()):
            assert torch.equal(p, q)
