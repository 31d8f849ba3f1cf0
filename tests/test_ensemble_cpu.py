""" fit_ensemble without a GPU: the ctypes mirror of PinnMember matches the C layout, the member cap is the header's,
the spec comparison names the part of the problem that differs, the member checks refuse duplicates and mixed devices,
and on a CPU device fit_ensemble is the sequential `fit` of every solver. """
import ctypes as C
import os
import re
import subprocess
import types
import warnings

import numpy as np
import pytest
import torch

from pydens_b200 import _native, Solver, D, V, fit_ensemble
from pydens_b200.ensemble import check_members, member_samplers, spec_difference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'pinn_b200.h')
FIELDS = ('params', 'exp_avg', 'exp_avg_sq', 'mask', 'step_tensors', 'n_step_tensors', 'opt_step0', 'points', 'seed',
          'step_counter', 'losses_ring')


def test_pinn_member_layout_matches_c(tmp_path):
    src = tmp_path / 'member.c'
    offs = ''.join(', offsetof(PinnMember, %s)' % f for f in FIELDS)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pinn_b200.h"\n'
                   'int main(){printf("%zu' + ' %zu' * len(FIELDS) + '\\n", sizeof(PinnMember)' + offs + ');'
                   'return 0;}\n')
    exe = tmp_path / 'member'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    got = list(map(int, subprocess.check_output([str(exe)]).split()))
    M = _native.PinnMember
    assert got == [C.sizeof(M)] + [getattr(M, f).offset for f in FIELDS]


def test_member_cap_matches_the_header():
    caps = dict(re.findall(r'#define\s+(PINN_MAX_MEMBERS)\s+(\d+)', open(HEADER).read()))
    assert int(caps['PINN_MAX_MEMBERS']) == _native.MAX_MEMBERS
    assert 'pinn_multi_step_ensemble' in _native.EXPORTS


def _eq(u, t):
    return D(u, t) - 2 * np.pi * torch.cos(2 * np.pi * t) + V('new_var', data=torch.Tensor([1.0]))


def _solver(eq=_eq, features=(12, 10, 1), domain=(0, 1), ic=1.0, seed=0):
    torch.manual_seed(seed)
    return Solver(eq, ndims=1, initial_condition=ic, domain=domain, layout='fafaf', features=list(features),
                  activation='Tanh', device='cpu', seed=seed)


def _spec(s):
    chain = s.model.conv_block.dense_chain()
    widths = [s.model.total] + [c[0].out_features for c in chain]
    m = s.model
    return _native.build_spec(widths, [c[1] for c in chain], m.ndims, m.nparams, m.boundary_condition is not None,
                              m.boundary_condition or 0.0, m.raw_initial_condition is not None, m.domain, s._traced)


def test_spec_difference_names_the_part():
    base = _spec(_solver())
    assert spec_difference(base, _spec(_solver(seed=3))) is None          # another initialisation: the same problem
    assert spec_difference(base, _spec(_solver(features=(16, 10, 1)))).startswith('network')
    assert spec_difference(base, _spec(_solver(domain=(0, 2)))).startswith('domain')
    assert spec_difference(base, _spec(_solver(ic=lambda *a: V('init', data=torch.Tensor([2.0]))))).startswith('ansatz')
    other = lambda u, t: D(u, t) - 3 * torch.sin(t) + V('new_var', data=torch.Tensor([1.0]))
    assert spec_difference(base, _spec(_solver(eq=other))).startswith('equation program')


def test_member_checks():
    a, b = types.SimpleNamespace(device=torch.device('cpu')), types.SimpleNamespace(device=torch.device('cpu'))
    check_members([a, b])
    with pytest.raises(ValueError, match='no solvers'):
        check_members([])
    with pytest.raises(ValueError, match='same Solver'):
        check_members([a, b, a])
    with pytest.raises(ValueError, match='cuda'):
        check_members([a, types.SimpleNamespace(device=torch.device('cuda', 0))])
    assert member_samplers(None, 3) == [None] * 3
    assert member_samplers([1, 2], 2) == [1, 2]
    with pytest.raises(ValueError, match='3 samplers for 2 solvers'):
        member_samplers([1, 2, 3], 2)


def test_cpu_device_fits_one_after_another():
    ens = [_solver(seed=j) for j in range(3)]
    solo = [_solver(seed=j) for j in range(3)]
    torch.manual_seed(7)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        fit_ensemble(ens, niters=5, batch_size=16)
    ours = [w for w in caught if 'fit_ensemble' in str(w.message)]
    assert len(ours) == 1 and 'cpu' in str(ours[0].message)
    torch.manual_seed(7)
    for s in solo:
        s.fit(niters=5, batch_size=16)
    for a, b in zip(ens, solo):
        assert len(a.losses) == 5
        np.testing.assert_array_equal(np.array(a.losses, dtype=np.float32), np.array(b.losses, dtype=np.float32))
        for p, q in zip(a.model.parameters(), b.model.parameters()):
            assert torch.equal(p, q)
    with pytest.raises(ValueError, match='same Solver'):
        fit_ensemble([ens[0], ens[0]], niters=5, batch_size=16)
