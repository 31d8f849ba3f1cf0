""" The compact per-point layout of the twelve-warp thread kernel (build_remat_plan in pinn_host_plan.h,
point_step<…, REMAT0 = true>), on the host build of the device code.  The layout keeps no row of the first layer's jet
(the forward pass builds it in rows the second hidden layer takes over later, the reverse pass rebuilds it) and puts the
output layer's adjoint into the program's scratch rows, so the arithmetic is that of the plan's own layout: the loss,
residual and every gradient must come out bit for bit the same, on the goldens' networks and on networks at the
block edges of the forward (16 columns) and reverse (4 rows x 8 columns) passes.  Residual layouts, oblique
directions, variables in the initial condition and networks of one hidden layer keep the plan's layout.
The GPU side is tests/test_gpu_occupancy.py. """
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import problems as P
import emul_harness as E

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'emul', 'pinn_emul_remat.cpp')

ORDER2 = [n for n in P.PROBLEMS if n not in P.HI_ORDER and n not in P.HI_DIRECTION]
# (base problem, hidden widths): the edges of the forward blocks (16 units) and of the reverse blocks (8 columns, 4 rows)
EDGES = [('poisson2d', [1, 1, 1]), ('poisson2d', [8, 7, 9]), ('poisson2d', [16, 17, 15]), ('poisson2d', [9, 16, 4]),
         ('poisson2d', [3, 33, 8, 5]), ('heat_param', [17, 8]), ('nonlinear', [12, 9, 13])]
REFUSED = ['poisson_skip', 'heat_resnet', 'mixed2d', 'heat1d_icvar', 'poisson_sin']


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('remat') / 'libremat.so')
    subprocess.check_call(['g++', '-O2', '-mfma', '-std=c++17', '-shared', '-fPIC', '-x', 'c++', '-Wno-unknown-pragmas',
                           '-o', out, SRC])
    return C.CDLL(out)


def _rows(lib, spec):
    rows = (C.c_int * 2)()
    msg = C.create_string_buffer(256)
    assert lib.remat_rows(C.byref(spec), rows, msg, 256) == 0, msg.value
    return rows[0], rows[1]


def _step(lib, spec, compact, params, points):
    params = np.ascontiguousarray(params, dtype=np.float32)
    points = np.ascontiguousarray(points, dtype=np.float32)
    out = np.zeros(spec.n_params + 4, dtype=np.float32)
    res = np.zeros(points.shape[0], dtype=np.float32)
    msg = C.create_string_buffer(256)
    rc = lib.remat_step(C.byref(spec), C.c_int(compact), params.ctypes.data_as(C.c_void_p),
                        points.ctypes.data_as(C.c_void_p), C.c_longlong(points.shape[0]), out.ctypes.data_as(C.c_void_p),
                        res.ctypes.data_as(C.c_void_p), msg, 256)
    assert rc == 0, msg.value
    return out, res


def _variant(monkeypatch, base, widths):
    name = '%s_%s' % (base, '_'.join(map(str, widths)))
    cfg = dict(P.PROBLEMS[base], features=list(widths) + [1])
    cfg['layout'] = 'fa' * len(widths) + 'f'
    monkeypatch.setitem(P.PROBLEMS, name, cfg)
    return name


def test_cfg2_rows(lib):
    """ cfg2 ([2, 10, 12, 15, 1], five jet channels, 8 scratch slots): 2 + 5 (12 + 15) + max(8, 10) = 147 rows, which
    twelve warps fit in the H100's 227 KB of shared memory next to the staged weights (148 is the most that fits);
    the plan's own layout has 200 """
    assert _rows(lib, E.spec_for('poisson2d')) == (200, 147)


@pytest.mark.parametrize('name', ORDER2)
def test_compact_layout_is_bit_identical(lib, name):
    spec = E.spec_for(name)
    rows, rows_c = _rows(lib, spec)
    if name in REFUSED:
        assert rows_c == -1, '%s: the compact layout must not apply' % name
        return
    if rows_c == -1:
        pytest.skip('the compact layout does not apply to this plan')
    assert rows_c < rows
    rng = np.random.RandomState(7)
    params = rng.uniform(-0.8, 0.8, size=spec.n_params).astype(np.float32)
    points = P.make_points(name, 100, seed=11)
    out0, res0 = _step(lib, spec, 0, params, points)
    out1, res1 = _step(lib, spec, 1, params, points)
    assert np.isfinite(out0).all() and np.isfinite(res0).all()
    assert np.array_equal(out0, out1), 'gradients differ in %d entries' % int((out0 != out1).sum())
    assert np.array_equal(res0, res1)
    # and the plan's layout here is the emulation harness's
    loss, res, grads = E.emul_step(spec, params, points)
    assert np.array_equal(res, res0) and np.array_equal(grads, out0[:spec.n_params])


@pytest.mark.parametrize('base,widths', EDGES)
def test_compact_layout_at_block_edges(lib, monkeypatch, base, widths):
    name = _variant(monkeypatch, base, widths)
    spec = E.spec_for(name)
    rows, rows_c = _rows(lib, spec)
    assert 0 < rows_c < rows
    rng = np.random.RandomState(3)
    params = rng.uniform(-0.9, 0.9, size=spec.n_params).astype(np.float32)
    points = P.make_points(name, 67, seed=5)
    out0, res0 = _step(lib, spec, 0, params, points)
    out1, res1 = _step(lib, spec, 1, params, points)
    assert np.isfinite(out0).all()
    assert np.array_equal(out0, out1) and np.array_equal(res0, res1)
