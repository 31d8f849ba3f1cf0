""" TEST INFRASTRUCTURE: drives tests/emul/libpinn_emul_coupled.so — a g++ build of the k-output form of the per-thread
device code (pydens_b200/csrc/pinn_device.cuh, point_step / point_forward with MULTI) — so the math of networks with
2..4 outputs can be checked on CPU.  The one-output entry points stay in emul_harness.py.  Not part of the product. """
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'emul', 'pinn_emul_coupled.cpp')
LIB = os.path.join(HERE, 'emul', 'libpinn_emul_coupled.so')
DEPS = [SRC] + [os.path.join(HERE, '..', 'pydens_b200', 'csrc', f) for f in ('pinn_device.cuh', 'pinn_host_plan.h')] \
    + [os.path.join(HERE, '..', 'include', 'pinn_b200.h')]
_lib = None


def lib():
    global _lib
    if _lib is None:
        stale = (not os.path.exists(LIB)) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS)
        if stale:
            subprocess.check_call(['g++', '-O2', '-mfma', '-std=c++17', '-shared', '-fPIC', '-x', 'c++',
                                   '-Wno-unknown-pragmas', '-o', LIB, SRC])
        _lib = C.CDLL(LIB)
    return _lib


def emul_coupled_step(spec, params, points, inv_n=None):
    """ The k-output step -> (loss, residual [n], grads [n_params]). """
    params = np.ascontiguousarray(params, dtype=np.float32)
    points = np.ascontiguousarray(points, dtype=np.float32)
    n = points.shape[0]
    out = np.zeros(spec.n_params + 4, dtype=np.float32)
    res = np.zeros(n, dtype=np.float32)
    msg = C.create_string_buffer(256)
    rc = lib().emul_coupled_step(C.byref(spec), params.ctypes.data_as(C.c_void_p), points.ctypes.data_as(C.c_void_p),
                                 C.c_longlong(n), C.c_float(1.0 / n if inv_n is None else inv_n),
                                 out.ctypes.data_as(C.c_void_p), res.ctypes.data_as(C.c_void_p), msg, 256)
    if rc:
        raise RuntimeError(msg.value.decode())
    return float(out[spec.n_params]), res, out[:spec.n_params]


def emul_coupled_forward(spec, params, points):
    """ u [n, k] of a network of k outputs. """
    params = np.ascontiguousarray(params, dtype=np.float32)
    points = np.ascontiguousarray(points, dtype=np.float32)
    n, k = points.shape[0], spec.widths[spec.n_layers]
    u = np.zeros((n, k), dtype=np.float32)
    msg = C.create_string_buffer(256)
    rc = lib().emul_coupled_forward(C.byref(spec), params.ctypes.data_as(C.c_void_p), points.ctypes.data_as(C.c_void_p),
                                    C.c_longlong(n), u.ctypes.data_as(C.c_void_p), msg, 256)
    if rc:
        raise RuntimeError(msg.value.decode())
    return u
