""" pydens_b200 — H100-native engine behind the pydens API.

Same import surface as the reference package (pydens/__init__.py:4-5):
`Solver, D, V, TorchModel, ConvBlockModel` + the sampler names (`NumpySampler`, …).
The fit step runs in hand-written sm_90a CUDA (libpinn_b200.so, C ABI in include/pinn_b200.h).
"""
from .model import D, V, TorchModel, ConvBlockModel, current_model
from .solver import Solver
from .sampler import *            # noqa: F401,F403  (NumpySampler, ConstantSampler, Sampler)

__version__ = '1.0.2+b200.1'
