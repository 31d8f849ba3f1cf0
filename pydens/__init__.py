""" Drop-in alias: `from pydens import Solver, D, V, NumpySampler` resolves to the H100 engine, so
notebooks written against analysiscenter/pydens run unchanged. """
from pydens_b200 import *                                   # noqa: F401,F403
from pydens_b200 import Solver, D, V, TorchModel, ConvBlockModel, __version__   # noqa: F401
from pydens_b200 import model as model_torch                # noqa: F401  (pydens.model_torch.* lookups)
