""" Drop-in checks of the public API against the reference project (analysiscenter/pydens): `Solver.reshape_and_concat`
against the reference's own classmethod, whose outputs on a fixed set of random argument mixes are stored in
tests/golden/reshape_and_concat.npz (written by oracle/make_reshape_golden.py). """
import os

import numpy as np
import pytest
import torch


def reshape_cases(n_cases=200, seed=0):
    """ Random argument mixes for `reshape_and_concat`: numbers, float32 / float64 arrays, lists, tensors, of shape
    (n,) or (n, 1).  Deterministic: the stored reference outputs are indexed by case. """
    rng = np.random.RandomState(seed)
    cases = []
    for _ in range(n_cases):
        n = int(rng.choice([1, 2, 5, 16]))
        args = []
        for _ in range(int(rng.randint(1, 5))):
            kind = int(rng.randint(7))
            if kind == 0:
                args.append(float(np.round(rng.uniform(-3, 3), 3)))
            elif kind == 1:
                args.append(int(rng.randint(-3, 4)))
            elif kind == 2:
                args.append(rng.uniform(-1, 1, size=n).astype(np.float32))
            elif kind == 3:
                args.append(rng.uniform(-1, 1, size=(n, 1)))
            elif kind == 4:
                args.append(list(np.round(rng.uniform(-1, 1, size=n), 3)))
            elif kind == 5:
                args.append(torch.tensor(rng.uniform(-1, 1, size=n), dtype=torch.float32))
            else:
                args.append(torch.tensor(rng.uniform(-1, 1, size=(n, 1)), dtype=torch.float32))
        cases.append(args)
    return cases


def test_reshape_and_concat_equals_the_reference_on_random_inputs(golden_dir):
    """ `Solver.reshape_and_concat` (reference model_torch.py:328-362) decides how `predict` and constraints read
    numbers / arrays / lists / tensors: same output as the reference's own classmethod on random argument mixes. """
    from pydens_b200 import Solver
    golden = np.load(os.path.join(golden_dir, 'reshape_and_concat.npz'))
    cases = reshape_cases()
    assert len(golden['raised']) == len(cases)
    for case, args in enumerate(cases):
        if golden['raised'][case]:                          # the reference rejects the mix: so must we
            with pytest.raises(Exception):
                Solver.reshape_and_concat(list(args))
            continue
        want = golden['out_%d' % case]
        got = Solver.reshape_and_concat(list(args))
        assert tuple(got.shape) == tuple(want.shape), (case, [type(a).__name__ for a in args])
        assert np.allclose(got.to(torch.float64).numpy(), want, rtol=1e-6, atol=1e-7), case
