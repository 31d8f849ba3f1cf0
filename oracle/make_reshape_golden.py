""" TEST INFRASTRUCTURE ONLY — write tests/golden/reshape_and_concat.npz from the UNMODIFIED reference.

    python oracle/make_reshape_golden.py --reference <checkout of analysiscenter/pydens>

Runs the reference's own `Solver.reshape_and_concat` (pydens/model_torch.py:328-362, imported as is through
oracle/batchflow_standin) on the argument mixes of `tests/test_reference_notebook.py: reshape_cases()` and stores,
per case, whether it raised and otherwise its output (float64, shape kept).
"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reference', required=True, help='checkout of the reference project')
    args = ap.parse_args()
    sys.path[:0] = [os.path.join(HERE, 'batchflow_standin'), os.path.abspath(args.reference), os.path.join(ROOT, 'tests')]
    import pydens as ref
    assert os.path.abspath(ref.__file__).startswith(os.path.abspath(args.reference)), ref.__file__
    from test_reference_notebook import reshape_cases
    cases = reshape_cases()
    raised = np.zeros(len(cases), dtype=bool)
    out = {}
    for i, case in enumerate(cases):
        try:
            want = ref.Solver.reshape_and_concat(list(case))
        except Exception:                                   # noqa: BLE001  (the reference rejects the mix)
            raised[i] = True
            continue
        out['out_%d' % i] = want.detach().double().numpy()
    path = os.path.join(ROOT, 'tests', 'golden', 'reshape_and_concat.npz')
    np.savez_compressed(path, raised=raised, **out)
    print('%d cases (%d rejected) -> %s' % (len(cases), int(raised.sum()), os.path.relpath(path, ROOT)))


if __name__ == '__main__':
    main()
