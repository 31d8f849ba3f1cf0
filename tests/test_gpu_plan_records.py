""" Every plan places and launches what tests/golden/plan_records.json recorded, bit for bit: for every registry problem
and placement override, the plan-creation return code, PinnPlanInfo, the workspace size, and the digests of one call of
pinn_step, pinn_step_adam, pinn_forward and (where they exist) the persistent kernels.  See tools/plan_records.py. """
import json
import os

import pytest
import torch

from tools import plan_records as R

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'plan_records.json')


def _fixture():
    with open(FIXTURE) as f:
        return json.load(f)


@pytest.mark.parametrize('name', R.names())
def test_plan_records_match_fixture(name):
    fx = _fixture()
    if R.device() != fx['device']:
        pytest.skip('the fixture was recorded on %s' % fx['device'])
    assert torch.cuda.is_available()
    want = fx['records'][name]
    got = R.problem_records(name)
    for o in R.OVERRIDES:
        assert got[o] == want[o], '%s under %s' % (name, o)
