""" N>1 on real GPUs (skipped with fewer than 2 devices): the sharded fit (NCCL all-reduce of the
[grads | loss] buffer, captured in the CUDA graph) follows the single-GPU fit on the same global batch. """
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(world, out, fused='1', problem='readme'):
    env = dict(os.environ, PYDENS_B200_PROGRESS='0', PYDENS_B200_FUSED_ALLREDUCE=fused)
    script = os.path.join(ROOT, 'tools', 'check_dp.py')
    if world == 1:
        cmd = [sys.executable, script, out, problem]
    else:
        cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(world),
               '--master-addr', '127.0.0.1', '--master-port', str(29600 + os.getpid() % 300), script, out, problem]
    subprocess.check_call(cmd, env=env, timeout=240)
    return json.load(open(out))


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpu_fit_matches_single_gpu(tmp_path):
    one = _run(1, str(tmp_path / 'w1.json'))
    a = np.asarray(one['losses'])
    for fused, mode in (('1', 'peer'), ('0', 'nccl')):     # in-kernel NVLink all-reduce, then plain NCCL
        two = _run(2, str(tmp_path / ('w2_%s.json' % mode)), fused)
        assert two['allreduce'] == mode
        b = np.asarray(two['losses'])
        assert a.shape == b.shape == (30,)
        assert np.max(np.abs(a - b) / np.abs(a)) <= 1e-4
        assert abs(one['params_norm'] - two['params_norm']) <= 1e-4 * one['params_norm']


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_gpu_tile_kernel_fit_matches_single_gpu(tmp_path):
    """ cfg5's network (tensor-core tile kernel, 51 KB gradient vector through the in-kernel NVLink all-reduce): the
    2-GPU fit on uneven shards of the same global batch follows the single-GPU fit. """
    one = _run(1, str(tmp_path / 'w1.json'), problem='wave3d')
    two = _run(2, str(tmp_path / 'w2.json'), problem='wave3d')
    assert one['tensor_core'] == 1 and two['tensor_core'] == 1 and two['allreduce'] == 'peer'
    a, b = np.asarray(one['losses']), np.asarray(two['losses'])
    assert a.shape == b.shape == (30,)
    assert np.max(np.abs(a - b) / np.abs(a)) <= 1e-4
    assert abs(one['params_norm'] - two['params_norm']) <= 1e-4 * one['params_norm']
