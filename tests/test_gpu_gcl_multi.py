"""Multi-GPU parity of the generalized contrastive loss (needs >= 2 GPUs on the box): the sharded step under torchrun
equals the oracle's R-replica simulation, with peer-memory collectives and with NCCL, and every rank ends with the same
weights and draws."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('comm', ['peer', 'nccl'])
@pytest.mark.parametrize('dist', ['logsumexp', 'normal'])
def test_two_rank_gcl_step_matches_oracle(dist, comm):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    env = dict(os.environ)
    env['SIMCLR_COMM'] = 'nccl' if comm == 'nccl' else 'peer_required'
    port = 29900 + os.getpid() % 90
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2',
           '--master-addr', '127.0.0.1', '--master-port', str(port),
           os.path.join(ROOT, 'scripts', 'gcl_multi_gpu_check.py'), dist]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    out = r.stdout + r.stderr
    lines = [l for l in out.splitlines() if l.startswith('GCL_MULTI_GPU_CHECK')]
    assert lines, out[-3000:]
    print(lines[0])
    assert '"ok": true' in lines[0], lines[0]
    assert ('"collectives": "nccl"' in lines[0]) == (comm == 'nccl'), lines[0]
    assert 'GCL_MULTI_GPU_IDENTICAL 1' in out
    assert r.returncode == 0, out[-2000:]
