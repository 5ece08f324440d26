"""Activation recomputation at two ranks (needs >= 2 GPUs): the sharded step with every block group recomputed
equals the step without recomputation bit for bit on both ranks, through the peer-memory SyncBN, eagerly and as
the segmented graph replay (scripts/recompute_multi_gpu_check.py)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_rank_recomputed_step_is_bit_identical():
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    env = dict(os.environ, SIMCLR_COMM='peer_required')
    port = 29900 + os.getpid() % 90
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2',
           '--master-addr', '127.0.0.1', '--master-port', str(port),
           os.path.join(ROOT, 'scripts', 'recompute_multi_gpu_check.py')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    out = r.stdout + r.stderr
    lines = [l for l in out.splitlines() if l.startswith('RECOMPUTE_MULTI_GPU_CHECK')]
    assert lines, out[-3000:]
    assert '"ok": true' in lines[0], lines[0]
