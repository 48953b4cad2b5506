"""The exchange step through torch.distributed, one rank per GPU: 8 ranks on a box with eight or more GPUs, 2 on a smaller
multi-GPU box, and 1 on a single GPU, where every kind still runs end to end (symmetric allocation and rendezvous, push
kernel, peer copies, NCCL all-gather) with the rank as its own only peer.  The push kernel alone, with several mapped
destinations on one GPU, is tests/test_snowfall_gpu.py::test_gather_push_writes_kept_rows_into_every_peer_buffer."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_every_gather_kind_reassembles_the_batch_on_every_rank():
    n = torch.cuda.device_count()
    if n < 1:
        pytest.skip('no CUDA device')
    n = 8 if n >= 8 else min(n, 2)
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', f'--nproc-per-node={n}', '--master-addr', '127.0.0.1',
           '--master-port', '29533', os.path.join(ROOT, 'tools', 'check_gather_ranks.py')]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    res = json.loads(p.stdout.strip().splitlines()[-1])
    for name in ('push', 'push_unicast', 'ce', 'nccl'):
        assert res[name]['ok_on_every_rank'], res
