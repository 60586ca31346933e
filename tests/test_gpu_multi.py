"""N-GPU == 1-GPU equivalence (HOPE row sharding, node2vec walk sharding) -- needs >= 2 GPUs; skipped
on a machine with one GPU.  The check itself is scripts/mgpu_check.py, launched with torchrun."""
import json
import os
import socket
import subprocess
import sys

import pytest

from conftest import REPO

pytestmark = pytest.mark.gpu


def test_two_gpu_equivalence(native_lib):
    n = native_lib.gemb_device_count()
    if n < 2:
        pytest.skip('needs >= 2 GPUs')
    s = socket.socket(); s.bind(('127.0.0.1', 0)); port = s.getsockname()[1]; s.close()
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2',
           '--master-addr', '127.0.0.1', '--master-port', str(port), os.path.join(REPO, 'scripts/mgpu_check.py')]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    line = [l for l in p.stdout.splitlines() if l.startswith('{')]
    assert p.returncode == 0 and line, p.stdout[-2000:] + p.stderr[-2000:]
    assert json.loads(line[-1])['ok']
