"""Sequence-parallel forward == single-GPU forward (needs >= 2 GPUs; skipped otherwise)."""
import os
import socket
import subprocess
import sys

import pytest

from tests.conftest import ROOT

pytestmark = pytest.mark.gpu


def test_sequence_parallel_matches_single_gpu():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={min(n, 2)}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "sp_check.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert "SP_PARITY_OK" in p.stdout, (p.stdout[-2000:], p.stderr[-2000:])


def test_sequence_parallel_two_ranks_on_one_gpu():
    """Same check with both ranks on cuda:0 over gloo (NCCL refuses duplicate devices): the sharded forward incl. the
    key-range partial attention + log-sum-exp merge of the overlapped path runs on a 1-GPU box too."""
    import torch
    assert torch.cuda.device_count() >= 1
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tools", "sp_check.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, SP_ONE_GPU="1"))
    assert "SP_PARITY_OK" in p.stdout, (p.stdout[-2000:], p.stderr[-2000:])
    assert "overlapped partials" in p.stdout
