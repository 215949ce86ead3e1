"""SwiGLU experts (hidden_act = 2) on two ranks (tests/multi_gpu_swiglu_worker.py): the router, caller and gated
routes, biases and a shared expert, every rank's out bit for bit a one-rank context's.  Skipped with fewer than two
GPUs."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_two_ranks():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "multi_gpu_swiglu_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-4000:] + "\n" + res.stderr[-4000:]
    for r in range(2):
        assert f"RANK {r} SWIGLU ALL OK" in res.stdout
