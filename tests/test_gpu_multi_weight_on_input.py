"""The router weight on the input with expert parallelism on 2 GPUs: one rank with the setting on, the other off, each
equal bit for bit to a one-GPU context holding all experts with its own setting.  Skipped with fewer than 2 GPUs."""
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


def test_ranks_with_different_settings():
    import torch

    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()),
           os.path.join(ROOT, "tests", "multi_gpu_weight_on_input_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-4000:] + "\n" + res.stderr[-4000:]
    for r in range(world):
        assert f"RANK {r} WEIGHT ON INPUT ALL OK" in res.stdout
