"""Expert parallelism through replayed CUDA graphs with a device-side token count per rank, on 2 and 4 GPUs
(tests/multi_gpu_graph_worker.py).  Skipped with fewer GPUs than the world size."""
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


@pytest.mark.parametrize("world", [2, 4])
def test_device_count_graphs_on_every_rank(world):
    import torch

    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "multi_gpu_graph_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert res.returncode == 0, res.stdout[-4000:] + "\n" + res.stderr[-4000:]
    for r in range(world):
        assert f"RANK {r} GRAPH ALL OK" in res.stdout
