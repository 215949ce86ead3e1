"""Expert parallelism on the caller's routing (MoEContext.forward_routed), on 2 and 4 GPUs, with the library's CUDA-IPC
slab and with torch symmetric memory: every rank passes its own routing and its own token count.  Skipped with fewer
GPUs than the world size."""
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


@pytest.mark.parametrize("symm", ["ipc", "torch"])
@pytest.mark.parametrize("world", [2, 4])
def test_per_rank_routing(world, symm):
    import torch

    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    env = dict(os.environ)
    env["FM_SYMM"] = symm
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "multi_gpu_routed_worker.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert res.returncode == 0, res.stdout[-4000:] + "\n" + res.stderr[-4000:]
    for r in range(world):
        assert f"RANK {r} ROUTED ALL OK" in res.stdout
