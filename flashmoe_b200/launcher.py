"""Multi-process harness: one worker process per GPU.

The reference shells out to `nvshmrun -n N -ppn P python worker.py <config>` (flashmoe/launcher.py:39-56); NVSHMEM's
launcher does not exist on this platform and is not needed -- peers are mapped with CUDA IPC -- so the workers are
started with torch's elastic launcher (`python -m torch.distributed.run`) on 127.0.0.1, or directly for one process.
"""
from __future__ import annotations

import os
import socket
import subprocess
import sys
from pathlib import Path
from typing import List, Optional


def _free_port() -> int:
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def build_command(config_path: str, n_processes: int, processes_per_node: int, hostfile: Optional[str] = None,
                  extra_args: Optional[List[str]] = None) -> List[str]:
    cfg = Path(config_path).resolve()
    if not cfg.exists():
        raise FileNotFoundError(f"Config file not found: {cfg}")
    worker = Path(__file__).resolve().parent / "worker.py"
    if n_processes < 1 or processes_per_node < 1:
        raise ValueError("n_processes and processes_per_node must be >= 1")
    if hostfile is not None or processes_per_node != n_processes:
        raise NotImplementedError("multi-node launches (hostfile / processes_per_node != n_processes) are out of scope: "
                                  "the dispatch/combine path is NVLink peer memory inside one NVSwitch box")
    tail = [str(worker), str(cfg)] + list(extra_args or [])
    if n_processes == 1:
        return [sys.executable] + tail
    return [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n_processes}",
            "--master-addr", "127.0.0.1", "--master-port", str(_free_port())] + tail


def launch_workers(config_path: str, n_processes: int = 1, processes_per_node: int = 1,
                   hostfile: Optional[str] = None, extra_args: Optional[List[str]] = None,
                   timeout: Optional[float] = None) -> subprocess.CompletedProcess:
    cmd = build_command(config_path, n_processes, processes_per_node, hostfile, extra_args)
    print("Launching FlashMoE (H100) with:", " ".join(cmd), flush=True)
    env = dict(os.environ)
    env["PYTHONPATH"] = str(Path(__file__).resolve().parent.parent) + os.pathsep + env.get("PYTHONPATH", "")
    res = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=timeout)
    print(res.stdout)
    if res.stderr:
        print("STDERR:", res.stderr, file=sys.stderr)
    if res.returncode != 0:
        raise subprocess.CalledProcessError(res.returncode, cmd, output=res.stdout, stderr=res.stderr)
    return res


# name kept for callers of the reference's flashmoe.launcher
nvshmrun_launcher = launch_workers
