"""Expert parallelism: every scenario of tests/multi_gpu_worker.py under torch.distributed.run, with the library's
CUDA-IPC slab or torch symmetric memory (torch.distributed._symmetric_memory -> fm_symm_use_external +
fm_symm_attach_ptrs).  Every scenario also runs on one rank, so its code runs on a one-GPU machine; a run with more
ranks than GPUs is skipped.  Without a GPU: every scenario's token counts build for 1, 2, 4 and 8 ranks, and the table
below names exactly the worker's scenarios."""
import os
import signal
import socket
import subprocess
import sys

import pytest

from tests import multi_gpu_worker as worker

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMEOUT_S = 600

WORLDS = {   # scenario: (worlds past 1, slabs)
    "parity": ((2, 4, 8), ("ipc",)),
    "parity_small": ((2,), ("torch",)),
    "routed": ((2, 4), ("ipc", "torch")),
    "varlen": ((2, 4), ("ipc", "torch")),
    "graph": ((2, 4), ("ipc",)),
    "shared": ((2,), ("ipc",)),
    "swiglu": ((2,), ("ipc",)),
    "weight_on_input": ((2,), ("ipc",)),
}
RUNS = [(s, 1, "ipc") for s in WORLDS] + [(s, w, symm) for s, (worlds, slabs) in WORLDS.items()
                                          for w in worlds for symm in slabs]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _signal_group(proc, sig):
    try:
        os.killpg(proc.pid, sig)
    except ProcessLookupError:
        pass


def torchrun(scenario, world, symm):
    """Run one scenario on `world` ranks with the `symm` slab and return its stdout.  torchrun starts every rank in a
    session of its own and, on SIGTERM, stops them (SIGKILL after 30 s) before it exits.  So a run that times out gets
    SIGTERM, and SIGKILL a minute later if torchrun is still alive; both go to the process group that torchrun leads in
    its own session."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "multi_gpu_worker.py"), scenario]
    proc = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, cwd=ROOT,
                            env=dict(os.environ, FM_SYMM=symm), start_new_session=True)
    try:
        out, err = proc.communicate(timeout=TIMEOUT_S)
    except subprocess.TimeoutExpired:
        _signal_group(proc, signal.SIGTERM)
        try:
            out, err = proc.communicate(timeout=60)
        except subprocess.TimeoutExpired:
            _signal_group(proc, signal.SIGKILL)
            out, err = proc.communicate()
        pytest.fail(f"timed out after {TIMEOUT_S} s\n{out[-4000:]}\n{err[-4000:]}")
    assert proc.returncode == 0, out[-4000:] + "\n" + err[-4000:]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("scenario,world,symm", RUNS)
def test_expert_parallel(scenario, world, symm):
    import torch

    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    out = torchrun(scenario, world, symm)
    for r in range(world):
        assert f"RANK {r} {scenario} ALL OK" in out


def test_table_names_the_worker_scenarios():
    assert set(WORLDS) == set(worker.SCENARIOS)


@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("scenario", list(WORLDS))
def test_token_counts(scenario, world):
    cases, counts_of, _ = worker.SCENARIOS[scenario]
    for ci, entry in enumerate(cases):
        cfg = worker.config(entry)
        if cfg.E % world:
            continue
        for rank in range(world):
            counts = counts_of(worker.Case(ci, cfg, entry, rank, world))
            assert counts and all(0 <= n <= cfg.S for n in counts), (ci, rank, counts)
