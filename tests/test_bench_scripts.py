"""The per-feature benchmark scripts (scripts/bench_*.py) on the CPU-only legs: the shared rounds loop with fake arms,
and every script's argument checks and its exit status without a CUDA device."""
import os
import subprocess
import sys

import pytest

from scripts import bench_common as common

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_rounds_warm_up_every_arm_settle_once_then_alternate():
    log = []
    arms = {k: (lambda k=k: log.append(k)) for k in "ABC"}
    name = {fn: k for k, fn in arms.items()}

    def window(fn):
        log.append("window " + name[fn])
        return len(log)

    times = common.alternate(arms, 2, 3, lambda: log.append("settle"), window)
    assert log == ["A", "A", "B", "B", "C", "C", "settle"] + [f"window {k}" for k in "ABC" * 3]
    assert times == {"A": [8, 11, 14], "B": [9, 12, 15], "C": [10, 13, 16]}

    log.clear()
    common.alternate(arms, 0, 1, lambda: log.append("settle"), window)
    assert log == ["settle", "window A", "window B", "window C"]


def test_medians_keep_every_window():
    assert common.medians({"ms": [3.0, 1.0, 2.0], "ms_b": [4.0]}) == {"ms": 2.0, "ms_runs": [3.0, 1.0, 2.0],
                                                                     "ms_b": 4.0, "ms_b_runs": [4.0]}


# Each script with a command line that is valid on its own, and the flag that names its workloads (if any).
SCRIPTS = {
    "bench_varlen.py": (["--tokens", "1"], None),
    "bench_graph.py": ([], None),
    "bench_routed.py": ([], "--configs"),
    "bench_gated.py": ([], "--configs"),
    "bench_shared.py": ([], "--configs"),
    "bench_swiglu.py": ([], "--shapes"),
}


def _run(script, *args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")   # no device, also on a machine that has one
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", script), *SCRIPTS[script][0], *args],
                          capture_output=True, text=True, cwd=ROOT, env=env, timeout=300)


def _json_lines(res):
    return [l for l in res.stdout.splitlines() if l.startswith("{")]


BAD = [pytest.param(script, args, args[0], id=f"{script[:-3]}-{what}") for script in sorted(SCRIPTS)
       for what, args in [("bad_tokens", ("--tokens", "8,x")), ("no_steps", ("--steps", "0"))]]
BAD += [pytest.param(script, (flag, "nope"), flag, id=f"{script[:-3]}-unknown_workload")
        for script, (_, flag) in sorted(SCRIPTS.items()) if flag]


@pytest.mark.parametrize("script,args,flag", BAD)
def test_bad_arguments_exit_2_naming_the_flag(script, args, flag):
    res = _run(script, *args)
    assert res.returncode == 2, res.stdout[-2000:] + res.stderr[-2000:]
    assert flag in res.stderr and not _json_lines(res)


@pytest.mark.parametrize("script", sorted(SCRIPTS))
def test_without_a_cuda_device_exit_3_and_print_no_result(script):
    res = _run(script)
    assert res.returncode == 3, res.stdout[-2000:] + res.stderr[-2000:]
    assert "no CUDA device" in res.stderr and not _json_lines(res)
