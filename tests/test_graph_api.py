"""CUDA-graph support and the device-side token count on the CPU-only legs: the new entry points in the header and the
binding table, their null-argument returns, and scripts/bench_graph.py's argument checks.  The GPU behaviour is in
test_gpu_graph.py."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

from flashmoe_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "flashmoe_b200.h")
NEW_SYMBOLS = ("fm_moe_forward_tokens_dev", "fm_last_launch")


def test_new_entry_points_are_declared_and_bound():
    text = open(HEADER).read()
    declared = set(re.findall(r"FM_API\s+[\w\s\*]+?\b(fm_\w+)\s*\(", text))
    for name in NEW_SYMBOLS:
        assert name in declared, f"{name} missing from the header"
        assert name in _lib.EXPORTED_SYMBOLS, f"{name} missing from the binding table"
    # the graph rules are written down next to the declarations
    assert "CUDA graph" in text and "fm_set_timeout_ms" in text.split("---- CUDA graphs ----")[1]


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        pytest.skip("native library not built")
    return _lib.load()


def test_null_context_and_null_count_are_rejected(lib):
    assert lib.fm_moe_forward_tokens_dev(None, None, None, None, None, None, None, None, None) == -1
    assert b"null context" in lib.fm_last_error()
    launches, n = ctypes.c_uint64(), ctypes.c_int32()
    assert lib.fm_last_launch(None, ctypes.byref(launches), ctypes.byref(n)) == -1
    assert b"null context" in lib.fm_last_error()


def test_null_count_pointer_is_rejected_before_any_cuda_call(lib):
    """A context cannot be created without a GPU; the count-pointer check comes before anything touches the context's
    device state, so a non-null dummy handle is enough to reach it."""
    dummy = ctypes.create_string_buffer(4096)
    rc = lib.fm_moe_forward_tokens_dev(ctypes.cast(dummy, ctypes.c_void_p), None, None, None, None, None, None, None, None)
    assert rc == -1 and b"n_tokens_dev" in lib.fm_last_error()


def _bench_graph(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "bench_graph.py"), *args], capture_output=True,
                          text=True, cwd=ROOT, timeout=300)


@pytest.mark.parametrize("args,flag", [
    (("--tokens", "1,4097"), "--tokens"),
    (("--tokens", "-1"), "--tokens"),
    (("--tokens", "8,x"), "--tokens"),
    (("--tokens", ""), "--tokens"),
    (("--layers", "0"), "--layers"),
    (("--steps", "0"), "--steps"),
    (("--rounds", "0"), "--rounds"),
    (("--warmup", "-1"), "--warmup"),
], ids=["above_S", "negative", "not_a_number", "empty", "no_layers", "no_steps", "no_rounds", "negative_warmup"])
def test_graph_benchmark_rejects_bad_arguments(args, flag):
    """scripts/bench_graph.py checks its arguments against the config before it needs a GPU."""
    res = _bench_graph("--config", "B", *args)
    assert res.returncode == 2, res.stdout[-2000:] + res.stderr[-2000:]
    assert flag in res.stderr and not [l for l in res.stdout.splitlines() if l.startswith("{")]
