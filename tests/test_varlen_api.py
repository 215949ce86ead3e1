"""Per-call token count (MoEContext.forward_tokens / fm_moe_forward_tokens) on the CPU-only legs: the capacity helper, the
C-ABI entry point's argument checks, and scripts/bench_varlen.py's argument checks.  The GPU behaviour is in
test_gpu_varlen.py."""
import os
import subprocess
import sys

import pytest

from flashmoe_b200 import _lib
from flashmoe_b200.config import BASELINE_CONFIGS, MoEConfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", sorted(BASELINE_CONFIGS))
def test_capacity_of_n_tokens_matches_the_config_at_S(name):
    cfg = BASELINE_CONFIGS[name]
    assert cfg.EC_of(cfg.S) == cfg.EC
    assert cfg.EC_of(0) == 0


def test_capacity_of_n_tokens_is_that_of_a_config_with_S_equal_n():
    for drop in (0, 1):
        base = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, capacity_factor=2, drop_tokens=drop)
        for n in (1, 7, 8, 9, 129, 300, 512):
            assert base.EC_of(n) == base.replace(sequence_len=n).EC
    assert MoEConfig(num_experts=8, expert_top_k=2).EC_of(16) == 4   # ceil(16 / 8) * 1 * 2


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        pytest.skip("native library not built")
    return _lib.load()


def test_forward_tokens_rejects_a_null_context(lib):
    assert lib.fm_moe_forward_tokens(None, None, 0, None, None, None, None, None, None) == -1
    assert b"null context" in lib.fm_last_error()
    assert lib.fm_moe_forward_tokens(None, None, -1, None, None, None, None, None, None) == -1


def _bench_varlen(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "bench_varlen.py"), *args], capture_output=True,
                          text=True, cwd=ROOT, timeout=300)


@pytest.mark.parametrize("tokens", ["1,4097", "-1", "8,x", ""])
def test_varlen_benchmark_rejects_bad_token_lists(tokens):
    """scripts/bench_varlen.py checks its token counts against the config's S before it needs a GPU."""
    res = _bench_varlen("--config", "B", "--tokens", tokens)
    assert res.returncode == 2, res.stdout[-2000:] + res.stderr[-2000:]
    assert "--tokens" in res.stderr and not [l for l in res.stdout.splitlines() if l.startswith("{")]
