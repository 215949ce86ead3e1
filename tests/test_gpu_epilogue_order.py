"""GEMM0 tiles that follow GEMM1 tiles on the same CTA share the epilogue staging area with them: h chunks are staged
there for the TMA stores and the GEMM1 epilogue transposes through it.  FM_G1_LAG=1 interleaves GEMM1 behind GEMM0, so
CTAs run GEMM1 -> GEMM0 and GEMM0 -> GEMM1 back to back.  d_model 256 gives GEMM0 tiles of 4 k-blocks (no more than the
pipeline's stages, so one consumer warpgroup can run a whole tile ahead of the other), and a capacity of 64 rows per
expert leaves the upper 64 rows of every row block empty (that warpgroup skips its GEMM1 epilogue).  Needs an H100."""
import numpy as np
import pytest

from flashmoe_b200.config import MoEConfig
from oracle import moe_oracle as mo
from tests.test_gpu_parity import _compare, _ctx
from tests.util import make_inputs, run_oracle

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fused", [1, 0])
def test_gemm1_then_gemm0_on_one_cta(monkeypatch, fused):
    # 64 experts, top-2, 2048 tokens, drop: 64 slots per expert (one row block, at most 64 valid rows);
    # 64 x (4 GEMM0 + 1 GEMM1) = 320 tiles on the 132 CTAs
    cfg = MoEConfig(num_experts=64, expert_top_k=2, sequence_len=2048, hidden_size=256, intermediate_size=1024)
    assert cfg.EC == 64
    monkeypatch.setenv("FM_G1_LAG", "1")
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    x, wg, we, _, _ = make_inputs(cfg, seed=500 + fused)
    ref = run_oracle(cfg, x, wg, we)
    ctx = _ctx(cfg)
    dev = ctx.device
    args = [t.to(dev) for t in (x, wg, we)]
    first = None
    for _ in range(3):   # three launches on the same inputs: every one must match the oracle and the first exactly
        out = ctx.forward(*args)
        ctx.synchronize()
        got = {"out": mo.to_bits(out.cpu().reshape(cfg.S, cfg.H)), "topk_idx": ctx.read("topk_idx"),
               "slot": ctx.read("slot"), "counts": ctx.read("counts"), "mcw": ctx.read("mcw"),
               "gate_out": ctx.read("gate_out"), "topk_w": ctx.read("topk_w")}
        _compare(cfg, got, ref)
        if first is None:
            first = got["out"].copy()
        else:   # both combine paths are deterministic (k = 2: two bf16 adds onto zero commute)
            assert np.array_equal(got["out"], first)
    ctx.close()
