"""Caller routing (fm_moe_forward_routed / MoEContext.forward_routed) on the CPU-only legs: the C-ABI declaration and
binding, the entry point's argument checks that need no context, and the two test references -- the torch statement
(tests/torch_routed.py) against the float64 exact-input one (tests/exact.py).  The GPU behaviour is in
test_gpu_routed.py."""
import os

import numpy as np
import pytest
import torch

from flashmoe_b200 import _lib
from flashmoe_b200.config import MoEConfig
from tests import exact as ex
from tests.torch_routed import INT32_MAX, moe_forward_routed_cpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_and_binding_exports_the_routed_entry_point():
    with open(os.path.join(ROOT, "include", "flashmoe_b200.h")) as f:
        header = f.read()
    assert "FM_API int fm_moe_forward_routed(" in header
    assert "fm_moe_forward_routed" in _lib.EXPORTED_SYMBOLS


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        pytest.skip("native library not built")
    return _lib.load()


def test_routed_call_rejects_a_null_context(lib):
    assert lib.fm_moe_forward_routed(None, None, 0, None, None, None, None, None, None, None, None) == -1
    assert b"null context" in lib.fm_last_error()
    assert lib.fm_moe_forward_routed(None, None, -1, None, None, None, None, None, None, None, None) == -1


def test_slots_from_routing_skips_minus_one():
    topk = np.array([[0, -1], [0, 0], [-1, -1], [1, 0]], np.int32)
    slot, counts, recv_cnt, kept = ex.slots_from_routing(topk, E=2, EC=2)
    assert slot.tolist() == [[0, INT32_MAX], [1, 2], [INT32_MAX, INT32_MAX], [0, 3]]
    assert counts.tolist() == [4, 1] and recv_cnt.tolist() == [2, 1]
    assert kept.tolist() == [[True, False], [True, False], [False, False], [True, False]]


def test_combine_routed_scales_k1_and_accumulates_in_pick_order():
    y = ex.f64_to_bf16(np.array([[[1.0, -3.0]], [[2.0, 0.5]]]))           # [n=2, k=1, H=2]
    w = ex.f32_to_bf16(np.array([[0.5], [3.0]], np.float32))
    out = ex.combine_routed(y, np.array([[True], [False]]), w)
    assert ex.bits_to_f64(out).tolist() == [[0.5, -1.5], [0.0, 0.0]]
    assert out[1].tolist() == [0, 0]                                      # +0, not -0
    # 256 + 1 + 1 in pick order rounds each add: (256 + 1 -> 256) + 1 -> 256, not 258
    y3 = ex.f64_to_bf16(np.array([[[256.0], [1.0], [1.0]]]).reshape(1, 3, 1))
    w3 = ex.f32_to_bf16(np.ones((1, 3), np.float32))
    assert ex.bits_to_f64(ex.combine_routed(y3, np.ones((1, 3), bool), w3)).tolist() == [[256.0]]


CASES = {
    "k1": (MoEConfig(num_experts=8, expert_top_k=1, sequence_len=128, hidden_size=128, intermediate_size=128), {}),
    "k2_bias": (MoEConfig(num_experts=8, expert_top_k=2, sequence_len=128, hidden_size=128, intermediate_size=192),
                dict(bias=True)),
    "k3_no_drop": (MoEConfig(num_experts=4, expert_top_k=3, sequence_len=128, hidden_size=64, intermediate_size=128,
                             drop_tokens=0), {}),
}


@pytest.mark.parametrize("name", list(CASES))
def test_torch_routed_forward_equals_exact_reference(name):
    cfg, gen = CASES[name]
    inp = ex.exact_inputs(cfg, seed=7000 + len(name), **gen)
    for n in (cfg.S, 37):
        topk, w = ex.routing_case(n, cfg.E, cfg.k, seed=n, hot=1, empty=(cfg.E - 1,),
                                  bad=[(3, 0, cfg.E), (5, cfg.k - 1, -7)])
        EC = cfg.EC_of(n)
        ref = ex.reference_launch("routed", inp, EC, n, routing=(topk, w))[0].out
        xp = inp.experts
        got = moe_forward_routed_cpu(inp.x.reshape(-1, cfg.H)[:n], torch.from_numpy(topk), torch.from_numpy(w), xp.w,
                                     EC=EC, act=0, bias_up=xp.bu, bias_down=xp.bd)
        ex.check_equal(ex.to_bits(got["out"]), ref, f"{name} n={n} out", ("token", "column"), signed_zero=False)
        run = ex.sanitize(topk, cfg.E)
        slot, counts, _, kept = ex.slots_from_routing(run, cfg.E, EC)
        assert (got["topk_idx"].numpy() == run).all() and (got["slot"].numpy() == slot).all()
        assert (got["counts"].numpy() == counts).all() and (got["kept"].numpy() == kept).all()
        # the case exercises what it is meant to: skips, duplicates, a dropped pick, an expert with nothing
        assert (run == -1).any() and counts[cfg.E - 1] == 0
        if cfg.drop_tokens:
            assert (~kept & (run >= 0)).any()
        if cfg.k > 1:
            assert (run[:, 0] == run[:, 1])[run[:, 0] >= 0].any()
