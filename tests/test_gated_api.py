"""Gated routing (fm_moe_forward_gated / MoEContext.forward_gated) on the CPU-only legs: the C-ABI declaration, struct
layout and binding, the null-context check, RouterSpec's checks, and the torch statement of the routing rule
(tests/torch_gated.py) against a float64 numpy one, on random tie-free inputs and on hand-built cases for each rule.
The GPU behaviour is in test_gpu_gated.py."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from flashmoe_b200 import _lib
from flashmoe_b200.router import RouterSpec
from tests.torch_gated import gated_routing_cpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header() -> str:
    with open(os.path.join(ROOT, "include", "flashmoe_b200.h")) as f:
        return f.read()


def test_header_declares_and_binding_exports_the_gated_entry_point():
    assert "FM_API int fm_moe_forward_gated(" in _header()
    assert "fm_moe_forward_gated" in _lib.EXPORTED_SYMBOLS


def test_router_struct_layout_matches_the_header():
    body = _header().split("typedef struct fm_router {")[1].split("} fm_router_t;")[0]
    fields = re.findall(r"(int32_t|float)\s+(\w+);", body)
    assert [name for _, name in fields] == [name for name, _ in _lib.FmRouter._fields_]
    types = {"int32_t": ctypes.c_int32, "float": ctypes.c_float}
    assert [types[t] for t, _ in fields] == [t for _, t in _lib.FmRouter._fields_]
    assert ctypes.sizeof(_lib.FmRouter) == 24
    assert [getattr(_lib.FmRouter, n).offset for n, _ in _lib.FmRouter._fields_] == [0, 4, 8, 12, 16, 20]


@pytest.fixture(scope="module")
def lib():
    if not _lib.LIB_PATH.exists():
        pytest.skip("native library not built")
    return _lib.load()


def test_gated_call_rejects_a_null_context(lib):
    r = RouterSpec().to_c()
    assert lib.fm_moe_forward_gated(None, None, 0, None, None, ctypes.byref(r), None, None, None, None, None,
                                    None) == -1
    assert b"null context" in lib.fm_last_error()


@pytest.mark.parametrize("kw", [dict(scoring="tanh"), dict(n_group=0), dict(n_group=33), dict(n_group=4, topk_group=0),
                                dict(n_group=4, topk_group=5), dict(n_group=4, topk_group=2, group_top=3),
                                dict(renormalize=2), dict(scale=0.0), dict(scale=-1.0), dict(scale=math.inf),
                                dict(scale=math.nan), dict(n_group=2.0)])
def test_router_spec_rejects_each_invalid_field(kw):
    with pytest.raises(ValueError):
        RouterSpec(**kw)


def test_router_spec_context_checks():
    RouterSpec("sigmoid", 8, 4, 2, True, 2.5).check(256, 8)
    with pytest.raises(ValueError, match="divide"):
        RouterSpec(n_group=3, topk_group=1).check(8, 2)
    with pytest.raises(ValueError, match="group size"):
        RouterSpec(n_group=8, topk_group=4, group_top=2).check(8, 2)
    with pytest.raises(ValueError, match="k=5"):
        RouterSpec(n_group=4, topk_group=2).check(8, 5)
    c = RouterSpec("sigmoid", 4, 2, 2, False, 2.5).to_c()
    assert (c.scoring, c.n_group, c.topk_group, c.group_top, c.renormalize, c.scale) == (1, 4, 2, 2, 0, 2.5)


# ----------------------------------------------------------------------------- float64 statement
def gated_routing_f64(logits: np.ndarray, router: RouterSpec, k: int, bias=None):
    """The same contract in float64 numpy, one token at a time."""
    n, E = logits.shape
    l = logits.astype(np.float64)
    if router.scoring == "softmax":
        z = np.exp(l - l.max(axis=1, keepdims=True))
        s = z / z.sum(axis=1, keepdims=True)
    else:
        s = 1.0 / (1.0 + np.exp(-l))
    c = s + (np.zeros(E) if bias is None else np.asarray(bias, np.float64))
    idx = np.zeros((n, k), np.int64)
    w = np.zeros((n, k))
    GS = E // router.n_group

    def pick(vals, ok):
        best, bi = -np.inf, None
        for i, v in enumerate(vals):
            if ok[i] and v > best:
                best, bi = v, i
        return 0 if bi is None else bi

    for t in range(n):
        allowed = np.ones(E, bool)
        if router.n_group > 1:
            g = np.sort(c[t].reshape(router.n_group, GS), axis=1)[:, ::-1]
            G = g[:, 0] if router.group_top == 1 else g[:, 0] + g[:, 1]
            kept = np.zeros(router.n_group, bool)
            for _ in range(router.topk_group):
                kept[pick(G, ~kept)] = True
            allowed = np.repeat(kept, GS)
        taken = np.zeros(E, bool)
        for j in range(k):
            e = pick(c[t], allowed & ~taken)
            idx[t, j] = e
            taken[e] = True
        w[t] = s[t, idx[t]]
        if router.renormalize:
            W = w[t].sum()
            w[t] = w[t] / W if W > 0 else 0.0
        w[t] *= router.scale
    return idx, w, s


RULES = {
    "deepseek_v3": (RouterSpec("sigmoid", 8, 4, 2, True, 2.5), 64, 8, True),
    "deepseek_v2": (RouterSpec("softmax", 8, 3, 1, False, 16.0), 64, 6, False),
    "qwen_olmoe": (RouterSpec("softmax", renormalize=False), 60, 4, False),
    "llama4": (RouterSpec("sigmoid", renormalize=False), 16, 1, False),
    "sigmoid_groups_e8": (RouterSpec("sigmoid", 4, 2, 2, True, 1.0), 8, 2, True),
}


@pytest.mark.parametrize("name", list(RULES))
def test_torch_statement_equals_float64_on_tie_free_inputs(name):
    router, E, k, with_bias = RULES[name]
    g = np.random.default_rng(sum(map(ord, name)))
    n = 256
    # tie-free: distinct logits per token far apart relative to fp32 error, distinct biases
    logits = np.stack([g.permutation(E) * 0.37 - E * 0.15 + g.random(E) * 0.05 for _ in range(n)]).astype(np.float32)
    bias = (g.permutation(E) * 0.013 - 0.2).astype(np.float32) if with_bias else None
    got = gated_routing_cpu(torch.from_numpy(logits), router, k, None if bias is None else torch.from_numpy(bias))
    idx, w, s = gated_routing_f64(logits, router, k, bias)
    assert np.array_equal(got["topk_idx"].numpy(), idx)
    np.testing.assert_allclose(got["topk_w"].numpy(), w, rtol=2e-6, atol=1e-30)
    np.testing.assert_allclose(got["scores"].numpy(), s, rtol=2e-6, atol=1e-12)


def _route(logits, router, k, bias=None):
    b = None if bias is None else torch.tensor(bias, dtype=torch.float32)
    r = gated_routing_cpu(torch.tensor([logits], dtype=torch.float32), router, k, b)
    idx, w, _ = gated_routing_f64(np.array([logits], np.float32), router, k, None if bias is None else
                                  np.array(bias, np.float32))
    assert r["topk_idx"][0].tolist() == idx[0].tolist()
    return r["topk_idx"][0].tolist(), r["topk_w"][0].tolist(), r["scores"][0]


def test_bias_pulls_a_low_score_expert_in_with_its_unbiased_weight():
    logits = [2.0, 1.0, 0.5, -3.0]
    idx, w, s = _route(logits, RouterSpec("sigmoid", renormalize=False), 2, bias=[0.0, 0.0, 0.0, 1.0])
    assert idx == [3, 0]
    assert w[0] == pytest.approx(float(s[3])) and w[0] < 0.05


def test_group_limit_excludes_the_global_top_k():
    # groups of 2: {0,1} {2,3} {4,5} {6,7}; the two best experts (0 and 6) sit in groups beaten by group sums
    logits = [5.0, -5.0, 3.0, 3.0, 2.9, 2.9, 4.9, -5.0]
    idx, _, _ = _route(logits, RouterSpec("sigmoid", 4, 2, 2, True, 1.0), 2)
    assert sorted(idx) == [2, 3]                       # groups {2,3} and {4,5} win on top-2 sums
    free, _, _ = _route(logits, RouterSpec("sigmoid", renormalize=True), 2)
    assert free == [0, 6]


def test_group_top_1_and_2_choose_different_groups():
    logits = [4.0, -4.0, 3.0, 3.0]                     # group 0 has the best max, group 1 the best top-2 sum
    one, _, _ = _route(logits, RouterSpec("sigmoid", 2, 1, 1, True, 1.0), 1)
    two, _, _ = _route(logits, RouterSpec("sigmoid", 2, 1, 2, True, 1.0), 1)
    assert one == [0] and two == [2]


def test_ties_go_to_the_lower_index():
    idx, _, _ = _route([1.0, 2.0, 2.0, 2.0, 0.0, 0.0], RouterSpec("softmax"), 3)
    assert idx == [1, 2, 3]
    # equal group scores: the lower group wins
    idx, _, _ = _route([1.0, 0.0, 0.0, 1.0], RouterSpec("sigmoid", 2, 1, 1, True, 1.0), 1)
    assert idx == [0]
    # NaN never compares greater; nothing left above -inf takes index 0
    idx, w, _ = _route([math.nan, math.nan, math.nan, math.nan], RouterSpec("softmax"), 2)
    assert idx == [0, 0] and w == [0.0, 0.0]


def test_renormalisation_and_scale():
    logits = [0.5, 1.5, -1.0, 0.0]
    idx, w, s = _route(logits, RouterSpec("sigmoid", scale=2.5), 2)
    s1, s0 = np.float32(s[1]), np.float32(s[0])
    W = np.float32(np.float32(0) + s1) + s0
    assert idx == [1, 0]
    assert w == [float(np.float32(s1 / W) * np.float32(2.5)), float(np.float32(s0 / W) * np.float32(2.5))]
    assert sum(w) == pytest.approx(2.5, rel=1e-6)


def test_llama4_style_k1_sigmoid():
    idx, w, s = _route([0.2, 1.7, -0.3, 1.2], RouterSpec("sigmoid", renormalize=False), 1)
    assert idx == [1] and w == [float(s[1])] and w[0] == pytest.approx(1 / (1 + math.exp(-1.7)), rel=1e-6)


def test_softmax_without_renormalisation():
    logits = [0.1, 2.0, 1.0, -1.0]
    idx, w, s = _route(logits, RouterSpec("softmax", renormalize=False), 2)
    p = np.exp(np.array(logits) - 2.0)
    p /= p.sum()
    assert idx == [1, 2]
    assert w == pytest.approx([p[1], p[2]], rel=1e-6) and sum(w) < 1
