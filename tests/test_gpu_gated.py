"""Gated forwards (MoEContext.forward_gated -> fm_moe_forward_gated) on one H100: a gated launch replayed through
forward_routed on its own routing (bit-identical), softmax scoring against the router, exact inputs against interval
references, DeepSeek-V3 parameters against tests/torch_gated.py, CUDA graphs with a device count and an in-place bias
update, NaN tokens, rejected contexts and arguments, and the nn.Module wrapper."""
import ctypes
import math

import numpy as np
import pytest
import torch

from flashmoe_b200 import _lib
from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests.test_gated_api import gated_routing_f64
from tests.torch_gated import moe_forward_gated_cpu
from tests.torch_routed import moe_forward_routed_cpu
from tests.util import check_output, make_inputs

pytestmark = pytest.mark.gpu


def _ctx(cfg, **kw):
    from flashmoe_b200.runtime import MoEContext

    return MoEContext(cfg, timeout_ms=5000, **kw)


def _cfg(E, k, S=512, H=256, P=512, **kw):
    return MoEConfig(num_experts=E, expert_top_k=k, sequence_len=S, hidden_size=H, intermediate_size=P, **kw)


def _bias(E, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(E, generator=g) * 0.05).float()


def _w_float(ctx, n):
    """The device's topk_w (bf16) as fp32: rne_bf16 of it is the same bits."""
    return torch.from_numpy(ctx.read("topk_w")[:n].astype(np.uint32) << 16).view(torch.float32)


V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
REPLAY = {
    # name: (cfg, fused, router, bias)
    "E8_k2_softmax_fused": (_cfg(8, 2), 1, RouterSpec("softmax", renormalize=False, scale=1.5), False),
    "E8_k2_sigmoid_groups_bias_gather": (_cfg(8, 2), 0, RouterSpec("sigmoid", 4, 2, 2, True, 2.0), True),
    "E8_k1_sigmoid_gather": (_cfg(8, 1), 0, RouterSpec("sigmoid", renormalize=False), False),
    "E64_k8_sigmoid_groups_bias_fused": (_cfg(64, 8), 1, RouterSpec("sigmoid", 8, 4, 2, True, 2.5), True),
    "E64_k2_softmax_groups_gather": (_cfg(64, 2), 0, RouterSpec("softmax", 8, 3, 1, False, 16.0), False),
    "E256_k8_deepseek_v3_fused": (_cfg(256, 8, H=128, P=128), 1, V3, True),
    "E384_k1_llama4_fused": (_cfg(384, 1, H=128, P=128), 1, RouterSpec("sigmoid", renormalize=False), False),
    "E384_k8_groups_bias_gather": (_cfg(384, 8, H=128, P=128), 0, RouterSpec("softmax", 32, 4, 2, True, 1.0), True),
}


@pytest.mark.parametrize("name", list(REPLAY))
def test_gated_launch_replayed_through_forward_routed(monkeypatch, name):
    """forward_gated, then forward_routed on its topk_idx and float(topk_w): out, slot, counts and recv_cnt are
    bit-identical; mcw = 1; n = S, 0, 1 and an odd count."""
    cfg, fused, router, with_bias = REPLAY[name]
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    x, wg, we, _, _ = make_inputs(cfg, seed=7)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd, wgd, wed = x.reshape(cfg.S, cfg.H).to(dev), wg.to(dev), we.to(dev)
    sb = _bias(cfg.E, 3).to(dev) if with_bias else None
    for n in (cfg.S, 0, 1, 301):
        out = ctx.forward_gated(xd[:n], wgd, wed, router, score_bias=sb).clone()
        ctx.synchronize()
        assert ctx.last_tokens == n
        idx = ctx.read("topk_idx")[:n].copy()
        want = {k: ctx.read(k)[:n].copy() for k in ("slot",)}
        want.update(counts=ctx.read("counts").copy(), recv_cnt=ctx.read("recv_cnt").copy())
        assert np.array_equal(ctx.read("mcw")[:n], np.ones(n, np.float32))
        assert ((idx >= 0) & (idx < cfg.E)).all()
        if router.n_group > 1 and n:
            gs = cfg.E // router.n_group
            assert (np.array([len(set(r)) for r in (idx // gs)]) <= router.topk_group).all()
        w = _w_float(ctx, n).to(dev)
        got = ctx.forward_routed(xd[:n], torch.from_numpy(idx).to(dev), w, wed)
        ctx.synchronize()
        assert torch.equal(got.view(torch.int16), out.view(torch.int16)), f"n={n}: out"
        assert np.array_equal(ctx.read("slot")[:n], want["slot"]), f"n={n}: slot"
        for k in ("counts", "recv_cnt"):
            assert np.array_equal(ctx.read(k), want[k]), f"n={n}: {k}"
    ctx.close()


@pytest.mark.parametrize("E,k", [(8, 2), (64, 4), (256, 8)])
def test_softmax_scoring_is_the_routers(E, k):
    """scoring = softmax, no groups, no bias, renormalize, scale 1: topk_idx and gate_out are the router's bits."""
    cfg = _cfg(E, k, H=128, P=128)
    x, wg, we, _, _ = make_inputs(cfg, seed=E)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd, wgd, wed = x.reshape(cfg.S, cfg.H).to(dev), wg.to(dev), we.to(dev)
    ctx.forward_tokens(xd, wgd, wed)
    ctx.synchronize()
    want_idx, want_go = ctx.read("topk_idx").copy(), ctx.read("gate_out").copy()
    ctx.forward_gated(xd, wgd, wed, RouterSpec())
    ctx.synchronize()
    assert np.array_equal(ctx.read("topk_idx"), want_idx)
    assert np.array_equal(ctx.read("gate_out"), want_go)
    ctx.close()


# ----------------------------------------------------------------------------- exact inputs
EXACT = {
    "E8_k2_sigmoid_groups_bias": (8, 2, RouterSpec("sigmoid", 4, 2, 2, True, 2.0), True, {}),
    "E8_k1_llama4_gather": (8, 1, RouterSpec("sigmoid", renormalize=False), False, {"FM_FUSED_COMBINE": "0"}),
    "E64_k3_softmax_groups_bias": (64, 3, RouterSpec("softmax", 8, 3, 1, False, 16.0), True, {}),
    "E64_k2_softmax_renorm": (64, 2, RouterSpec("softmax"), False, {}),
}


@pytest.mark.parametrize("name", list(EXACT))
def test_exact_inputs(monkeypatch, name):
    E, k, router, with_bias, env = EXACT[name]
    for kk, v in env.items():
        monkeypatch.setenv(kk, v)
    cfg = MoEConfig(num_experts=E, expert_top_k=k, sequence_len=256, hidden_size=128, intermediate_size=192)
    inp = ex.exact_inputs(cfg, seed=9000 + sum(map(ord, name)))
    ctx = _ctx(cfg)
    bias = (np.random.default_rng(len(name)).permutation(E) * 2.0 ** -9 - 0.05).astype(np.float32) if with_bias \
        else None
    run = ex.Launcher(ctx, "gated", inp, router=router, score_bias=bias)
    st = ex.Stats()
    amb_total = tok_total = 0
    for n in (cfg.S, 0, 1, 97):
        amb_total += run.run(n, stats=st)[2]
        tok_total += n
    ctx.close()
    print(f"\n[{name}] ambiguous tokens {amb_total} of {tok_total}; {st.line()}")
    assert amb_total <= max(0, tok_total // 1000), f"{amb_total} ambiguous tokens of {tok_total}"


def _hand_built_logits():
    """(router, k, E, bias, logits rows): the CPU tests' cases (tests/test_gated_api.py), on the 2^-6 grid."""
    return [
        (RouterSpec("sigmoid", renormalize=False), 2, 4, [0.0, 0.0, 0.0, 1.0], [[2.0, 1.0, 0.5, -3.0]]),
        (RouterSpec("sigmoid", 4, 2, 2, True, 1.0), 2, 8, None, [[5.0, -5.0, 3.0, 3.0, 2.90625, 2.90625, 4.90625, -5.0]]),
        (RouterSpec("sigmoid", 2, 1, 1, True, 1.0), 1, 4, None, [[4.0, -4.0, 3.0, 3.0]]),
        (RouterSpec("sigmoid", 2, 1, 2, True, 1.0), 1, 4, None, [[4.0, -4.0, 3.0, 3.0]]),
        (RouterSpec("softmax"), 3, 8, None, [[1.0, 2.0, 2.0, 2.0, 0.0, 0.0, -1.0, -1.0]]),
        (RouterSpec("sigmoid", 2, 1, 1, True, 1.0), 1, 4, None, [[1.0, 0.0, 0.0, 1.0]]),
        (RouterSpec("sigmoid", scale=2.5), 2, 4, None, [[0.5, 1.5, -1.0, 0.0]]),
        (RouterSpec("sigmoid", renormalize=False), 1, 4, None, [[0.1875, 1.6875, -0.3125, 1.1875]]),
        (RouterSpec("softmax", renormalize=False), 2, 4, None, [[0.125, 2.0, 1.0, -1.0]]),
    ]


@pytest.mark.parametrize("case", range(len(_hand_built_logits())))
def test_hand_built_cases_on_the_device(case):
    """Token t has x = e_t and Wg_eff[:, t] = its logits, so the device's logits are exactly the planned ones."""
    router, k, E, bias, rows = _hand_built_logits()[case]
    cfg = MoEConfig(num_experts=E, expert_top_k=k, sequence_len=128, hidden_size=128, intermediate_size=128)
    n = len(rows)
    x = torch.zeros(cfg.S, cfg.H)
    wg_eff = torch.zeros(E, cfg.H)
    for t, row in enumerate(rows):
        x[t, t] = 1.0
        wg_eff[:, t] = torch.tensor(row)
    ctx = _ctx(cfg)
    dev = ctx.device
    wg = wg_eff.reshape(-1).reshape(cfg.H, E).bfloat16().to(dev)
    assert torch.equal(wg.cpu().reshape(-1).reshape(E, cfg.H).float(), wg_eff)
    we = torch.zeros(E, 2, cfg.P, cfg.H, dtype=torch.bfloat16, device=dev)
    sb = torch.tensor(bias, dtype=torch.float32, device=dev) if bias is not None else None
    ctx.forward_gated(x[:n].bfloat16().to(dev), wg, we, router, score_bias=sb)
    ctx.synchronize()
    logits = np.array(rows, np.float32)
    idx, w, _ = gated_routing_f64(logits, router, k, None if bias is None else np.array(bias, np.float32))
    assert ctx.read("topk_idx")[:n].tolist() == idx.tolist()
    got_w = (ctx.read("topk_w")[:n].astype(np.uint32) << 16).view(np.float32)
    np.testing.assert_allclose(got_w, w, rtol=2 ** -7)
    ctx.close()


def test_deepseek_v3_parameters_against_the_torch_statement():
    cfg = _cfg(256, 8, S=1024, H=256, P=256)
    x, wg, we, _, _ = make_inputs(cfg, seed=77)
    bias = _bias(cfg.E, 5)
    ctx = _ctx(cfg)
    dev = ctx.device
    xs = x.reshape(cfg.S, cfg.H)
    out = ctx.forward_gated(xs.to(dev), wg.to(dev), we.to(dev), V3, score_bias=bias.to(dev))
    ctx.synchronize()
    ref = moe_forward_gated_cpu(xs, wg, we, V3, cfg.k, EC=cfg.EC, score_bias=bias)
    idx = ctx.read("topk_idx")
    same = (idx == ref["topk_idx"].numpy()).all(axis=1)
    assert same.mean() >= 0.99, f"picks differ on {int((~same).sum())} of {cfg.S} tokens"
    go = ex.bits_to_f64(ctx.read("gate_out"))
    np.testing.assert_allclose(go, ref["gate_out"].double().numpy(), rtol=2 ** -7, atol=1e-6)
    w = ex.bits_to_f64(ctx.read("topk_w"))
    np.testing.assert_allclose(w[same], ex.bits_to_f64(ex.f32_to_bf16(ref["w"].numpy()))[same], rtol=2 ** -6)
    # out against the torch forward on the device's own routing (near-tied picks may differ from the statement's)
    own = moe_forward_routed_cpu(xs, torch.from_numpy(idx), _w_float(ctx, cfg.S), we, EC=cfg.EC)
    check_output(ex.to_bits(out.cpu()), ex.to_bits(own["out"]), what="DeepSeek-V3 gated out")
    check_output(ex.to_bits(out.cpu()), ex.to_bits(ref["out"]), rows_ok=same, what="DeepSeek-V3 out vs torch_gated")
    ctx.close()


def test_cuda_graph_with_a_device_count_follows_bias_updates():
    cfg = _cfg(64, 4, S=512, H=128, P=128)
    router = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
    _, wg, we, _, _ = make_inputs(cfg, seed=41)
    ctx = _ctx(cfg)
    dev = ctx.device
    wgd, wed = wg.to(dev), we.to(dev)
    x_full = torch.zeros(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev)
    out_full = torch.zeros_like(x_full)
    n_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    sb = torch.zeros(cfg.E, dtype=torch.float32, device=dev)
    ctx.forward_gated(x_full, wgd, wed, router, score_bias=sb)   # warm-up outside the capture
    torch.cuda.synchronize(dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ctx.forward_gated(x_full, wgd, wed, router, score_bias=sb, out=out_full, n_tokens=n_dev)
    g = torch.Generator().manual_seed(43)
    for i, n in enumerate((cfg.S, 1, 0, 333, 128, cfg.S)):
        x_full.copy_(torch.randn(cfg.S, cfg.H, generator=g).bfloat16())
        sb.zero_()
        if i > 0:
            sb[i] = 10.0   # (in place, after the capture: every token's first pick must follow it)
        n_dev.fill_(n)
        graph.replay()
        torch.cuda.synchronize(dev)
        assert ctx.launch_record()[1] == n
        got = out_full[:n].clone()
        idx = ctx.read("topk_idx")[:n].copy()
        want = ctx.forward_gated(x_full[:n], wgd, wed, router, score_bias=sb)
        ctx.synchronize()
        assert np.array_equal(ctx.read("topk_idx")[:n], idx), f"replay {i}: routing"
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"replay {i}, n={n}"
        if i > 0:
            assert (idx[:, 0] == i).all(), f"replay {i}: the bias update was not followed"
    ctx.close()


def test_nan_token_stays_in_range_and_alone():
    cfg = _cfg(64, 4, S=256, H=128, P=128)
    x, wg, we, _, _ = make_inputs(cfg, seed=61)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd, wgd, wed = x.reshape(cfg.S, cfg.H).to(dev), wg.to(dev), we.to(dev)
    for router in (RouterSpec("softmax"), RouterSpec("sigmoid", 8, 2, 2, True, 1.0)):
        ref = ctx.forward_gated(xd, wgd, wed, router).clone()
        ctx.synchronize()
        ref_idx = ctx.read("topk_idx").copy()
        bad = xd.clone()
        bad[5] = float("nan")
        got = ctx.forward_gated(bad, wgd, wed, router)
        ctx.synchronize()
        idx = ctx.read("topk_idx")
        assert ((idx >= 0) & (idx < cfg.E)).all()
        others = np.arange(cfg.S) != 5
        assert np.array_equal(idx[others], ref_idx[others])
        # rows of other tokens keep their bits unless they shared a capacity-limited expert with token 5
        same = (got.view(torch.int16) == ref.view(torch.int16)).all(dim=1).cpu().numpy()
        assert same[others].mean() > 0.9
    ctx.close()


@pytest.mark.parametrize("kw", [dict(num_experts=1, expert_top_k=1), dict(is_training=1)], ids=["E1", "training"])
def test_rejected_contexts(kw):
    cfg = _cfg(8, 2, S=128, H=128, P=128).replace(**kw)
    ctx = _ctx(cfg)
    dev = ctx.device
    x = torch.zeros(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev)
    wg = torch.zeros(cfg.H, cfg.E, dtype=torch.bfloat16, device=dev)
    we = torch.zeros(cfg.E, 2, cfg.P, cfg.H, dtype=torch.bfloat16, device=dev)
    with pytest.raises(_lib.FlashMoEError) as ei:
        ctx.forward_gated(x, wg, we, RouterSpec())
    assert ei.value.code == -1 and ("E = 1" in str(ei.value) or "is_training" in str(ei.value))
    ctx.close()


def test_bad_struct_fields_and_misaligned_bias_are_rejected():
    cfg = _cfg(8, 2, S=128, H=128, P=128)
    ctx = _ctx(cfg)
    dev = ctx.device
    L, c = ctx._L, ctx._ctx
    x = torch.zeros(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev)
    wg = torch.zeros(cfg.H, cfg.E, dtype=torch.bfloat16, device=dev)
    we = torch.zeros(cfg.E, 2, cfg.P, cfg.H, dtype=torch.bfloat16, device=dev)
    o = torch.zeros_like(x)
    sb = torch.zeros(cfg.E + 4, dtype=torch.float32, device=dev)

    def call(r, bias=None):
        return L.fm_moe_forward_gated(c, x.data_ptr(), cfg.S, None, wg.data_ptr(),
                                      None if r is None else ctypes.byref(r), bias, we.data_ptr(), None, None,
                                      o.data_ptr(), None)

    good = dict(scoring=1, n_group=4, topk_group=2, group_top=2, renormalize=1, scale=2.5)
    assert call(_lib.FmRouter(**good)) == 0
    ctx.synchronize()
    bad = [dict(scoring=2), dict(n_group=0), dict(n_group=33), dict(n_group=3), dict(topk_group=0),
           dict(topk_group=5), dict(group_top=0), dict(group_top=3), dict(n_group=8, topk_group=1, group_top=2),
           dict(n_group=8, topk_group=1, group_top=1), dict(renormalize=2), dict(scale=0.0), dict(scale=-1.0),
           dict(scale=math.inf), dict(scale=math.nan)]
    for b in bad:
        assert call(_lib.FmRouter(**{**good, **b})) == -1, b
        assert b"router" in L.fm_last_error() or b"k = " in L.fm_last_error(), b
    assert call(None) == -1 and b"router" in L.fm_last_error()
    assert call(_lib.FmRouter(**good), sb.data_ptr() + 4) == -1 and b"score_bias" in L.fm_last_error()
    assert call(_lib.FmRouter(**good), sb.data_ptr() + 16) == 0
    ctx.synchronize()
    with pytest.raises(RuntimeError, match="float32"):
        ctx.forward_gated(x, wg, we, RouterSpec(), score_bias=sb[: cfg.E].double())
    with pytest.raises(RuntimeError, match="16-byte"):
        ctx.forward_gated(x, wg, we, RouterSpec(), score_bias=sb[1: cfg.E + 1])
    with pytest.raises(ValueError, match="k=2"):
        ctx.forward_gated(x, wg, we, RouterSpec(n_group=8, topk_group=1))   # one kept group of one expert
    ctx.close()


def test_layer_with_a_router_rule_and_return_routing():
    from flashmoe_b200.layer import FlashMoELayer

    cfg = _cfg(64, 4, S=256, H=128, P=128)
    router = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
    layer = FlashMoELayer(cfg, bias=True, router=router, score_bias=True)
    dev = layer.ctx.device
    assert layer.score_bias.dtype == torch.float32 and tuple(layer.score_bias.shape) == (cfg.E,)
    layer.score_bias.copy_(torch.linspace(-0.1, 0.1, cfg.E))
    x = torch.randn(1, cfg.S, cfg.H, generator=torch.Generator().manual_seed(51)).bfloat16().to(dev)
    res = layer(x, return_routing=True)
    want = layer.ctx.forward_gated(x, layer.gate_weight, layer.expert_weight, router, score_bias=layer.score_bias,
                                   bias_up=layer.bias_up, bias_down=layer.bias_down)
    layer.ctx.synchronize()
    assert torch.equal(res.out.view(torch.int16), want.view(torch.int16))
    assert torch.equal(res.topk_idx, torch.from_numpy(layer.ctx.read("topk_idx")))
    assert torch.equal(res.topk_weight.view(torch.int16),
                       torch.from_numpy(layer.ctx.read("topk_w").view(np.int16)))
    assert res.topk_weight.float().sum(dim=1).sub(2.5).abs().max() < 0.05
    with pytest.raises(ValueError):
        FlashMoELayer(cfg, score_bias=True)
    layer.ctx.close()
