"""SwiGLU experts (hidden_act = 2) end to end: the routing tables equal a ReLU context's bit for bit on the same x and
gate; a forward captured once in a CUDA graph with a device-side count and replayed at n = S, 301, 1, 0 (rows past n
NaN) equals eager calls bit for bit; and FlashMoELayer with a shared expert and a router rule matches a Hugging
Face-style torch SwiGLU at Mixtral-8x7B and DeepSeek-V3 layer shapes within tests/util.py's parity rule (h, and out
from the device's h).  Needs an H100."""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests import exact_swiglu as sw
from tests import util

pytestmark = pytest.mark.gpu

V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)


def _cfg(act, E=16, k=2, S=512, H=320, P=320, **kw):
    return MoEConfig(num_experts=E, expert_top_k=k, sequence_len=S, hidden_size=H, intermediate_size=P, hidden_act=act,
                     **kw)


@pytest.mark.parametrize("route,k,training", [("router", 2, 0), ("router", 1, 1), ("gated", 4, 0)])
def test_routing_tables_equal_relu_context(route, k, training):
    from flashmoe_b200.runtime import MoEContext

    router_kw = dict(zero_tokens=2, wg_range=1 if route == "gated" else 4)
    inp = sw.swiglu_inputs(_cfg(2, k=k, is_training=training), 31 + k, bias=True, **router_kw)
    # the ReLU weights exact_inputs draws for the same x and gate weights
    relu_we = ex.exact_inputs(_cfg(0, k=k, is_training=training), 31 + k, x_range=1, **router_kw).experts.w.cuda()
    res = {}
    for act in (0, 2):
        cfg = _cfg(act, k=k, is_training=training)
        ctx = MoEContext(cfg, timeout_ms=10000)
        try:
            x, wg, we, bu, bd = inp.device(ctx.device)
            if act == 0:
                we, bu, bd = relu_we, None, None
            x = x.reshape(cfg.S, cfg.H)
            got = {}
            for n in (cfg.S, 301):
                if route == "gated":
                    ctx.forward_gated(x[:n], wg, we, V3, bias_up=bu, bias_down=bd)
                else:
                    ctx.forward_tokens(x[:n], wg, we, bias_up=bu, bias_down=bd)
                ctx.synchronize()
                for name in ("topk_idx", "topk_w", "slot", "mcw") + (("gate_out",) if route == "router" else ()):
                    got[(n, name)] = ctx.read(name)[:n].copy()
                for name in ("counts", "recv_cnt") + (("aux_loss",) if training else ()):
                    got[(n, name)] = ctx.read(name).copy()
            res[act] = got
        finally:
            ctx.close()
    for key, a in res[0].items():
        b = res[2][key]
        if key[1] == "aux_loss":   # summed across CTAs with float atomics: the order, and so the last bits, vary by run
            np.testing.assert_allclose(a, b, rtol=1e-5, atol=0, err_msg=f"{key} differs")
            continue
        assert a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8)), f"{key} differs"


def test_graph_replays_equal_eager():
    from flashmoe_b200.runtime import MoEContext

    cfg = _cfg(2, k=2, P=192)
    inp = sw.swiglu_inputs(cfg, 77, bias=True)
    sh = sw.shared_swiglu(cfg.H, 192, 78, bias=True)
    ctx = MoEContext(cfg, timeout_ms=10000, shared_inter=192)
    try:
        dev = ctx.device
        x, wg, we, bu, bd = inp.device(dev)
        x = x.reshape(cfg.S, cfg.H)
        se = ex.shared_expert(sh, dev)
        S, H = cfg.S, cfg.H
        eager = {}
        for n in (S, 301, 1, 0):
            out = ctx.forward_tokens(x[:n], wg, we, bias_up=bu, bias_down=bd, shared_expert=se)
            ctx.synchronize()
            eager[n] = (ex.to_bits(out.cpu()).copy(), ctx.read("hidden").copy(), ctx.read("topk_idx")[:n].copy())
        x_full = x.clone()
        cnt = torch.tensor([S], dtype=torch.int32, device=dev)
        out = torch.full((S, H), 3.0, dtype=torch.bfloat16, device=dev)
        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            ctx.forward_tokens(x_full, wg, we, bias_up=bu, bias_down=bd, out=out, n_tokens=cnt, shared_expert=se)
        torch.cuda.current_stream(dev).wait_stream(s)
        ctx.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            ctx.forward_tokens(x_full, wg, we, bias_up=bu, bias_down=bd, out=out, n_tokens=cnt, shared_expert=se)
        for n in (S, 301, 1, 0):
            x_full.copy_(x)
            x_full[n:] = float("nan")
            out.fill_(3.0)
            cnt.fill_(n)
            g.replay()
            ctx.synchronize()
            assert ctx.launch_record()[1] == n
            assert (out[n:] == 3.0).all(), f"replay n={n}: rows past n written"
            o, h, idx = eager[n]
            assert np.array_equal(ex.to_bits(out[:n].cpu()), o), f"replay n={n}: out differs from the eager call"
            assert np.array_equal(ctx.read("topk_idx")[:n], idx), f"replay n={n}: topk_idx differs"
            if n == S:
                assert np.array_equal(ctx.read("hidden"), h), "replay: hidden differs from the eager call"
    finally:
        ctx.close()


def test_binding_rejects_the_other_layout():
    """flashmoe._C.moe_forward's shape check on the compiled configuration (ReLU, config B): the SwiGLU layout
    [nLx, 3, P, H] is rejected with the ReLU / GELU message, and so is a wrong P."""
    from flashmoe import _C

    _C.initialize()
    try:
        cc = _C.get_compiled_config()
        S, H, P, E = cc["S"], cc["H"], cc["P"], cc["E"]
        nlx = _C.get_num_local_experts()
        x = torch.zeros(1, S, H, dtype=torch.bfloat16, device="cuda")
        wg = torch.zeros(H, E, dtype=torch.bfloat16, device="cuda")
        with pytest.raises(RuntimeError, match=re.escape("Expert weights must have up and down projections [nLx, 2, P, H]")):
            _C.moe_forward(x, wg, torch.zeros(nlx, 3, P, H, dtype=torch.bfloat16, device="cuda"))
        with pytest.raises(RuntimeError, match=re.escape(f"Expert weights must be [*, 2, P={P}, H={H}]")):
            _C.moe_forward(x, wg, torch.zeros(nlx, 2, P // 2, H, dtype=torch.bfloat16, device="cuda"))
    finally:
        _C.finalize()


def torch_swiglu_moe(x, topk_idx, slot, topk_w, mcw, we, shared_w=None, hidden=None, shared_hidden=None):
    """A Hugging Face-style SwiGLU MoE (gate_proj, up_proj, act_fn(gate) * up, down_proj per expert, routing-weighted
    sum, plus the shared expert) in torch, from the bf16 weights, rounding to bf16 where the kernel does: h once, y,
    y / mcw, each weighted term, and the output after each add in pick order.  we [E, 3, P, H] in the kernel's layout;
    topk_idx -1 = a dropped pick.  `hidden` [E, pEC, P] / `shared_hidden` [n, Ps] (bf16): take h from there (the
    device's, by packet slot) instead of computing it.  Returns (out [n, H], h of every kept pick [picks, P] in
    (expert, token) order, the shared expert's h [n, Ps] or None)."""
    E, _, P, H = we.shape
    n, k = topk_idx.shape
    xf = x.float()

    def gate_up(rows, w3):
        return (F.silu(rows @ w3[0].float().T) * (rows @ w3[1].float().T)).bfloat16()

    def down(h, w3, p):
        return (h.float() @ w3[2].reshape(H, p).float().T).bfloat16().float()

    y = torch.zeros(n, k, H, device=x.device)
    hs = []
    for e in range(E):
        tok, j = (topk_idx == e).nonzero(as_tuple=True)
        if tok.numel():
            h = gate_up(xf[tok], we[e]) if hidden is None else hidden[e, slot[tok, j]]
            hs.append(h)
            y[tok, j] = down(h, we[e], P)
    q = (y / mcw[:, None, None]).bfloat16().float()
    out = torch.zeros(n, H, device=x.device)
    for j in range(k):
        term = (topk_w[:, j, None].float() * q[:, j]).bfloat16().float()
        out = torch.where((topk_idx[:, j] >= 0)[:, None], (out + term).bfloat16().float(), out)
    h_s = None
    if shared_w is not None:
        h_s = gate_up(xf, shared_w) if shared_hidden is None else shared_hidden
        out = (out + down(h_s, shared_w, shared_w.shape[1])).bfloat16().float()
    return out, torch.cat(hs), h_s


@pytest.mark.parametrize("shape", ["mixtral_8x7b", "deepseek_v3"])
def test_layer_matches_torch_swiglu(shape):
    """Mixtral-8x7B (E 8, k 2, H 4096, P 14336) on the built-in router, and DeepSeek-V3's layer (H 7168, P 2048, k 8,
    the V3 rule, a shared expert of Ps 2048) with 128 of its 256 experts, so that the layer's float32 weight
    initialisation fits beside the torch reference on one card.  Two checks, each within the parity rule: h (routed
    and shared) against torch's, and out against torch's combine of the device's h.  (A single end-to-end comparison
    at K = 4096-14336 compounds the last-bit differences of two accumulation orders through two bf16 roundings.)"""
    from flashmoe_b200.layer import FlashMoELayer

    if shape == "mixtral_8x7b":
        cfg = _cfg(2, E=8, k=2, S=512, H=4096, P=14336)
        layer = FlashMoELayer(cfg, device=0)
    else:
        cfg = _cfg(2, E=128, k=8, S=512, H=7168, P=2048)
        layer = FlashMoELayer(cfg, device=0, router=V3, shared_inter=2048)
    assert "act=swiglu" in repr(layer)
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(1, cfg.S, cfg.H, generator=g).bfloat16().cuda()
    res = layer(x, return_routing=True)
    ctx = layer.ctx
    # the kernel's combine weights: topk_w over mcw (router: the picks' probability sum; a rule's launch: 1)
    mcw = torch.from_numpy(ctx.read("mcw")[:cfg.S].copy()).float().cuda()
    kept = res.slot < cfg.EC
    idx = torch.where(kept, res.topk_idx.long(), torch.full((), -1, dtype=torch.long)).cuda()
    slot = res.slot.long().cuda()

    def bf16(a):
        return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).view(torch.bfloat16).cuda()

    hidden = bf16(ctx.read("hidden"))
    h_s = bf16(ctx.read("shared_hidden")[:cfg.S]) if layer.shared_weight is not None else None
    xs = x.view(cfg.S, cfg.H)
    _, h_ref, hs_ref = torch_swiglu_moe(xs, idx, slot, res.topk_weight.cuda(), mcw, layer.expert_weight,
                                        layer.shared_weight)
    ref, h_dev, _ = torch_swiglu_moe(xs, idx, slot, res.topk_weight.cuda(), mcw, layer.expert_weight,
                                     layer.shared_weight, hidden=hidden, shared_hidden=h_s)
    util.check_output(ex.to_bits(h_dev), ex.to_bits(h_ref), what=f"{shape} h")
    if h_s is not None:
        util.check_output(ex.to_bits(h_s), ex.to_bits(hs_ref), what=f"{shape} shared h")
    util.check_output(ex.to_bits(res.out.view(cfg.S, cfg.H)), ex.to_bits(ref.bfloat16()), what=f"{shape} out")
    ctx.close()
