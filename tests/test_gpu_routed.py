"""Forwards on the caller's routing (MoEContext.forward_routed -> fm_moe_forward_routed) on one H100: the router's own
routing replayed (bit-identical bookkeeping and rows), every stage exact on inputs whose sums are exact in fp32
(tests/exact.py), random inputs at config B against tests/torch_routed.py, invalid indices, CUDA graphs with a
device-side count, rejected contexts, argument checks and the nn.Module wrapper."""
import numpy as np
import pytest
import torch

from flashmoe_b200 import _lib
from flashmoe_b200.config import BASELINE_CONFIGS, MoEConfig
from tests import exact as ex
from tests.torch_routed import moe_forward_routed_cpu
from tests.util import check_output, make_inputs

pytestmark = pytest.mark.gpu

SMALL = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512)
CONFIG_B = BASELINE_CONFIGS["B"]


def _ctx(cfg, **kw):
    from flashmoe_b200.runtime import MoEContext

    return MoEContext(cfg, timeout_ms=5000, **kw)


def _packets(ctx, name):
    """recv_x / hidden rows of every packet up to its row count (padding rows excluded)."""
    a, cnt = ctx.read(name), ctx.read("recv_cnt")
    return [a[e, :c].copy() for e, c in enumerate(cnt)]


def _torch_router(x, wg, k):
    """What a model's own router might do on the device: x @ Wg, softmax, top-k, renormalise."""
    p = torch.softmax(x.float() @ wg.float(), dim=-1)
    w, i = torch.topk(p, k, dim=-1)
    return i.to(torch.int32), (w / w.sum(-1, keepdim=True)).float()


@pytest.mark.parametrize("cfg,fused", [(SMALL, 1), (SMALL, 0), (SMALL.replace(num_experts=32), 1),
                                       (CONFIG_B, 1), (CONFIG_B, 0)],
                         ids=["small_fused", "small_gather", "small_E32", "configB_fused", "configB_gather"])
def test_router_routing_replayed(monkeypatch, cfg, fused):
    """forward_tokens, then forward_routed on its topk_idx with arbitrary weights: slot, counts, recv_cnt, recv_x and
    hidden are bit-identical to the router launch."""
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    x, wg, we, _, _ = make_inputs(cfg, seed=11)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd, wgd, wed = x.reshape(cfg.S, cfg.H).to(dev), wg.to(dev), we.to(dev)
    for n in (cfg.S, 301):
        ctx.forward_tokens(xd[:n], wgd, wed)
        ctx.synchronize()
        want = {k: ctx.read(k)[:n].copy() for k in ("topk_idx", "slot")}
        want.update(counts=ctx.read("counts").copy(), recv_cnt=ctx.read("recv_cnt").copy())
        rx, hid = _packets(ctx, "recv_x"), _packets(ctx, "hidden")
        idx = torch.from_numpy(want["topk_idx"]).to(dev)
        w = torch.rand(n, cfg.k, generator=torch.Generator().manual_seed(n)).to(dev)
        ctx.forward_routed(xd[:n], idx, w, wed)
        ctx.synchronize()
        assert ctx.last_tokens == n
        for k in ("topk_idx", "slot"):
            assert np.array_equal(ctx.read(k)[:n], want[k]), f"n={n}: {k}"
        for k in ("counts", "recv_cnt"):
            assert np.array_equal(ctx.read(k), want[k]), f"n={n}: {k}"
        for name, ref in (("recv_x", rx), ("hidden", hid)):
            got = _packets(ctx, name)
            assert all(np.array_equal(a, b) for a, b in zip(got, ref)), f"n={n}: {name}"
        assert np.array_equal(ctx.read("mcw")[:n], np.ones(n, np.float32))
    ctx.close()


def _exact_case(k, act=0, bias=False):
    cfg = MoEConfig(num_experts=8, expert_top_k=k, sequence_len=256, hidden_size=128, intermediate_size=192,
                    hidden_act=act)
    gen = dict(bias=bias)
    if act:
        gen.update(gelu_friendly=True, x_range=3, up_range=4)
    return cfg, gen


EXACT = {f"k{k}_fused{f}": (*_exact_case(k), {"FM_FUSED_COMBINE": str(f)}) for k in (1, 2) for f in (1, 0)}
EXACT["k3"] = (*_exact_case(3), {})
EXACT["bias_gelu_k2"] = (*_exact_case(2, act=1, bias=True), {})
EXACT["bias_gelu_k1_gather"] = (*_exact_case(1, act=1, bias=True), {"FM_FUSED_COMBINE": "0"})


@pytest.mark.parametrize("name", list(EXACT))
def test_every_stage_exact(monkeypatch, name):
    """Skewed routing that overflows one expert's capacity, -1 and duplicate picks, an expert with nothing; n = 0, 1,
    an odd count and S on one context.  out bit-exact; rows without a kept pick +0."""
    cfg, gen, env = EXACT[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    inp = ex.exact_inputs(cfg, seed=5000 + sum(map(ord, name)), **gen)
    ctx = _ctx(cfg)
    st = ex.Stats()
    for n in (cfg.S, 0, 1, 97):
        topk, w = ex.routing_case(n, cfg.E, cfg.k, seed=n + 17, hot=2, empty=(5,))
        if n > 1:
            topk[1] = -1                                          # a token with no pick at all
        run = ex.Launcher(ctx, "routed", inp, routing=(topk, w))
        out = run.launch(n)
        ctx.synchronize()
        assert out.shape == (n, cfg.H)
        d, _ = run.read(out, n)
        run.check(d, None, n, stats=st)
        if n == cfg.S:
            slot = d.slot
            assert (slot == ex.INT32_MAX).any() and ((slot >= cfg.EC) & (slot < ex.INT32_MAX)).any()
    ctx.close()
    print(f"\n[{name}] {st.line()}")


def test_random_inputs_config_B_with_a_torch_router():
    cfg = CONFIG_B
    x, wg, we, _, _ = make_inputs(cfg, seed=21)
    ctx = _ctx(cfg)
    dev = ctx.device
    xd = x.reshape(cfg.S, cfg.H).to(dev)
    idx, w = _torch_router(xd, wg.to(dev), cfg.k)
    out = ctx.forward_routed(xd, idx, w, we.to(dev))
    ctx.synchronize()
    ref = moe_forward_routed_cpu(x.reshape(cfg.S, cfg.H), idx.cpu(), w.cpu(), we, EC=cfg.EC)
    assert np.array_equal(ctx.read("slot"), ref["slot"].numpy())
    check_output(ex.to_bits(out.cpu()), ex.to_bits(ref["out"]), what="config B routed out")
    ctx.close()


def test_invalid_index_is_reported_once_and_treated_as_minus_one():
    cfg = SMALL
    inp_x, _, we, _, _ = make_inputs(cfg, seed=31)
    ctx = _ctx(cfg)
    dev = ctx.device
    x, wed = inp_x.reshape(cfg.S, cfg.H).to(dev), we.to(dev)
    topk, w = ex.routing_case(cfg.S, cfg.E, cfg.k, seed=3, skip_frac=0.0)
    clean = topk.copy()
    clean[100, 1] = -1
    clean[400, 0] = -1
    bad = topk.copy()
    bad[100, 1] = cfg.E
    bad[400, 0] = -7
    w_d = torch.from_numpy(w).to(dev)
    ref = ctx.forward_routed(x, torch.from_numpy(clean).to(dev), w_d, wed).clone()
    ctx.synchronize()
    out = ctx.forward_routed(x, torch.from_numpy(bad).to(dev), w_d, wed)
    torch.cuda.synchronize(dev)
    with pytest.raises(_lib.FlashMoEError) as ei:
        ctx.check()
    assert ei.value.code == -1
    msg = str(ei.value)
    assert "topk_idx[100, 1] = 8" in msg or "topk_idx[400, 0] = -7" in msg, msg
    ctx.check()                                                  # reported once
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))
    assert np.array_equal(ctx.read("topk_idx"), clean)
    ctx.forward_routed(x, torch.from_numpy(clean).to(dev), w_d, wed)
    ctx.synchronize()                                            # the next launch is clean
    ctx.close()


def test_cuda_graph_torch_router_then_routed_call_with_a_device_count():
    """One capture of (torch router on the device -> forward_routed with a device count), replayed over several n and
    inputs, interleaved with eager router calls on the same context; every replay bit-identical to the eager routed
    call on the same routing."""
    cfg = SMALL
    _, wg, we, _, _ = make_inputs(cfg, seed=41)
    ctx = _ctx(cfg)
    dev = ctx.device
    wgd, wed = wg.to(dev), we.to(dev)
    x_full = torch.zeros(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev)
    out_full = torch.zeros_like(x_full)
    n_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    ctx.forward_tokens(x_full, wgd, wed)                         # warm-up outside the capture
    torch.cuda.synchronize(dev)
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        idx_s, w_s = _torch_router(x_full, wgd, cfg.k)           # (the allocator's warm-up for the capture)
    torch.cuda.current_stream(dev).wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        idx_s, w_s = _torch_router(x_full, wgd, cfg.k)
        ctx.forward_routed(x_full, idx_s, w_s, wed, out=out_full, n_tokens=n_dev)
    g = torch.Generator().manual_seed(43)
    for i, n in enumerate((cfg.S, 1, 0, 333, 128, cfg.S)):
        x_full.copy_(torch.randn(cfg.S, cfg.H, generator=g).bfloat16())
        n_dev.fill_(n)
        graph.replay()
        torch.cuda.synchronize(dev)
        got, idx, w = out_full[:n].clone(), idx_s[:n].clone(), w_s[:n].clone()
        tables = (ctx.read("slot")[:n].copy(), ctx.read("counts").copy())
        assert ctx.launch_record()[1] == n
        ctx.forward_tokens(x_full[: max(n, 1)], wgd, wed)        # an eager router call in between
        want = ctx.forward_routed(x_full[:n], idx, w, wed)
        ctx.synchronize()
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"replay {i}, n={n}"
        assert np.array_equal(ctx.read("slot")[:n], tables[0]) and np.array_equal(ctx.read("counts"), tables[1])
    ctx.close()


@pytest.mark.parametrize("kw", [dict(num_experts=1, expert_top_k=1), dict(is_training=1)], ids=["E1", "training"])
def test_rejected_contexts(kw):
    cfg = SMALL.replace(**kw)
    ctx = _ctx(cfg)
    dev = ctx.device
    x = torch.zeros(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev)
    we = torch.zeros(cfg.E, 2, cfg.P, cfg.H, dtype=torch.bfloat16, device=dev)
    idx = torch.zeros(cfg.S, cfg.k, dtype=torch.int32, device=dev)
    w = torch.ones(cfg.S, cfg.k, dtype=torch.float32, device=dev)
    with pytest.raises(_lib.FlashMoEError) as ei:
        ctx.forward_routed(x, idx, w, we)
    assert ei.value.code == -1 and ("E = 1" in str(ei.value) or "is_training" in str(ei.value))
    ctx.close()


def test_argument_checks():
    cfg = SMALL
    ctx = _ctx(cfg)
    dev = ctx.device
    L, c = ctx._L, ctx._ctx
    x = torch.zeros(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev)
    we = torch.zeros(cfg.E, 2, cfg.P, cfg.H, dtype=torch.bfloat16, device=dev)
    idx = torch.zeros(cfg.S, cfg.k, dtype=torch.int32, device=dev)
    w = torch.ones(cfg.S, cfg.k, dtype=torch.float32, device=dev)
    n_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    args = (idx.data_ptr(), w.data_ptr(), we.data_ptr(), None, None, x.data_ptr(), None)
    assert L.fm_moe_forward_routed(c, x.data_ptr(), cfg.S + 1, None, *args) == -1
    assert b"n_tokens" in L.fm_last_error()
    assert L.fm_moe_forward_routed(c, x.data_ptr(), 5, n_dev.data_ptr(), *args) == -1
    assert b"n_tokens_dev" in L.fm_last_error()
    assert L.fm_moe_forward_routed(c, x.data_ptr(), 5, None, None, w.data_ptr(), we.data_ptr(), None, None,
                                   x.data_ptr(), None) == -1
    with pytest.raises(RuntimeError, match="int32"):
        ctx.forward_routed(x, idx.long(), w, we)
    with pytest.raises(RuntimeError, match="float32"):
        ctx.forward_routed(x, idx, w.bfloat16(), we)
    with pytest.raises(RuntimeError, match=r"\[n="):
        ctx.forward_routed(x[:5], idx, w, we)
    ctx.close()


def test_layer_converts_torch_topk_routing():
    from flashmoe_b200.layer import FlashMoELayer

    cfg = SMALL
    layer = FlashMoELayer(cfg, bias=True)
    dev = layer.ctx.device
    x = torch.randn(1, cfg.S, cfg.H, generator=torch.Generator().manual_seed(51)).bfloat16().to(dev)
    p = torch.softmax(x.reshape(cfg.S, cfg.H).float() @ layer.gate_weight.float(), dim=-1)
    w, i = torch.topk(p, cfg.k, dim=-1)                          # int64 indices
    w = w.bfloat16()
    res = layer(x, return_routing=True, topk_idx=i, topk_weight=w)
    want = layer.ctx.forward_routed(x, i.to(torch.int32), w.float(), layer.expert_weight, bias_up=layer.bias_up,
                                    bias_down=layer.bias_down)
    layer.ctx.synchronize()
    assert torch.equal(res.out.view(torch.int16), want.view(torch.int16))
    assert torch.equal(res.topk_idx, i.cpu().to(torch.int32))
    assert torch.equal(res.topk_weight.view(torch.int16), w.cpu().view(torch.int16))
    layer.ctx.close()
