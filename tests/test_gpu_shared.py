"""Shared experts (fm_moe_forward_shared, `shared_expert=` on the forward calls) on one H100: the definition
out[t] = rne_bf16(r[t] + s[t]) bit for bit against the same context's call without one, on every route, k, combine,
activation, bias, Ps and token count; s itself against the dense E = 1 path and the exact-input references; graphs with
a device-side count; the argument checks; and the layer.  Two ranks: tests/test_gpu_multi.py's "shared" scenario."""
import ctypes

import numpy as np
import pytest
import torch

from flashmoe_b200 import _lib
from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests.util import make_inputs

pytestmark = pytest.mark.gpu

# E = 16, P = 256: Ps = 64, 320 (a partial 256-column tile), P and 2P; DeepSeek-V3's rule at 8 groups of 2
BASE = MoEConfig(num_experts=16, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=256)
S, H, P = BASE.S, BASE.H, BASE.P
PS = (64, 320, P, 2 * P)
NS = (S, 0, 1, 301)
V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
TABLES = ("topk_idx", "topk_w", "mcw", "slot", "counts", "recv_cnt", "gate_out")


def _ctx(cfg, shared_inter=2 * P, **kw):
    from flashmoe_b200.runtime import MoEContext

    return MoEContext(cfg, timeout_ms=10000, shared_inter=shared_inter, **kw)


def _bits(t):
    return t.view(torch.int16)


def _shared(ps, seed, bias, dev):
    from flashmoe_b200.runtime import SharedExpert

    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(2, ps, H, generator=g) * H ** -0.5).bfloat16().to(dev)
    bu = (torch.randn(ps, generator=g) * 0.1).bfloat16().to(dev) if bias else None
    bd = (torch.randn(H, generator=g) * 0.1).bfloat16().to(dev) if bias else None
    return SharedExpert(w, bu, bd)


def _rne_add(r, s):
    return (r.float() + s.float()).bfloat16()


class Route:
    """One route's forward on a context, with or without a shared expert."""

    def __init__(self, ctx, name, seed):
        cfg, dev = ctx.cfg, ctx.device
        x, wg, we, bu, bd = make_inputs(cfg, seed=seed, bias=True)
        self.ctx, self.name = ctx, name
        self.x, self.wg, self.we = x.reshape(cfg.S, cfg.H).to(dev), wg.to(dev), we.to(dev)
        self.bu, self.bd = bu.to(dev), bd.to(dev)
        idx, w = ex.routing_case(cfg.S, cfg.E, cfg.k, seed=seed + 1)
        self.idx, self.w = torch.from_numpy(idx).to(dev), torch.from_numpy(w).to(dev)

    def __call__(self, n, shared=None, out=None, n_tokens=None, x=None):
        c = self.ctx
        x = self.x[:n] if x is None else x
        m = x.shape[0]
        kw = dict(bias_up=self.bu, bias_down=self.bd, out=out, n_tokens=n_tokens)
        if shared is not None:
            kw["shared_expert"] = shared
        if self.name == "router":
            return c.forward_tokens(x, self.wg, self.we, **kw)
        if self.name == "routed":
            return c.forward_routed(x, self.idx[:m], self.w[:m], self.we, **kw)
        return c.forward_gated(x, self.wg, self.we, V3, **kw)


def _tables(ctx, n, name):
    names = TABLES + (("aux_loss",) if ctx.cfg.is_training else ())
    return {t: ctx.read(t)[:n].copy() if t not in ("counts", "recv_cnt", "aux_loss") else ctx.read(t).copy()
            for t in names if not (t == "gate_out" and name == "routed")}


def _check_definition(route, n, shared, what):
    ctx = route.ctx
    plain = route(n).clone()
    ctx.synchronize()
    want_tables = _tables(ctx, n, route.name)
    sentinel = torch.full((S, H), 7.0, dtype=torch.bfloat16, device=ctx.device)
    out = sentinel[:n]
    route(n, shared=shared, out=out if n else None)
    ctx.synchronize()
    sy = torch.from_numpy(ctx.read("shared_y")[:n].copy()).view(torch.bfloat16).to(ctx.device)
    assert torch.equal(_bits(out), _bits(_rne_add(plain, sy))), f"{what}: out != rne(out_plain + shared_y)"
    for t, got in _tables(ctx, n, route.name).items():
        want = want_tables[t]
        if t == "aux_loss":
            # gML is an fp32 atomicAdd of every CTA's column sums in arrival order (as in the reference), so two launches
            # agree only up to that order, with or without a shared expert; gMeC is exact
            E = ctx.cfg.E
            assert np.array_equal(got[E:2 * E], want[E:2 * E]), f"{what}: gMeC differs"
            assert np.allclose(got, want, rtol=1e-5, atol=0), f"{what}: aux_loss differs beyond fp32 summation order"
        else:
            assert np.array_equal(got, want), f"{what}: {t} differs from the call without a shared expert"


@pytest.mark.parametrize("k,fused,act", [(1, 1, 0), (1, 0, 1), (2, 1, 1), (2, 0, 0), (4, 0, 0), (4, 0, 1), (1, 1, 1),
                                         (2, 1, 0), (2, 0, 1), (1, 0, 0)])
def test_definition_bit_for_bit(monkeypatch, k, fused, act):
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    ctx = _ctx(BASE.replace(expert_top_k=k, hidden_act=act))
    try:
        for ri, name in enumerate(("router", "routed", "gated")):
            route = Route(ctx, name, seed=100 * k + 10 * act + ri)
            for bias in (False, True):
                for ps in PS:
                    shared = _shared(ps, seed=ps + bias, bias=bias, dev=ctx.device)
                    for n in NS:
                        _check_definition(route, n, shared, f"{name} k={k} fused={fused} act={act} bias={bias} "
                                                            f"Ps={ps} n={n}")
    finally:
        ctx.close()


def test_training_context_router_route():
    ctx = _ctx(BASE.replace(is_training=1))
    try:
        route = Route(ctx, "router", seed=5)
        for n in NS:
            _check_definition(route, n, _shared(P, 6, True, ctx.device), f"training n={n}")
    finally:
        ctx.close()


@pytest.mark.parametrize("act", [0, 1])
def test_shared_y_is_the_dense_path(act):
    """s = the output of an E = 1, k = 1 context with P = Ps on x: the same tiles and roundings."""
    ctx = _ctx(BASE.replace(hidden_act=act))
    try:
        route = Route(ctx, "router", seed=7)
        for ps in (64, 320, 2 * P):
            dense = _ctx(BASE.replace(num_experts=1, expert_top_k=1, intermediate_size=ps, hidden_act=act),
                         shared_inter=None)
            wg1 = torch.ones(H, 1, dtype=torch.bfloat16, device=ctx.device)
            for bias in (False, True):
                se = _shared(ps, seed=ps + 11 * bias, bias=bias, dev=ctx.device)
                for n in (S, 301, 1):
                    route(n, shared=se)
                    ctx.synchronize()
                    got = ctx.read("shared_y")[:n]
                    want = dense.forward_tokens(route.x[:n], wg1, se.w[None].contiguous(),
                                                bias_up=None if se.bias_up is None else se.bias_up[None].contiguous(),
                                                bias_down=None if se.bias_down is None else se.bias_down[None].contiguous())
                    dense.synchronize()
                    assert np.array_equal(got, _bits(want).cpu().numpy().view(np.uint16)), \
                        f"act={act} Ps={ps} bias={bias} n={n}: shared_y differs from the dense path"
            dense.close()
    finally:
        ctx.close()


def test_shared_y_exact_reference_relu():
    """On exact inputs (every fp32 partial sum exact) s equals the float64 reference bit for bit."""
    ps = 320
    inp = ex.exact_inputs(BASE.replace(num_experts=1, expert_top_k=1, intermediate_size=ps), seed=21, bias=True)
    ctx = _ctx(BASE)
    try:
        dev = ctx.device
        route = Route(ctx, "router", seed=22)
        xp = inp.experts
        se = ex.shared_expert(xp, dev)
        x = inp.x.reshape(S, H).to(dev)
        route(S, shared=se, x=x)
        ctx.synchronize()
        y = xp.y(0, xp.h(0, inp.x64, "shared h").lo, "shared y")
        ex.check_equal(ctx.read("shared_y"), y.lo, "shared_y", ("token", "column"))
    finally:
        ctx.close()


def test_graph_device_count_and_weight_updates():
    ctx = _ctx(BASE)
    try:
        dev = ctx.device
        route = Route(ctx, "router", seed=31)
        se = _shared(320, 32, True, dev)
        x_full = route.x.clone()
        cnt = torch.tensor([S], dtype=torch.int32, device=dev)
        out = torch.full((S, H), 3.0, dtype=torch.bfloat16, device=dev)
        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            route(S, shared=se, out=out, n_tokens=cnt, x=x_full)   # warm-up
        torch.cuda.current_stream(dev).wait_stream(s)
        ctx.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            route(S, shared=se, out=out, n_tokens=cnt, x=x_full)
        w2 = _shared(320, 33, True, dev)
        for step, n in enumerate((S, 1, 0, 301, 301)):
            if step == 4:   # in-place update of the shared weights' contents
                se.w.copy_(w2.w)
                se.bias_up.copy_(w2.bias_up)
                se.bias_down.copy_(w2.bias_down)
            x_full.copy_(route.x)
            x_full[n:] = float("nan")
            out.fill_(3.0)
            cnt.fill_(n)
            g.replay()
            ctx.synchronize()
            got = out.clone()
            want = route(n, shared=se)
            ctx.synchronize()
            assert torch.equal(_bits(got[:n]), _bits(want)), f"replay n={n} step {step}"
            assert (got[n:] == 3.0).all(), f"replay n={n}: rows past n written"
    finally:
        ctx.close()


def test_layer_on_every_route():
    from flashmoe_b200.layer import FlashMoELayer
    from flashmoe_b200.runtime import SharedExpert

    for router in (None, V3):
        layer = FlashMoELayer(BASE, bias=True, router=router, shared_inter=320)
        layer.shared_bias_up.normal_(0, 0.1)
        layer.shared_bias_down.normal_(0, 0.1)
        assert "shared_inter=320" in layer.extra_repr()
        dev = layer.ctx.device
        x = torch.randn(1, 301, H, device=dev).bfloat16()
        se = SharedExpert(layer.shared_weight, layer.shared_bias_up, layer.shared_bias_down)
        kw = dict(bias_up=layer.bias_up, bias_down=layer.bias_down, shared_expert=se)
        got = layer(x).clone()
        if router is None:
            want = layer.ctx.forward_tokens(x, layer.gate_weight, layer.expert_weight, **kw)
        else:
            want = layer.ctx.forward_gated(x, layer.gate_weight, layer.expert_weight, router, **kw)
        layer.ctx.synchronize()
        assert torch.equal(_bits(got), _bits(want))
        if router is None:   # the caller's routing
            idx = torch.randint(0, BASE.E, (301, BASE.k), device=dev)
            w = torch.rand(301, BASE.k, device=dev)
            got = layer(x, topk_idx=idx, topk_weight=w).clone()
            want = layer.ctx.forward_routed(x, idx.int(), w, layer.expert_weight, **kw)
            layer.ctx.synchronize()
            assert torch.equal(_bits(got), _bits(want))
        layer.ctx.close()


# ------------------------------------------------------------------ rejections (C-ABI)
class Call:
    def __init__(self, ctx, seed):
        dev = ctx.device
        self.ctx = ctx
        self.route = Route(ctx, "router", seed)
        self.se = _shared(320, seed + 1, True, dev)
        self.out = torch.empty(S, H, dtype=torch.bfloat16, device=dev)
        self.router = V3.to_c()

    def args(self):
        r, se = self.route, self.se
        return dict(x=r.x.data_ptr(), n=S, n_dev=None, gw=r.wg.data_ptr(), router=None, sb=None, idx=None, w=None,
                    we=r.we.data_ptr(), bu=r.bu.data_ptr(), bd=r.bd.data_ptr(), out=self.out.data_ptr(),
                    sw=se.w.data_ptr(), sbu=se.bias_up.data_ptr(), sbd=se.bias_down.data_ptr(), inter=320,
                    null_shared=False)

    def call(self, a):
        st = _lib.FmSharedExpert(a["sw"], a["sbu"], a["sbd"], a["inter"])
        return self.ctx._L.fm_moe_forward_shared(
            self.ctx._ctx, a["x"], a["n"], a["n_dev"], a["gw"], a["router"], a["sb"], a["idx"], a["w"], a["we"], a["bu"],
            a["bd"], None if a["null_shared"] else ctypes.byref(st), a["out"],
            torch.cuda.current_stream(self.ctx.device).cuda_stream)

    def good(self):
        assert self.call(self.args()) == 0, self.ctx._L.fm_last_error()
        self.ctx.synchronize()
        return _bits(self.out).clone()


BAD = {
    "null_shared": (dict(null_shared=True), -1, r"^shared must point to an fm_shared_expert_t"),
    "null_w": (dict(sw=None), -1, r"^shared->w must be a non-null device pointer"),
    "inter_zero": (dict(inter=0), -1, r"^shared->inter = 0 must be a positive multiple of 64"),
    "inter_96": (dict(inter=96), -1, r"^shared->inter = 96 must be a positive multiple of 64"),
    "inter_above_reserved": (dict(inter=4 * P), -1, r"^shared->inter = 1024 is above the reserved 512"),
    "misaligned_w": (lambda a: dict(sw=a["sw"] + 2), -1, r"^shared->w must be 16-byte aligned"),
    "misaligned_bias_up": (lambda a: dict(sbu=a["sbu"] + 2), -1, r"^shared->bias_up must be 16-byte aligned"),
    "misaligned_bias_down": (lambda a: dict(sbd=a["sbd"] + 2), -1, r"^shared->bias_down must be 16-byte aligned"),
    "gate_w_with_topk": (lambda a: dict(idx=a["out"]), -1, r"^topk_idx / topk_w are the caller's routing"),
    "router_without_gate_w": (dict(gw=None, router="rule"), -1, r"^router needs gate_w"),
    "score_bias_without_router": (lambda a: dict(sb=a["out"]), -1, r"^score_bias needs gate_w and router"),
}


@pytest.fixture(scope="module")
def call_env():
    ctx = _ctx(BASE)
    c = Call(ctx, seed=41)
    want = c.good()
    yield c, want
    ctx.close()


@pytest.mark.parametrize("case", list(BAD))
def test_rejected(call_env, case):
    import re

    c, want = call_env
    bad, code, pattern = BAD[case]
    a = c.args()
    a.update(bad(a) if callable(bad) else bad)
    if a["router"] == "rule":
        a["router"] = ctypes.byref(c.router)
    launches = c.ctx.launch_count
    assert c.call(a) == code
    msg = c.ctx._L.fm_last_error().decode()
    assert re.search(pattern, msg), msg
    assert c.ctx.launch_count == launches
    assert torch.equal(c.good(), want)


def test_rejected_contexts_and_reservations():
    ctx = _ctx(BASE, shared_inter=None)   # no reservation
    c = Call(ctx, seed=42)
    launches = ctx.launch_count
    assert c.call(c.args()) == -3 and b"fm_shared_reserve" in ctx._L.fm_last_error()
    assert ctx.launch_count == launches
    for bad in (0, -64, 96):
        assert ctx._L.fm_shared_reserve(ctx._ctx, bad) == -1
    assert ctx._L.fm_shared_reserve(ctx._ctx, 2 * P) == 0
    want = c.good()
    assert ctx._L.fm_shared_reserve(ctx._ctx, 2 * P) == -3 and b"already reserved" in ctx._L.fm_last_error()
    assert torch.equal(c.good(), want)
    ctx.close()
    dense = _ctx(BASE.replace(num_experts=1, expert_top_k=1), shared_inter=None)
    assert dense._L.fm_shared_reserve(dense._ctx, 64) == -1 and b"num_experts > 1" in dense._L.fm_last_error()
    c = Call(dense, seed=43)
    assert c.call(c.args()) == -1 and b"num_experts > 1" in dense._L.fm_last_error()
    assert dense.launch_count == 0
    dense.close()
