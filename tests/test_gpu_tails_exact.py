"""GELU, SwiGLU and the sigmoid router over their tails on exact inputs (tests/exact_tails.py), every launch checked
stage by stage: h and h_s inside the whole-line intervals (GELU below zero and its -0 tail, SwiGLU's subnormal sigma band
and its +-0 cliff), y, ret_y and out bit for bit from the device's own h, and on the gated routes gate_out, picks and
weights against saturated scores with no ambiguous token.  Routes: the router, the caller's routing, the DeepSeek-V3
rule and a Llama-4-style sigmoid k = 1, dense E = 1 and a shared expert; the fused (k <= 2) and gather combines; P = 320,
a partial last GEMM0 tile for both activations.  Per-region counts are printed and must all be nonzero.  Needs an H100."""
import dataclasses

import numpy as np
import pytest
import torch

from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests import exact_gated as eg
from tests import exact_routed as er
from tests import exact_shared as es
from tests import exact_swiglu as sw
from tests import exact_tails as et
from tests import test_gpu_subchunks as gs

pytestmark = pytest.mark.gpu

V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
LLAMA4 = RouterSpec("sigmoid", renormalize=False)


def _cfg(act, E=16, k=2, S=512, H=320, P=320):
    return MoEConfig(num_experts=E, expert_top_k=k, sequence_len=S, hidden_size=H, intermediate_size=P, hidden_act=act)


@dataclasses.dataclass(frozen=True)
class Case:
    cfg: MoEConfig
    route: str = "router"     # "router", "routed" (the caller's) or "gated"
    router: RouterSpec = V3
    shared: int = 0           # Ps of a shared expert (0: none)
    bias: bool = True
    env: tuple = ()
    ns: tuple = (512, 301)

    @property
    def gather(self):
        return dict(self.env).get("FM_FUSED_COMBINE") == "0" or self.cfg.k > 2


CASES = {
    "gelu_router_k2_fused": Case(_cfg(1, k=2)),
    "gelu_routed_k4_gather": Case(_cfg(1, k=4), route="routed"),
    "gelu_gated_v3_k4": Case(_cfg(1, k=4), route="gated"),
    "gelu_gated_llama4_k1_gather": Case(_cfg(1, k=1), route="gated", router=LLAMA4, env=(("FM_FUSED_COMBINE", "0"),)),
    "gelu_dense_E1": Case(_cfg(1, E=1, k=1)),
    "gelu_shared_router_k2": Case(_cfg(1, k=2), shared=192),
    "swiglu_router_k2_gather": Case(_cfg(2, k=2), env=(("FM_FUSED_COMBINE", "0"),)),
    "swiglu_routed_k1": Case(_cfg(2, k=1), route="routed"),
    "swiglu_gated_v3_k2_fused": Case(_cfg(2, k=2), route="gated"),
    "swiglu_gated_llama4_k1": Case(_cfg(2, k=1), route="gated", router=LLAMA4, bias=False),
    "swiglu_dense_E1": Case(_cfg(2, E=1, k=1)),
    "swiglu_shared_gated_v3_k2": Case(_cfg(2, k=2), route="gated", shared=192),
}


def _seed(name):
    return 12000 + sum(map(ord, name))


def _activation_regions(c: Case, inp, toks, n, se):
    """Region counts of the rows every expert (and the shared expert) processed in one launch."""
    reg = {}
    x = inp.x64[:n]
    for e, t in enumerate(toks):
        if len(t) == 0:
            continue
        if c.cfg.hidden_act == 1:
            v = x[t] @ inp.w_up64[e].T + (0 if inp.bu is None else inp.bias64("up")[e])
            et.add_regions(reg, et.gelu_regions(v))
        else:
            wg_, wu, bg, bu = inp.gate_up64(e)
            et.add_regions(reg, et.swiglu_regions(x[t] @ wg_.T + (0 if bg is None else bg),
                                                  x[t] @ wu.T + (0 if bu is None else bu)))
    if se is not None and n:
        if c.cfg.hidden_act == 1:
            v = x @ se.w_up64.T + (0 if se.bu64 is None else se.bu64)
            et.add_regions(reg, {f"h_s {k}": v for k, v in et.gelu_regions(v).items()})
        else:
            w = se.w.double().numpy()
            b = None if se.bu is None else se.bu.double().numpy()
            g, u = x @ w[0].T + (0 if b is None else b[0]), x @ w[1].T + (0 if b is None else b[1])
            et.add_regions(reg, {f"h_s {k}": v for k, v in et.swiglu_regions(g, u).items()})
    return reg


def run_case(name: str, c: Case, monkeypatch):
    from flashmoe_b200.runtime import MoEContext

    for key, v in c.env:
        monkeypatch.setenv(key, v)
    cfg, act = c.cfg, c.cfg.hidden_act
    seed = _seed(name)
    gated = c.route == "gated"
    kw = dict(zero_tokens=2 if cfg.E > 1 and not gated else 0, saturate=gated)
    inp = (et.gelu_tail_inputs if act == 1 else et.swiglu_tail_inputs)(cfg, seed, c.bias, **kw)
    base = inp if act == 1 else inp.base
    se = None
    if c.shared:
        se = (et.gelu_tail_shared if act == 1 else et.swiglu_tail_shared)(cfg.H, c.shared, seed + 3, c.bias)
    sbias = et.score_bias(cfg.E) if gated and c.router.n_group > 1 else None
    routing = er.routing_case(cfg.S, cfg.E, cfg.k, seed, hot=3, hot_frac=0.3) if c.route == "routed" else None
    st, regions, amb_total = ex.Stats(), {}, 0
    ctx = MoEContext(cfg, timeout_ms=10000, shared_inter=c.shared or None)
    try:
        dev_ = ctx.device
        x, wg, we, bu, bd = inp.device(dev_)
        x = x.reshape(cfg.S, cfg.H)
        se_dev = None
        if se is not None:
            se_dev = se.device(dev_) if act == 1 else _shared_swiglu_device(se, dev_)
        sb = None if sbias is None else torch.from_numpy(sbias).to(dev_)
        for n in c.ns:
            fkw = dict(bias_up=bu, bias_down=bd, shared_expert=se_dev)
            if gated:
                out = ctx.forward_gated(x[:n], wg, we, c.router, score_bias=sb, **fkw)
            elif routing is not None:
                idx, w = (torch.from_numpy(a[:n]).to(dev_) for a in routing)
                out = ctx.forward_routed(x[:n], idx, w, we, **fkw)
            else:
                out = ctx.forward_tokens(x[:n], wg, we, **fkw)
            ctx.synchronize()
            dev = gs._device(ctx, cfg, out, n, c.gather, gate_out=act == 1 or gated)
            if cfg.E == 1:
                dev.recv_x = None   # the dense path reads x in place
            s_bits = None
            if se is not None:
                h_s = ctx.read("shared_hidden")[:n].copy()
                y_s = ctx.read("shared_y")[:n].copy()
                if act == 1:
                    es.check_shared(base, se, h_s, y_s, n, act, st)
                else:
                    h_ref, y_ref = sw.shared_reference(se, base.x64[:n], h_s)
                    st.add("h_s", h_s.size, ex.rounded_count(h_ref),
                           ex._interval_check(h_s, h_ref, "h_s", ("token", "column")))
                    ex.check_equal(y_s, y_ref.lo, "y_s", ("token", "column"), signed_zero=False)
                s_bits = y_s
            if gated:
                logits = base.x64[:n] @ base.wg_eff64.T
                amb_total += eg.check_gated_routing(logits, sbias, c.router, cfg.k, dev.topk_idx, dev.gate_out,
                                                    dev.topk_w, (base.x64[:n], base.wg_eff64))
                et.add_regions(regions, et.router_regions(logits, sbias, c.router))
            if act == 1:
                if c.route == "router":
                    ex.check_forward(base, dev, cfg.EC_of(n), n=n, stats=st, shared_s=s_bits)
                else:
                    w_f = eg.weights_f32(dev.topk_w) if gated else routing[1][:n]
                    idx = dev.topk_idx if gated else routing[0][:n]
                    er.check_routed_forward(base, dev, idx, w_f, cfg.EC_of(n), st, shared_s=s_bits)
            else:
                sw.check_experts(inp, dev, cfg.EC_of(n), n, st, shared_s=s_bits, unscaled_k1=c.route == "router")
                if routing is not None:
                    ex.check_equal(dev.topk_idx, er.sanitize(routing[0][:n], cfg.E), "topk_idx", ("token", "pick"))
                if c.route == "router" and cfg.E > 1:
                    ex.check_topk(dev.topk_idx, ex.router_reference(base.x64[:n], base.wg_eff64, cfg.k))
            slot, _, _, _ = er.slots_from_routing(dev.topk_idx, cfg.E, cfg.EC_of(n))
            toks = ex.packet_tokens(dev.topk_idx, slot, cfg.E, cfg.EC_of(n))
            et.add_regions(regions, _activation_regions(c, inp, toks, n, se))
            print(f"  n={n}: ok")
    finally:
        ctx.close()
    return st, regions, amb_total


def _shared_swiglu_device(sh: sw.SharedSwiglu, dev):
    from flashmoe_b200.runtime import SharedExpert

    return SharedExpert(*(None if t is None else t.to(dev) for t in (sh.w, sh.bu, sh.bd)))


def _required(c: Case):
    act = c.cfg.hidden_act
    need = ["GELU v < 0", "GELU -0 tail"] if act == 1 else ["SwiGLU |g| > 4", "SwiGLU subnormal sigma", "SwiGLU cliff"]
    if c.shared:
        need += [f"h_s {k}" for k in need]
    if c.route == "gated":
        need += ["saturated score ties", "+0 scores"]
        if c.router.n_group > 1:
            need += ["absorbed biases", "tied group scores"]
    return need


@pytest.mark.parametrize("name", list(CASES))
def test_tails_every_stage_exact(monkeypatch, name):
    c = CASES[name]
    st, regions, amb = run_case(name, c, monkeypatch)
    print(f"\n[{name}] regions: " + ", ".join(f"{k} {v}" for k, v in regions.items()))
    print(f"[{name}] ambiguous tokens {amb}; {st.line()}")
    empty = [k for k in _required(c) if regions.get(k, 0) == 0]
    assert not empty, f"regions left empty: {empty}"
    assert amb == 0, f"{amb} ambiguous tokens"
