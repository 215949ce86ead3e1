"""GELU, SwiGLU and the sigmoid router over their tails on exact inputs (tests/exact_tails.py), every launch checked
stage by stage: h and h_s inside the whole-line intervals (GELU below zero and its -0 tail, SwiGLU's subnormal sigma band
and its +-0 cliff), y, ret_y and out bit for bit from the device's own h, and on the gated routes gate_out, picks and
weights against saturated scores with no ambiguous token.  Routes: the router, the caller's routing, the DeepSeek-V3
rule and a Llama-4-style sigmoid k = 1, dense E = 1 and a shared expert; the fused (k <= 2) and gather combines; P = 320,
a partial last GEMM0 tile for both activations.  Per-region counts are printed and must all be nonzero.  Needs an H100."""
import dataclasses

import pytest

from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests import exact_tails as et

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


def _activation_regions(inp, toks, n, se):
    """Region counts of the rows every expert (and the shared expert) processed in one launch."""
    reg = {}
    x = inp.x64[:n]
    for e, t in enumerate(toks):
        if len(t):
            et.add_regions(reg, et.activation_regions(inp.experts, e, x[t]))
    if se is not None and n:
        et.add_regions(reg, {f"h_s {k}": v for k, v in et.activation_regions(se, 0, x).items()})
    return reg


def run_case(name: str, c: Case, monkeypatch):
    from flashmoe_b200.runtime import MoEContext

    for key, v in c.env:
        monkeypatch.setenv(key, v)
    cfg = c.cfg
    seed = _seed(name)
    gated = c.route == "gated"
    inp = et.tail_inputs(cfg, seed, c.bias, zero_tokens=2 if cfg.E > 1 and not gated else 0, saturate=gated)
    se = et.tail_shared(cfg.H, c.shared, seed + 3, cfg.hidden_act, c.bias) if c.shared else None
    sbias = et.score_bias(cfg.E) if gated and c.router.n_group > 1 else None
    routing = ex.routing_case(cfg.S, cfg.E, cfg.k, seed, hot=3, hot_frac=0.3) if c.route == "routed" else None
    st, regions, amb_total = ex.Stats(), {}, 0
    ctx = MoEContext(cfg, timeout_ms=10000, shared_inter=c.shared or None)
    try:
        run = ex.Launcher(ctx, c.route, inp, routing=routing, router=c.router, score_bias=sbias)
        for n in c.ns:
            dev, _, amb = run.run(n, se, st)
            amb_total += amb
            if gated:
                et.add_regions(regions, et.router_regions(inp.x64[:n] @ inp.wg_eff64.T, sbias, c.router))
            slot, _, _, _ = ex.slots_from_routing(dev.topk_idx, cfg.E, cfg.EC_of(n))
            toks = ex.packet_tokens(dev.topk_idx, slot, cfg.E, cfg.EC_of(n))
            et.add_regions(regions, _activation_regions(inp, toks, n, se))
            print(f"  n={n}: ok")
    finally:
        ctx.close()
    return st, regions, amb_total


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
