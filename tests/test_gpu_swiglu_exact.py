"""SwiGLU experts (hidden_act = 2) on exact inputs (tests/exact_swiglu.py), every launch checked stage by stage
(exact.check_launch): the routing, every element of `hidden` inside its interval, ret_y and out from the device's own h,
and the shared expert's h_s, y_s and out = rne(r + s).  Cases: the router, the caller's routing (-1 picks, duplicates, an empty expert and
skew past EC) and the gated (DeepSeek-V3 rule) routes; k = 1, 2, 4 on the fused
combine and the gather combine; with and without biases; P = 64 and 128 mod 256 (partial last GEMM0 tile, P = 320,
and whole tiles, P = 384) beside a partial H tile with TN1 = 2; n = S, 301, 1, 0; a context whose CTAs hold more than
128 tokens; E = 1 dense; shared experts of Ps = 64, 192, P; a training context.  Needs an H100."""
import dataclasses

import pytest

from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests import exact_swiglu as sw

pytestmark = pytest.mark.gpu

V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
N_GRID = -1   # a launch's n: grid * 128 + 1 (tokens per CTA above 128)


def _cfg(E=16, k=2, S=512, H=320, P=320, **kw):
    return MoEConfig(num_experts=E, expert_top_k=k, sequence_len=S, hidden_size=H, intermediate_size=P, hidden_act=2,
                     **kw)


@dataclasses.dataclass(frozen=True)
class Case:
    cfg: MoEConfig
    ns: tuple = (512, 301, 1, 0)
    route: str = "router"       # "router", "routed" (the caller's) or "gated"
    bias: bool = True
    shared: tuple = ()     # Ps of the launches' shared expert (one launch per Ps at each n); () = none
    env: tuple = ()


CASES = {
    "k1_fused": Case(_cfg(k=1)),
    "k2_fused_P320": Case(_cfg(k=2)),
    "k2_fused_P384_nobias": Case(_cfg(k=2, P=384), bias=False),
    "k2_gather": Case(_cfg(k=2), env=(("FM_FUSED_COMBINE", "0"),)),
    "k4_gather_P192": Case(_cfg(k=4, P=192)),
    "routed_k1": Case(_cfg(k=1), route="routed"),
    "routed_k2_P192": Case(_cfg(k=2, P=192), route="routed"),
    "routed_k4_gather_nobias": Case(_cfg(k=4), route="routed", bias=False),
    "shared_routed": Case(_cfg(k=2), ns=(512, 301), route="routed", shared=(192,)),
    "gated_v3_k1": Case(_cfg(k=1), route="gated"),
    "gated_v3_k4": Case(_cfg(k=4, P=384), route="gated"),
    "dense_E1": Case(_cfg(E=1, k=1, P=320), ns=(512, 301, 1)),
    "shared_router": Case(_cfg(k=2), ns=(512, 301, 1), shared=(64, 192, 320)),
    "shared_gated_nobias": Case(_cfg(k=2, P=384), ns=(512, 301), route="gated", bias=False, shared=(192, 384)),
    "tpc_over_128": Case(_cfg(k=2, S=20480, P=192), ns=(20480, N_GRID)),
    "training": Case(_cfg(k=2, is_training=1), ns=(512, 301)),
}


def _seed(name):
    return 9000 + sum(map(ord, name))


def _routing(name: str, c: Case):
    """(topk_idx, topk_w) for the S tokens of a caller-routed case: skew past EC onto expert 3, duplicates, -1 picks
    and an empty expert (E - 1)."""
    return ex.routing_case(c.cfg.S, c.cfg.E, c.cfg.k, _seed(name), hot=3, hot_frac=0.3, empty=(c.cfg.E - 1,))


def run_case(name: str, c: Case, monkeypatch):
    """Every launch of the case checked; returns (Stats, ambiguous tokens, tokens)."""
    from flashmoe_b200.runtime import MoEContext

    for key, v in c.env:
        monkeypatch.setenv(key, v)
    inp = sw.swiglu_inputs(c.cfg, _seed(name), bias=c.bias, zero_tokens=2 if c.cfg.E > 1 else 0,
                           wg_range=1 if c.route == "gated" else 4)
    st, amb, tok = ex.Stats(), 0, 0
    ctx = MoEContext(c.cfg, timeout_ms=10000, shared_inter=max(c.shared) if c.shared else None)
    try:
        grid = ctx.dims["grid"]
        run = ex.Launcher(ctx, c.route, inp, routing=_routing(name, c) if c.route == "routed" else None, router=V3)
        for n in c.ns:
            n = grid * 128 + 1 if n == N_GRID else n
            for ps in (c.shared or (None,)):
                sh = None if ps is None else sw.shared_swiglu(c.cfg.H, ps, _seed(name) + ps, bias=c.bias)
                amb += run.run(n, sh, st)[2]
                tok += n
                print(f"  n={n} Ps={ps}: ok")
    finally:
        ctx.close()
    return st, amb, tok


@pytest.mark.parametrize("name", list(CASES))
def test_swiglu_every_stage_exact(monkeypatch, name):
    st, amb, tok = run_case(name, CASES[name], monkeypatch)
    print(f"\n[{name}] ambiguous tokens {amb} of {tok}; {st.line()}")
    h = st.d["hidden"]
    assert h[0] > 0 and h[1] > 0.5 * h[0], f"only {h[1]} of {h[0]} h elements needed rounding"
    assert amb <= ex.MAX_AMBIGUOUS * tok, f"{amb} ambiguous tokens of {tok}"
