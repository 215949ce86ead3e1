"""The shared expert on exact inputs (tests/exact_shared.py), every launch checked stage by stage: the routing tables,
h_s (read back as `shared_hidden`) and y_s against float64 references, and out = rne(r + s) against the route's own
reference composed with s.  Cases: tile tails (H in {192, 320} x Ps in {64, 192, 320, 1408}, partial last Ps and H
tiles, TN1 = 2) with ReLU and GELU on the router, routed and gated routes at n = S, 301, 1, 0; both combines at k = 1, 2,
4, 8 (the router's unscaled k = 1 copy, routed rows with -1, duplicates, an empty expert and skew past EC); GEMM1 lag
modes and many local GEMM0 blocks (E = 256, 1024); 32 row blocks; CTAs whose tokens span two row blocks (tpc > 128);
Ps and n changing on one context; a captured graph replayed over device-side counts; a training context; and
DeepSeek-V3 / Kimi K2 and Llama 4 layer shapes.  Needs an H100; tests/test_shared_exact_cases.py checks the cases and
the checker on the CPU."""
import dataclasses
import time
from typing import Optional

import numpy as np
import pytest
import torch

from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests import exact_gated as eg
from tests import exact_shared as es
from tests import test_gpu_exact as gx

pytestmark = pytest.mark.gpu

V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
LLAMA4 = RouterSpec("sigmoid", renormalize=False)
TAIL_H, TAIL_PS = (192, 320), (64, 192, 320, 1408)
N_GRID = -1            # a launch's n: grid * BLOCK_M + 1 on the context's own grid (tpc > BLOCK_M)


def _cfg(E=16, k=2, S=512, H=256, P=128, **kw):
    return MoEConfig(num_experts=E, expert_top_k=k, sequence_len=S, hidden_size=H, intermediate_size=P, **kw)


@dataclasses.dataclass(frozen=True)
class Case:
    route: str                   # "router", "routed" or "gated"
    cfg: MoEConfig
    launches: tuple              # (Ps, n) of each launch on one context
    env: tuple = ()
    reach: tuple = ()            # regime features some launch must reach on a 132-SM H100 (test_shared_exact_cases)

    @property
    def seed(self):
        return 7000 + sum(map(ord, repr((self.route, self.cfg.E, self.cfg.k, self.cfg.H, self.cfg.S, self.env))))

    @property
    def act(self):
        return self.cfg.hidden_act

    @property
    def lag(self):
        return int(dict(self.env).get("FM_G1_LAG", -1))


def _tail(route, H, act):
    return Case(route, _cfg(H=H, hidden_act=act), tuple((ps, n) for ps in TAIL_PS for n in (512, 301, 1, 0)),
                reach=("ps_tail", "h_tail") + (("TN1>1",) if H > 256 else ()))


CASES = {}
for H in TAIL_H:
    for act in (0, 1):
        for route in ("router", "routed", "gated"):
            CASES[f"tails_{route}_H{H}_{'gelu' if act else 'relu'}"] = _tail(route, H, act)
for k in (1, 2, 4, 8):
    for fused in ((1, 0) if k <= 2 else (0,)):
        for route in ("router", "routed") + (("gated",) if k in (1, 8) else ()):
            CASES[f"combine_{route}_k{k}_{'fused' if fused else 'gather'}"] = Case(
                route, _cfg(k=k, H=320), ((320, 512), (320, 301), (320, 1)), env=(("FM_FUSED_COMBINE", str(fused)),))
for lag in (1, 2):
    for fused in (1, 0):
        CASES[f"g1_lag{lag}_fused{fused}"] = Case("router", _cfg(H=320), ((320, 512), (1408, 301)),
                                                  env=(("FM_G1_LAG", str(lag)), ("FM_FUSED_COMBINE", str(fused))),
                                                  reach=("split_blk<E",))
CASES["E256_local_blocks"] = Case("routed", _cfg(E=256, S=1024), ((320, 1024), (320, 301)))
CASES["E1024_local_blocks"] = Case("router", _cfg(E=1024, S=1024), ((320, 1024), (192, 301)))
CASES["rb32_Ps2048_H1024"] = Case("routed", _cfg(S=4096, H=1024), ((2048, 4096), (2048, 301)), reach=("s_rb>=32",))
CASES["tpc_over_128"] = Case("router", _cfg(S=20480, H=320), ((320, 20480), (320, N_GRID), (64, 1)),
                             reach=("tpc>128", "rb_per_cta>=2"))
CASES["one_context_many_launches"] = Case("router", _cfg(S=1024, H=320),
                                          ((64, 1024), (2048, 1), (320, 301), (64, 0), (2048, 1024)))


def launch_ns(c: Case, grid: int):
    return [(ps, grid * es.BLOCK_M + 1 if n == N_GRID else n) for ps, n in c.launches]


def case_inputs(c: Case):
    """Routed-expert inputs: exact_inputs with biases; ReLU router cases with exact ties, x = 0 tokens and exp
    underflow, GELU ones gelu_friendly (x >= 0), gated ones with small logits (sigmoid's flat tail stays clear)."""
    gen = dict(bias=True, zero_tokens=4)
    if c.act:
        gen.update(gelu_friendly=True, x_range=3, up_range=4)
    elif c.route == "router":
        gen.update(ties=gx.tie_groups(c.cfg.E), underflow_tokens=8)
    if c.route == "gated":
        gen.update(wg_range=1)
    return ex.exact_inputs(c.cfg, seed=c.seed, **gen)


def case_shared(c: Case, Ps: int) -> ex.Experts:
    """The shared expert of a launch with intermediate size Ps: GELU ones gelu_friendly, with W_down_s sparse enough
    that GEMM1's sums stay exact over long Ps."""
    kw = dict(bias=True)
    if c.act:
        kw.update(gelu_friendly=True, up_range=4, down_density=min(1.0, 64 / Ps))
    return es.shared_inputs(c.cfg.H, Ps, seed=c.seed + Ps, act=c.act, **kw)


def case_routing(c: Case):
    """(topk_idx, topk_w) for all S tokens of a routed case: skew past EC onto expert 3, duplicates, -1 picks and an
    empty expert (E - 1)."""
    cfg = c.cfg
    return ex.routing_case(cfg.S, cfg.E, cfg.k, c.seed, hot=3, hot_frac=0.3 if cfg.E <= 16 else 0.05, empty=(cfg.E - 1,))


def case_score_bias(c: Case) -> Optional[np.ndarray]:
    if c.route != "gated":
        return None
    E = c.cfg.E
    return ((np.random.default_rng(c.seed).permutation(E) - E // 2) * 2.0 ** -11).astype(np.float32)


def case_regime(c: Case, Ps: int, n: int, grid: int = eg.H100_SMS) -> es.Regime:
    return es.regime(c.cfg.H, Ps, n, grid, c.cfg.E, c.lag)


def reached(c: Case, grid: int = eg.H100_SMS) -> set:
    """The regime features the case's launches reach on `grid` CTAs."""
    got = set()
    for ps, n in launch_ns(c, grid):
        r = case_regime(c, ps, n, grid)
        got |= {f for f, ok in (("ps_tail", r.ps_tail and n), ("h_tail", r.h_tail and n), ("TN1>1", r.TN1 > 1 and n),
                                ("s_rb>=32", r.s_rb >= 32), ("tpc>128", r.tpc > es.BLOCK_M),
                                ("rb_per_cta>=2", r.rb_per_cta >= 2), ("split_blk<E", r.split_blk < c.cfg.E)) if ok}
    return got


def _ctx(cfg, shared_inter):
    from flashmoe_b200.runtime import MoEContext

    return MoEContext(cfg, timeout_ms=10000, shared_inter=shared_inter)


def launcher(c: Case, ctx, inp) -> ex.Launcher:
    return ex.Launcher(ctx, c.route, inp, routing=case_routing(c) if c.route == "routed" else None, router=V3,
                       score_bias=case_score_bias(c))


TOTAL = ex.Stats()


@pytest.mark.parametrize("name", list(CASES))
def test_shared_every_stage_exact(monkeypatch, name):
    c = CASES[name]
    for key, v in c.env:
        monkeypatch.setenv(key, v)
    t0 = time.time()
    inp = case_inputs(c)
    ctx = _ctx(c.cfg, max(ps for ps, _ in c.launches))
    st, amb, tok = ex.Stats(), 0, 0
    try:
        grid = ctx.dims["grid"]
        missing = set(c.reach) - reached(c, grid)
        assert not missing, f"the launches do not reach {sorted(missing)} on {grid} CTAs"
        run = launcher(c, ctx, inp)
        print(f"\n[{name}] grid {grid}")
        for ps, n in launch_ns(c, grid):
            amb += run.run(n, case_shared(c, ps), st)[2]
            tok += n
            print(f"  Ps={ps} n={n}: {case_regime(c, ps, n, grid).line()}")
    finally:
        ctx.close()
    TOTAL.merge(st)
    print(f"  ambiguous tokens {amb} of {tok}; {time.time() - t0:.1f} s\n  Stats: {st.line()}")
    assert amb <= ex.MAX_AMBIGUOUS * tok, f"{amb} ambiguous tokens of {tok}"


def test_shared_hidden_readback():
    """`shared_hidden` is refused before any launch with a shared expert, then holds [S, Ps] of the last such launch
    (a later launch without one leaves it, and its Ps, as they were)."""
    from flashmoe_b200._lib import FlashMoEError

    c = Case("router", _cfg(H=320), ())
    inp = case_inputs(c)
    ctx = _ctx(c.cfg, 1408)
    try:
        with pytest.raises(FlashMoEError, match=r"h_s exists only after a launch with one"):
            ctx.read("shared_hidden")
        run = launcher(c, ctx, inp)
        for ps in (1408, 192):
            _, rec, _ = run.run(301, case_shared(c, ps))
            assert ctx.read("shared_hidden").shape == (c.cfg.S, ps)
        run.launch(301)
        ctx.synchronize()
        assert np.array_equal(ctx.read("shared_hidden")[:301], rec.h_s)
    finally:
        ctx.close()


def test_graph_device_count_replays_exact():
    """A forward with a shared expert captured with a device-side count, replayed at n = S, 1, 0, 301, 129, S with NaN
    rows past n in x; every replay checked stage by stage, and out's rows past n left untouched."""
    c = Case("router", _cfg(H=320), ())
    t0 = time.time()
    inp = case_inputs(c)
    ps = 320
    se = case_shared(c, ps)
    ctx = _ctx(c.cfg, ps)
    st = ex.Stats()
    try:
        dev = ctx.device
        run = launcher(c, ctx, inp)
        S, H = c.cfg.S, c.cfg.H
        sed = ex.shared_expert(se, dev)
        x_full = run.x.clone()
        cnt = torch.tensor([S], dtype=torch.int32, device=dev)
        out = torch.full((S, H), 3.0, dtype=torch.bfloat16, device=dev)
        s = torch.cuda.Stream(dev)
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            run.launch(S, sed, out=out, n_tokens=cnt, x=x_full)   # warm-up
        torch.cuda.current_stream(dev).wait_stream(s)
        ctx.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            run.launch(S, sed, out=out, n_tokens=cnt, x=x_full)
        for n in (S, 1, 0, 301, 129, S):
            x_full.copy_(run.x)
            x_full[n:] = float("nan")
            out.fill_(3.0)
            cnt.fill_(n)
            g.replay()
            ctx.synchronize()
            assert ctx.launch_record()[1] == n
            assert (out[n:] == 3.0).all(), f"replay n={n}: rows past n written"
            d, rec = run.read(out[:n], n, shared=True)
            run.check(d, rec, n, se, st)
    finally:
        ctx.close()
    TOTAL.merge(st)
    print(f"\n[graph replays, {time.time() - t0:.1f} s] {st.line()}")


def test_training_context_aux_unchanged():
    """Router route on an is_training = 1 context: every stage exact with the shared expert, and gML / gMeC / loss
    inside exact_gated.check_aux's intervals."""
    c = Case("router", _cfg(H=320, is_training=1), ())
    inp = case_inputs(c)
    ps = 320
    se = case_shared(c, ps)
    ctx = _ctx(c.cfg, ps)
    st = ex.Stats()
    try:
        run = launcher(c, ctx, inp)
        grid = ctx.dims["grid"]
        for n in (512, 301, 1, 0):
            d, _, _ = run.run(n, se, st)
            ref = ex.router_reference(inp.x64[:n], inp.wg_eff64, c.cfg.k)
            eg.check_aux(ctx.read("aux_loss").copy(), ref, d.counts, n,
                         eg.regime(c.cfg.E, c.cfg.k, n, grid, eg.tc_router(c.cfg.E)))
            st.add("gML/gMeC/loss", 2 * c.cfg.E + 1)
    finally:
        ctx.close()
    TOTAL.merge(st)
    print(f"\n[training] {st.line()}")


# ----------------------------------------------------------------------------- model shapes
# (name, config, router, Ps): the routed part at these sizes is checked exactly by test_gpu_subchunks' dsv3_layer_shape;
# here it is the same context's call without a shared expert, and out = rne(r_dev + s_ref)
LAYERS = {
    "dsv3_kimi_k2": (_cfg(E=256, k=8, S=2048, H=7168, P=2048), V3, 2048),
    "llama4": (_cfg(E=16, k=1, S=1024, H=5120, P=8192), LLAMA4, 8192),
}


def layer_shared(name):
    cfg, _, ps = LAYERS[name]
    return es.shared_inputs(cfg.H, ps, seed=8000 + len(name), act=cfg.hidden_act, up_range=2, down_range=2)


@pytest.mark.parametrize("name", list(LAYERS))
def test_model_shape_exact(name):
    cfg, router, ps = LAYERS[name]
    t0 = time.time()
    li = eg.layer_inputs(cfg, seed=8100 + len(name))
    se = layer_shared(name)
    ctx = _ctx(cfg, ps)
    st = ex.Stats()
    try:
        dev = ctx.device
        x = li.x.reshape(cfg.S, cfg.H).to(dev)
        wg = li.wg.to(dev)
        g = torch.Generator(device=dev).manual_seed(8200 + len(name))
        we = (torch.randn(cfg.E, 2, cfg.P, cfg.H, device=dev, generator=g) * cfg.H ** -0.5).bfloat16()
        sed = ex.shared_expert(se, dev)
        grid = ctx.dims["grid"]
        for n in (cfg.S, 301):
            r = ctx.forward_gated(x[:n], wg, we, router).clone()
            ctx.synchronize()
            tables = {t: ctx.read(t)[:n].copy() for t in ("topk_idx", "topk_w", "mcw", "slot", "gate_out")}
            tables["counts"] = ctx.read("counts").copy()
            out = ctx.forward_gated(x[:n], wg, we, router, shared_expert=sed)
            ctx.synchronize()
            for t, want in tables.items():
                got = ctx.read(t)[:n] if t != "counts" else ctx.read(t)
                ex.check_equal(got, want, f"{t} (vs the call without a shared expert)", ("row", "column")[:want.ndim])
            st.add("routing tables", sum(v.size for v in tables.values()))
            h_s, y_s = ctx.read("shared_hidden")[:n].copy(), ctx.read("shared_y")[:n].copy()
            ex.shared_stage(li.x64[:n], se, ex.SharedRecord(h_s, y_s), st)
            r_bits = ex.to_bits(r.cpu())
            want = ex.add_shared(ex.Rounded(r_bits, r_bits, 0), y_s)
            ex.check_equal(ex.to_bits(out.cpu()), want.lo, "out = rne(r_dev + s)", ("token", "column"),
                           signed_zero=False)
            st.add("out = rne(r + s)", want.lo.size, ex.rounded_count(want))
            print(f"\n[{name}] n={n}: {es.regime(cfg.H, ps, n, grid, cfg.E).line()}")
    finally:
        ctx.close()
    TOTAL.merge(st)
    print(f"[{name}, {time.time() - t0:.1f} s] {st.line()}")


def test_zz_report_totals():
    print(f"\n[all shared-expert exact checks] {TOTAL.line()}")
