"""The router where a CTA's tokens span several sub-chunks, on exact inputs (tests/exact.py), every stage checked.

A CTA routes its ceil(n / grid) tokens in sub-chunks of TS tokens (tests/exact_gated.py `regime`); everything after the
first sub-chunk -- the logits loop, the GEMV's re-staged gate weights, the score bias staged only by the first one,
the picks written at (s0 + ti) * k, the training column sums, slot_ranks over tpc * k entries -- is its own regime.
These cases enter it on the plain router (CUDA-core GEMV and tensor cores, up to a full tpc * k = G_SEL_MAX scratch),
on gated launches with the rules of DeepSeek-V3, Kimi K2, Qwen-MoE, Llama 4 and a 32-group softmax, on routed launches
and in training mode.  Each case runs at n = S, at n = grid * TS + 1 (CTAs whose last sub-chunk holds one token, and
trailing CTAs with none) and at n = 1, on one context.  Needs an H100; tests/test_subchunk_cases.py checks the cases
and their checkers on the CPU."""
import dataclasses
import os
import time
from typing import Optional

import numpy as np
import pytest
import torch

from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from oracle import moe_oracle as mo
from tests import exact as ex
from tests import exact_gated as eg
from tests import test_gpu_exact as gx

pytestmark = pytest.mark.gpu

V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
KIMI_K2 = RouterSpec("sigmoid", renormalize=True, scale=2.827)
QWEN = RouterSpec("softmax", renormalize=False)
LLAMA4 = RouterSpec("sigmoid", renormalize=False)
GROUPS_1024 = RouterSpec("softmax", 32, 4, 2, False, 1.0)


@dataclasses.dataclass(frozen=True)
class Case:
    kind: str                          # "router", "gated" or "routed"
    cfg: MoEConfig
    min_sub: int                       # sub-chunks of the fullest CTA at n = S on a 132-SM H100
    full_scratch: bool = False         # tpc * k = G_SEL_MAX at n = S on a 132-SM H100
    router: Optional[RouterSpec] = None
    bias_log2: Optional[int] = None    # score bias (permutation(E) - E / 2) * 2^bias_log2; None: no bias
    env: tuple = ()
    gen: tuple = ()                    # exact_inputs keyword arguments
    layer: bool = False                # exact_gated.layer_inputs (a model-sized layer) instead of exact_inputs
    amb_share: float = 0.001           # ambiguous tokens allowed (their picks are not checked)

    @property
    def seed(self):
        return 5000 + self.cfg.E + 7 * self.cfg.k


def _cfg(E, k, S, H=128, P=128, **kw):
    return MoEConfig(num_experts=E, expert_top_k=k, sequence_len=S, hidden_size=H, intermediate_size=P, **kw)


S_MAX_K8 = eg.regime(256, 8, 0, eg.H100_SMS, True).s_max    # 135168: tpc * k = 8192 on 132 SMs
CASES = {
    "router_E16_k2": Case("router", _cfg(16, 2, 131072), 2),
    "router_E384_k8": Case("router", _cfg(384, 8, 8192), 2),
    "router_E1024_k2": Case("router", _cfg(1024, 2, 4096), 3),
    "router_E1024_k2_gather": Case("router", _cfg(1024, 2, 4096), 3, env=(("FM_FUSED_COMBINE", "0"),)),
    "router_E256_k8_full_scratch": Case("router", _cfg(256, 8, S_MAX_K8), 17, True),
    # (sigmoid: logits kept small, so that scores a grid step apart do not meet in sigmoid's flat tail; softmax over
    # 1024 experts: large logits, so that probabilities stand clear of the wide intervals of a 1024-term denominator)
    "gated_dsv3": Case("gated", _cfg(256, 8, 16384), 2, router=V3, bias_log2=-11, gen=(("wg_range", 1),)),
    "gated_dsv3_full_scratch": Case("gated", _cfg(256, 8, S_MAX_K8), 17, True, router=V3, bias_log2=-11,
                                    gen=(("wg_range", 1),)),
    "gated_kimi_k2": Case("gated", _cfg(384, 8, 16384), 3, router=KIMI_K2, bias_log2=-11, gen=(("wg_range", 1),)),
    # (a 1024-term softmax denominator widens every probability's interval to about 1e-3 relative: up to 0.25 %
    # of the tokens are left undecided, 0.12 % on a 132-SM H100)
    "gated_E1024_groups": Case("gated", _cfg(1024, 2, 4096), 3, router=GROUPS_1024, bias_log2=-9,
                               gen=(("wg_range", 8),), amb_share=0.0025),
    "gated_qwen_E128": Case("gated", _cfg(128, 8, 32768), 2, router=QWEN),
    "gated_llama4_E128_k1": Case("gated", _cfg(128, 1, 32768), 2, router=LLAMA4),
    "routed_E256_k8_full_scratch": Case("routed", _cfg(256, 8, S_MAX_K8), 17, True),
    "routed_E1024_k2": Case("routed", _cfg(1024, 2, 4096), 3),
    "training_E1024_k2": Case("router", _cfg(1024, 2, 4096, is_training=1), 3),
    "training_E128_k2": Case("router", _cfg(128, 2, 32768, is_training=1), 2),
    # DeepSeek-V3's own layer: 112 k-blocks of d_model in each of the tensor-core router's two passes
    "dsv3_layer_shape": Case("gated", _cfg(256, 8, 4096, H=7168, P=2048), 1, router=V3, bias_log2=-11, layer=True),
}


def max_ambiguous(c: Case, n: int) -> int:
    """Tokens whose picks the intervals cannot decide are not checked; at most a share c.amb_share of them may be."""
    return int(n * c.amb_share)


def case_regime(c: Case, n: int, grid: int = eg.H100_SMS, env=None) -> eg.Regime:
    """The regime of n tokens on `grid` CTAs, on the router path the case's environment and `env` (default: this
    process's environment, which the kernel reads too) select."""
    env = {**(os.environ if env is None else env), **dict(c.env)}
    return eg.regime(c.cfg.E, c.cfg.k, n, grid, eg.tc_router(c.cfg.E, env) and c.kind != "routed")


def token_counts(c: Case, grid: int = eg.H100_SMS, env=None):
    """n = S, n = grid * TS + 1 where that is below S, and n = 1."""
    mid = grid * case_regime(c, c.cfg.S, grid, env).TS + 1
    return (c.cfg.S,) + ((mid,) if mid < c.cfg.S else ()) + (1,)


def for_device(c: Case, sms: int) -> Case:
    """A full-scratch case sized for a device of `sms` SMs (S = the largest that fills tpc * k = G_SEL_MAX there);
    every other case as it is."""
    if not c.full_scratch:
        return c
    return dataclasses.replace(c, cfg=c.cfg.replace(sequence_len=eg.regime(c.cfg.E, c.cfg.k, 0, sms, False).s_max))


def case_inputs(c: Case):
    if c.layer:
        return eg.layer_inputs(c.cfg, seed=c.seed)
    gen = dict(c.gen)
    if c.kind == "router":   # the router cases of tests/test_gpu_exact.py: exact ties, x = 0 tokens, exp underflow
        gen = dict(ties=gx.tie_groups(c.cfg.E), zero_tokens=4, underflow_tokens=8)
    return ex.exact_inputs(c.cfg, seed=c.seed, **gen)


def case_bias(c: Case) -> Optional[np.ndarray]:
    if c.bias_log2 is None:
        return None
    E = c.cfg.E
    return ((np.random.default_rng(c.seed).permutation(E) - E // 2) * 2.0 ** c.bias_log2).astype(np.float32)


def case_routing(c: Case):
    """(topk_idx, topk_w) of a routed case for all S tokens: skew past EC onto expert 3, duplicates, -1 and an empty
    expert (E - 1); the first n rows are a launch's routing."""
    E, k = c.cfg.E, c.cfg.k
    return ex.routing_case(c.cfg.S, E, k, c.seed, hot=3, hot_frac=0.05, empty=(E - 1,))


def _check_training(ctx, c, inp, dev, n, rg):
    """gML / gMeC / loss against the intervals of exact_gated.check_aux, and against the C oracle with
    test_gpu_parity.test_training_mode_aux_loss_matches_oracle's tolerances."""
    cfg = c.cfg
    aux = ctx.read("aux_loss").copy()
    ref = ex.router_reference(inp.x64[:n], inp.wg_eff64, cfg.k)
    eg.check_aux(aux, ref, dev.counts, n, rg)
    xb = ex.to_bits(inp.x.reshape(cfg.S, cfg.H))[:n]
    gml, gmec, loss = mo.aux_loss(xb, mo.gate_weights_effective(ex.to_bits(inp.wg), cfg.E, cfg.H), k=cfg.k,
                                  EC=cfg.EC_of(n))
    np.testing.assert_allclose(aux[:cfg.E], gml, rtol=2e-5, atol=1e-7)
    np.testing.assert_allclose(aux[cfg.E:2 * cfg.E], gmec, rtol=1e-6)
    np.testing.assert_allclose(aux[2 * cfg.E], loss, rtol=2e-5)


@pytest.mark.parametrize("name", list(CASES))
def test_subchunks_every_stage_exact(monkeypatch, name):
    from flashmoe_b200.runtime import MoEContext

    c = for_device(CASES[name], torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count)
    cfg = c.cfg
    for key, v in c.env:
        monkeypatch.setenv(key, v)
    t_start = time.time()
    inp = case_inputs(c)
    bias = case_bias(c)
    ctx = MoEContext(cfg, timeout_ms=10000)
    try:
        grid = ctx.dims["grid"]
        rg = case_regime(c, cfg.S, grid)
        print(f"\n[{name}] grid {grid}, S {cfg.S}: tpc {rg.tpc}, TS {rg.TS}, fullest CTA's sub-chunks "
              f"{len(rg.sub_chunks)} {rg.sub_chunks}, tpc * k {rg.sel_entries}")
        if c.kind != "routed":
            assert len(rg.sub_chunks) >= c.min_sub, f"the fullest CTA takes {len(rg.sub_chunks)} sub-chunks"
        if c.full_scratch:
            assert rg.sel_entries == eg.G_SEL_MAX, f"tpc * k = {rg.sel_entries}, not the full router scratch"
        run = ex.Launcher(ctx, c.kind, inp, routing=case_routing(c) if c.kind == "routed" else None,
                          router=c.router, score_bias=bias)
        st = ex.Stats()
        amb = 0
        for n in token_counts(c, grid):
            d, _, a = run.run(n, stats=st)
            amb += a
            if cfg.is_training:
                _check_training(ctx, c, inp, d, n, case_regime(c, n, grid))
                st.add("gML/gMeC/loss", 2 * cfg.E + 1)
            rn = case_regime(c, n, grid)
            print(f"  n={n}: fullest CTA {len(rn.sub_chunks)} sub-chunk(s) {rn.sub_chunks[:4]}"
                  f"{' ...' if len(rn.sub_chunks) > 4 else ''}")
    finally:
        ctx.close()
    tok = sum(token_counts(c, grid))
    print(f"  ambiguous tokens {amb} of {tok}; {time.time() - t_start:.1f} s\n  Stats: {st.line()}")
    assert amb <= max_ambiguous(c, tok), f"{amb} ambiguous tokens of {tok}"
