"""Every stage of the forward, checked element by element on inputs whose sums are exact in fp32 (tests/exact.py):
top-k, gate_out, topk_w, mcw, slots, counts, recv_cnt, the dispatched rows, h, the returned y and the output, on every
launch.  Shapes cover the router paths (lane groups, CUDA-core GEMV, tensor-core router with one and two passes over
d_model), exact ties and exp underflow, GEMM tile tails, planned packet sizes, both combine paths, the GEMM1 lag modes,
the dense path, per-call token counts and repeated launches.  Needs an H100."""
import time

import numpy as np
import pytest

from flashmoe_b200.config import BASELINE_CONFIGS, MoEConfig
from tests import exact as ex

pytestmark = pytest.mark.gpu

MIN_H_ROUNDED, MIN_OUT_ROUNDED = 0.02, 0.2   # shares of h / out elements (k >= 2) whose exact value needs rounding


def _lpt(E):
    """Lanes per token of the router's softmax / top-k (fm_kernel.cuh softmax_topk_lanes)."""
    if E <= 8:
        p = 1
        while p < E:
            p <<= 1
        return p
    return 4 if E <= 128 else 8 if E <= 256 else 16 if E <= 512 else 32


def tie_groups(E):
    """Duplicated Wg_eff rows: the first and the last expert, two experts on the same lane, two on neighbouring lanes,
    and a pair split across the tensor-core router's 128-expert pass boundary."""
    L = _lpt(E)
    groups = [(0, E - 1)]
    if 1 + L < E - 1:
        groups.append((1, 1 + L))
    groups.append((2, 3) if E > 4 else (1, 2))
    if E > 133:
        groups.append((5, 133))
    return groups


def _cfg(E=8, k=2, S=512, H=128, P=128, **kw):
    return MoEConfig(num_experts=E, expert_top_k=k, sequence_len=S, hidden_size=H, intermediate_size=P, **kw)


def _routing_case(E, k, S=512, H=128, P=128, **cfg_kw):
    return _cfg(E, k, S, H, P, **cfg_kw), dict(ties=tie_groups(E), zero_tokens=4, underflow_tokens=8)


def _planned(counts, seed):
    fc = np.repeat(np.arange(len(counts)), counts)
    return np.random.default_rng(seed).permutation(fc)


# name -> (config, generator keyword arguments, environment)
CASES = {}
for E, k in ((4, 3), (8, 2), (16, 2), (17, 2), (64, 4), (128, 8), (129, 2), (256, 2), (257, 2), (1024, 2)):
    cfg, gen = _routing_case(E, k)
    for tc in ((0, 1) if E <= 256 else (None,)):
        env = {} if tc is None else {"FM_TC_GATE": str(tc)}
        CASES[f"router_E{E}_k{k}" + ("" if tc is None else f"_tc{tc}")] = (cfg, gen, env)
CASES["E32_router_subchunks"] = (*_routing_case(32, 2, S=20480), {})
for H in (64, 192, 320):
    CASES[f"H{H}"] = (*_routing_case(8, 2, H=H), {})
for P in (64, 192, 448):
    CASES[f"P{P}"] = (*_routing_case(8, 2, P=P), {})
CASES["H2048_S8192"] = (_cfg(8, 2, S=8192, H=2048),
                        dict(ties=tie_groups(8), zero_tokens=4, underflow_tokens=8, wg_range=1), {})
CASES["packets_0_1_127_128_129"] = (_cfg(8, 1, drop_tokens=0),
                                    dict(first_choice=_planned([0, 1, 127, 128, 129, 127, 0, 0], 1)), {})
CASES["packet_cut_at_EC"] = (_cfg(8, 1), dict(first_choice=_planned([0, 1, 63, 64, 65, 200, 119, 0], 2)), {})
CASES["capacity_factor_2"] = (_cfg(8, 2, capacity_factor=2),
                              dict(first_choice=_planned([257, 255, 0, 0, 0, 0, 0, 0], 3)), {})
CASES["no_drop_k2"] = (_cfg(8, 2, drop_tokens=0), dict(first_choice=_planned([300, 0, 100, 0, 50, 62, 0, 0], 4)), {})
CASES["mini_batch_3"] = (*_routing_case(8, 2, S=128, mini_batch=3), {})
CASES["bias_relu"] = (_cfg(8, 2), dict(bias=True, ties=[(0, 7)], zero_tokens=4), {})
CASES["bias_gelu"] = (_cfg(8, 2, hidden_act=1), dict(bias=True, gelu_friendly=True, x_range=3, up_range=4,
                                                     ties=[(0, 7)], zero_tokens=4), {})
CASES["gelu_gather"] = (_cfg(8, 2, hidden_act=1), dict(bias=True, gelu_friendly=True, x_range=3, up_range=4),
                        {"FM_FUSED_COMBINE": "0"})
CASES["fused_k1"] = (*_routing_case(8, 1), {})
CASES["fused_k2"] = (*_routing_case(8, 2), {})
CASES["gather_k1"] = (*_routing_case(8, 1), {"FM_FUSED_COMBINE": "0"})
CASES["gather_k2"] = (*_routing_case(8, 2), {"FM_FUSED_COMBINE": "0"})
CASES["k3"] = (*_routing_case(8, 3), {})
CASES["k8"] = (*_routing_case(16, 8), {})
for lag in (1, 2):   # TCM = 3: an odd number of row blocks per packet (test_alternate_kernel_modes' odd_row_blocks)
    for fused in (1, 0):
        CASES[f"g1_lag{lag}_fused{fused}"] = (_cfg(4, 2, S=768, H=256, P=512), dict(zero_tokens=4),
                                              {"FM_G1_LAG": str(lag), "FM_FUSED_COMBINE": str(fused)})
CASES["dense_E1"] = (_cfg(1, 1, S=256, P=512), {}, {})
CASES["dense_E1_general_path"] = (_cfg(1, 1, S=256, P=512), {}, {"FM_DENSE_E1": "0"})

# multi-launch cases: (config, generator keyword arguments) per launch, checked in full
EPILOGUE_ORDER = _cfg(64, 2, S=2048, H=256, P=1024)       # tests/test_gpu_epilogue_order.py's shape
CONFIG_B = BASELINE_CONFIGS["B"]
CONFIG_B_GEN = dict(x_range=8, wg_range=2, up_range=4, down_range=3)
TOKEN_COUNTS = (1, 31, 129, 300, 0, 512)
TOKENS_CFG = _cfg(8, 2, S=512)


def _ctx(cfg):
    from flashmoe_b200.runtime import MoEContext

    return MoEContext(cfg, timeout_ms=5000)


def _launch_and_check(ctx, inp, stats, n=None):
    """One forward on `inp` (n = None: MoEContext.forward of all S tokens, else forward_tokens of n), checked."""
    run = ex.Launcher(ctx, "router", inp)
    out = run.launch(n)
    ctx.synchronize()
    n = inp.cfg.S if n is None else n
    dev, _ = run.read(out, n)
    run.check(dev, None, n, stats=stats)


TOTAL = ex.Stats()


@pytest.mark.parametrize("name", list(CASES))
def test_every_stage_exact(monkeypatch, name):
    cfg, gen, env = CASES[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    inp = ex.exact_inputs(cfg, seed=1000 + sum(map(ord, name)), **gen)
    st = ex.Stats()
    ctx = _ctx(cfg)
    try:
        _launch_and_check(ctx, inp, st)
    finally:
        ctx.close()
    TOTAL.merge(st)
    print(f"\n[{name}] {st.line()}")


def test_token_counts_on_one_context():
    """forward_tokens with n = 1, 31, 129, 300, 0, 512 on one context; every call checked at capacity EC_of(n)."""
    cfg = TOKENS_CFG
    inp = ex.exact_inputs(cfg, seed=2000, ties=tie_groups(cfg.E), zero_tokens=4, underflow_tokens=8)
    st = ex.Stats()
    ctx = _ctx(cfg)
    try:
        for n in TOKEN_COUNTS:
            _launch_and_check(ctx, inp, st, n=n)
    finally:
        ctx.close()
    TOTAL.merge(st)
    print(f"\n[token counts] {st.line()}")


@pytest.mark.parametrize("fused", [1, 0])
def test_epilogue_order_shape_five_launches(monkeypatch, fused):
    """GEMM1 then GEMM0 tiles on one CTA (FM_G1_LAG=1) at tests/test_gpu_epilogue_order.py's shape: five launches with
    different inputs on one context, each checked in full."""
    monkeypatch.setenv("FM_G1_LAG", "1")
    monkeypatch.setenv("FM_FUSED_COMBINE", str(fused))
    cfg = EPILOGUE_ORDER
    st = ex.Stats()
    ctx = _ctx(cfg)
    try:
        for i in range(5):
            inp = ex.exact_inputs(cfg, seed=3000 + 10 * fused + i, ties=tie_groups(cfg.E), zero_tokens=4)
            _launch_and_check(ctx, inp, st)
    finally:
        ctx.close()
    TOTAL.merge(st)
    print(f"\n[epilogue order, fused={fused}] {st.line()}")


def test_config_B_three_launches_and_gather(monkeypatch):
    """Full-size config B: three fused launches with different inputs on one context, every element of hidden and out
    checked; then one gather-path launch on a second context for ret_y."""
    cfg = CONFIG_B
    st = ex.Stats()
    t0 = time.time()
    ctx = _ctx(cfg)
    try:
        for i in range(3):
            _launch_and_check(ctx, ex.exact_inputs(cfg, seed=4000 + i, **CONFIG_B_GEN), st)
    finally:
        ctx.close()
    monkeypatch.setenv("FM_FUSED_COMBINE", "0")
    ctx = _ctx(cfg)
    try:
        _launch_and_check(ctx, ex.exact_inputs(cfg, seed=4010, **CONFIG_B_GEN), st)
    finally:
        ctx.close()
    TOTAL.merge(st)
    print(f"\n[config B, {time.time() - t0:.1f} s] {st.line()}")


def test_zz_report_totals():
    print(f"\n[all exact checks] {TOTAL.line()}")
