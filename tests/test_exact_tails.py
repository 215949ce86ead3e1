"""The tail references (exact.gelu_rounded, exact_swiglu.silu_mul_rounded, exact_gated.sigmoid_bounds and the exact
selection values of check_gated_routing) on the CPU: an fp32 step-by-step emulation of the kernel's gelu_erf, silu_mul
and sigmoid_score, with erff and ex2 at the ends of their documented errors, lies inside them at every grid point; they
equal the earlier references where those applied; the tail inputs (tests/exact_tails.py) populate every region with no
ambiguous token; and the checkers reject planted faults.  CPU only."""
import numpy as np
import pytest
from scipy.special import erf, erfc

from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests import exact_gated as eg
from tests import exact_swiglu as sw
from tests import exact_tails as et

V3 = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)
LLAMA4 = RouterSpec("sigmoid", renormalize=False)
GELU_V = np.arange(-12 * 8, 10 * 8 + 1) / 8.0            # 2^-3 grid over [-12, 10]
SWIGLU_G = np.arange(-2 * 140, 2 * 140 + 1) / 2.0        # 1/2 grid over [-140, 140]
LOGITS = np.arange(-110 * 64, 110 * 64 + 1) / 64.0       # 2^-6 grid over [-110, 110]


def _inside(bits, r: ex.Rounded) -> np.ndarray:
    k = ex.order_key(bits)
    return (k >= ex.order_key(r.lo)) & (k <= ex.order_key(r.hi))


# ----------------------------------------------------------------------------- fp32 emulations of the kernel
def _erff_choices(t):
    """erff(t) as an fp32 number: correctly rounded, and at both ends of its 2-ulp bound (clamped to [-1, 1])."""
    e = erf(t)
    du = ex.ERFF_ULP * ex.ulp32(e)
    return [e.astype(np.float32), np.maximum(ex.f32_up(e - du), np.float32(-1)),
            np.minimum(ex.f32_down(e + du), np.float32(1))]


def gelu_emul(v, e32=None):
    """gelu_erf in fp32 steps: 0.5f * v * (1.0f + erff(v * 0.70710678f)); erff's result `e32` (default correctly
    rounded)."""
    v32 = np.asarray(v, np.float32)
    t = (v32 * ex.SQRT1_2_F32).astype(np.float32)
    e = erf(t.astype(np.float64)).astype(np.float32) if e32 is None else e32
    return ((np.float32(0.5) * v32).astype(np.float32) * (np.float32(1) + e).astype(np.float32)).astype(np.float32)


def _ex2_choices(a):
    """ex2.approx.ftz(a) as fp32: correctly rounded, and the innermost fp32 values at both ends of 2^-21 relative;
    +inf from a = 128 on or past the fp32 range, +0 below 2^-126."""
    p = np.exp2(np.minimum(a, 1000.0))
    out = []
    for v in (p, ex.f32_up(p * (1 - ex.EPS_EX2)).astype(np.float64), ex.f32_down(p * (1 + ex.EPS_EX2)).astype(np.float64)):
        with np.errstate(over="ignore"):
            f = np.where((a >= 128) | (v > ex.FLT_MAX), np.inf, v).astype(np.float32)
        out.append(np.where(f < 2.0 ** -126, np.float32(0), f).astype(np.float32))
    return out


def sigmoid_emul(l, p32=None):
    """sigmoid_score in fp32 steps: __frcp_rn(__fadd_rn(1, ex2(fl(-l * log2e)))); ex2's result `p32`."""
    a = (-np.asarray(l, np.float32) * ex.LOG2E_F32).astype(np.float32)
    p = _ex2_choices(a.astype(np.float64))[0] if p32 is None else p32
    with np.errstate(over="ignore"):
        return (np.float32(1) / (np.float32(1) + p).astype(np.float32)).astype(np.float32)


def silu_mul_emul(g, u, p32=None):
    g32, u32 = np.asarray(g, np.float32), np.asarray(u, np.float32)
    return ((g32 * sigmoid_emul(g32, p32)).astype(np.float32) * u32).astype(np.float32)


# ----------------------------------------------------------------------------- emulation inside the references
def test_gelu_emulation_inside_the_interval_over_the_whole_line():
    r = ex.gelu_rounded(GELU_V)
    t = (GELU_V.astype(np.float32) * ex.SQRT1_2_F32).astype(np.float32).astype(np.float64)
    for e32 in _erff_choices(t):
        h = ex.f32_to_bf16(gelu_emul(GELU_V, e32))
        bad = ~_inside(h, r)
        assert not bad.any(), f"v = {GELU_V[bad][:5]}: emulated {h[bad][:5]}, interval {r.lo[bad][:5]} .. {r.hi[bad][:5]}"
    # the cancellation the relative bound cannot cover, and the -0 tail (correctly rounded erff)
    h = gelu_emul(np.array([-5.0, -5.5, -6.0, -8.0]))
    assert abs(h[0] / -1.433e-6 - 1) > 0.03 and h[1] < -1.5e-7 and h[2] == 0 and h[3] == 0
    assert np.signbit(h[2]) and 0.5 * -6.0 * erfc(6.0 / np.sqrt(2)) < -5e-9   # -0, while GELU(-6) is a normal bf16
    assert (ex.order_key(r.hi[GELU_V <= -6]) == 0).all() and (ex.order_key(r.lo[(GELU_V >= -1) & (GELU_V != 0)]) != 0).all()


def test_silu_mul_emulation_inside_the_interval_over_g_in_pm140():
    g = np.repeat(SWIGLU_G, 6)
    u = np.tile([-7.0, -3.0, -1.0, 1.0, 3.0, 7.0], SWIGLU_G.size)
    r = sw.silu_mul_rounded(g, u)
    a = sw.power_arg(g)
    for p32 in _ex2_choices(a):
        h = ex.f32_to_bf16(silu_mul_emul(g, u, p32))
        bad = ~_inside(h, r)
        assert not bad.any(), f"g = {g[bad][:5]}, u = {u[bad][:5]}: emulated {h[bad][:5]}, [{r.lo[bad][:5]}, {r.hi[bad][:5]}]"
    # the cliff: from g = -89 (fl(-g log2e) >= 128) h is exactly +-0, while the real value still rounds to a nonzero
    # bf16 number; the subnormal sigma band just above it
    assert sw.power_arg(np.array([-88.5]))[0] < 128 <= sw.power_arg(np.array([-89.0]))[0]
    cliff = (g <= -89) & (g >= -94)
    assert (ex.order_key(r.lo[cliff]) == 0).all() and (ex.order_key(r.hi[cliff]) == 0).all()
    assert (ex.order_key(ex.f64_to_bf16(r.exact[cliff])) != 0).all()
    band = np.isin(g, [-88.5, -88.0, -87.5])
    s = sigmoid_emul(g[band])
    assert (s < 2.0 ** -126).all() and (s > 0).all()
    assert (ex.order_key(r.lo[band]) != 0).all()


def test_sigmoid_emulation_inside_the_bounds_exact_where_saturated():
    lo, hi, mid = eg.sigmoid_bounds(LOGITS)
    a = (-LOGITS * float(ex.LOG2E_F32)).astype(np.float32).astype(np.float64)
    for p32 in _ex2_choices(a):
        s = sigmoid_emul(LOGITS, p32).astype(np.float64)
        bad = (s < lo) | (s > hi)
        assert not bad.any(), f"l = {LOGITS[bad][:5]}: emulated {s[bad][:5]}, bounds {lo[bad][:5]} .. {hi[bad][:5]}"
    assert (lo[LOGITS >= 18] == 1).all() and (hi[LOGITS >= 18] == 1).all()
    assert (lo[LOGITS <= -89] == 0).all() and (hi[LOGITS <= -89] == 0).all()
    assert (lo[np.abs(LOGITS) < 17] < hi[np.abs(LOGITS) < 17]).all()


# ----------------------------------------------------------------------------- equal to the earlier references
def test_tail_references_equal_the_earlier_ones_where_those_applied():
    from scipy.special import erf as erf64

    v = GELU_V[GELU_V >= 0]
    gl = 0.5 * v * (1.0 + erf64(v / np.sqrt(2.0)))
    r = ex.gelu_rounded(v)
    assert np.array_equal(r.lo, ex.f64_to_bf16(gl * (1 - ex.EPS_GELU)))
    assert np.array_equal(r.hi, ex.f64_to_bf16(gl * (1 + ex.EPS_GELU)))
    assert not r.wide_ok.any()
    g = np.repeat(SWIGLU_G[SWIGLU_G >= sw.G_MIN], 3)
    u = np.tile([-5.0, 1.0, 2.0], g.size // 3)
    r = sw.silu_mul_rounded(g, u)
    with np.errstate(over="ignore"):
        vv = g / (1.0 + np.exp(-g)) * u
    e = sw.eps_swiglu(g)
    a, b = ex.f64_to_bf16(vv * (1 - e)), ex.f64_to_bf16(vv * (1 + e))
    swap = ex.order_key(a) > ex.order_key(b)
    assert np.array_equal(r.lo, np.where(swap, b, a)) and np.array_equal(r.hi, np.where(swap, a, b))
    lo, hi, _ = eg.sigmoid_bounds(LOGITS)
    s = 1.0 / (1.0 + np.exp(-LOGITS))
    eps = 2.0 ** -21 + 2.0 ** -24 * (np.abs(LOGITS) * 1.01 + 3)
    # the earlier sigmoid interval left out fl32(log2 e)'s own error (|l| 2^-26 relative in the power, which the
    # emulation above reaches for |l| near 50); the corrected one contains it, and is within 2^-21 of it for |l| <= 4
    old = (LOGITS > -86) & (LOGITS < 17)
    assert ((lo <= s * (1 - eps)) & (hi >= s * (1 + eps)))[old].all()
    small = np.abs(LOGITS) <= 4
    assert np.allclose(lo[small], (s * (1 - eps))[small], rtol=2 ** -21, atol=0)
    sat = LOGITS >= 18   # the saturated value lies inside the earlier interval
    assert ((s * (1 - eps))[sat] <= 1).all() and ((s * (1 + eps))[sat] >= 1).all()


# ----------------------------------------------------------------------------- the tail inputs
def _cfg(act, E=16, k=2, S=512, H=320, P=320):
    return MoEConfig(num_experts=E, expert_top_k=k, sequence_len=S, hidden_size=H, intermediate_size=P, hidden_act=act)


def test_gelu_tail_inputs_reach_every_region_and_keep_gemm1_exact():
    cfg = _cfg(1)
    inp = et.tail_inputs(cfg, 5, bias=True)
    st = ex.check_preconditions(inp, cfg.EC, 0.3, 0.3)   # the reference's own launch passes every check
    assert st.d["hidden"][2] > 0
    regions = {}
    for e in range(cfg.E):
        et.add_regions(regions, et.activation_regions(inp.experts, e, inp.x64))
    assert regions["GELU v < 0"] > 1000 and regions["GELU -0 tail"] > 100, regions
    v = inp.experts.pre(0, inp.x64)[0]
    assert v.min() >= -11 and v.max() < 200 and (v[:, ~et.tail_columns(cfg.P)] >= 0).all()


def test_swiglu_tail_inputs_reach_every_region_and_keep_gemm1_exact():
    cfg = _cfg(2)
    inp = et.tail_inputs(cfg, 6, bias=True)
    xp = inp.experts
    regions = {}
    for e in range(cfg.E):
        g, u = xp.pre(e, inp.x64)
        et.add_regions(regions, et.swiglu_regions(g, u))
        xp.y(e, xp.h(e, inp.x64).lo)   # asserts exact sums
        assert np.abs(g).max() <= 136
    assert all(v > 50 for v in regions.values()), regions


@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("router,k", [(V3, 4), (V3, 2), (LLAMA4, 1)], ids=["v3_k4", "v3_k2", "llama4_k1"])
def test_saturating_router_inputs_are_decided(act, router, k):
    """Every token of the saturated-router inputs is decided (ties by the lower index or group, absorbed biases),
    and the regions are populated; the reference's own launch passes check_gated_routing."""
    cfg = _cfg(act, k=k)
    inp = et.tail_inputs(cfg, 7, bias=False, saturate=True)
    bias = et.score_bias(cfg.E) if router.n_group > 1 else None
    logits = inp.x64 @ inp.wg_eff64.T
    picks, w, gate_out = eg.reference_routing(router, bias, k, inp.x64, inp.wg_eff64)
    amb = eg.check_gated_routing(logits, bias, router, k, picks, gate_out, ex.f32_to_bf16(w), (inp.x64, inp.wg_eff64))
    assert amb == 0
    reg = et.router_regions(logits, bias, router)
    assert reg["saturated score ties"] > 100 and reg["+0 scores"] > 50, reg
    if bias is not None:
        assert reg["absorbed biases"] > 100 and reg["tied group scores"] > 100, reg


# ----------------------------------------------------------------------------- planted faults
def _rejects(got_bits, r: ex.Rounded):
    with pytest.raises(AssertionError, match="outside the reference"):
        ex._interval_check(got_bits, r, "h", ("element",), max_width=None)


def test_gelu_checker_accepts_the_kernel_and_rejects_tanh_and_relu_below_zero():
    r = ex.gelu_rounded(GELU_V)
    ex._interval_check(ex.f32_to_bf16(gelu_emul(GELU_V)), r, "h", ("element",))
    v = GELU_V
    tanh = 0.5 * v * (1 + np.tanh(np.sqrt(2 / np.pi) * (v + 0.044715 * v ** 3)))
    _rejects(ex.f64_to_bf16(tanh), r)
    _rejects(ex.f64_to_bf16(np.where(v < 0, 0.0, gelu_emul(v))), r)
    neg = GELU_V < 0   # below zero alone too, where the intervals are wide
    rn = ex.gelu_rounded(v[neg])
    _rejects(ex.f64_to_bf16(tanh[neg]), rn)


def test_swiglu_checker_rejects_a_clamped_exponent_and_one_minus_sigmoid():
    g = np.repeat(SWIGLU_G, 2)
    u = np.tile([-3.0, 2.0], SWIGLU_G.size)
    r = sw.silu_mul_rounded(g, u)
    ex._interval_check(ex.f32_to_bf16(silu_mul_emul(g, u)), r, "h", ("element",))
    g32, u32 = g.astype(np.float32), u.astype(np.float32)
    with np.errstate(over="ignore"):
        clamped = g32 / (np.float32(1) + np.exp(np.clip(-g32, -20, 20)).astype(np.float32)) * u32
        one_minus = g32 * (np.float32(1) - sigmoid_emul(-g32)) * u32
    _rejects(ex.f32_to_bf16(clamped.astype(np.float32)), r)
    _rejects(ex.f32_to_bf16(one_minus.astype(np.float32)), r)


def _hand_routing(rows, bias, router, k, E):
    logits = np.array(rows, np.float64)
    x = np.eye(len(rows), 8)
    wg = np.zeros((E, 8))
    wg[:, : len(rows)] = logits.T
    sc = eg.scores(router, k, x, wg)
    return logits, x, wg, sc


def test_saturated_ties_go_to_the_lower_index_and_group():
    """Logits >= 18 all score 1.0: picks by bias, then the lower index; a bias of 2^-26 is absorbed; group scores 2
    tie and the lower group is kept.  The checker rejects the higher index and a bias added before saturation."""
    E, k = 16, 4
    b = et.score_bias(E)
    rows = [[30.0, 31.0, 20.0, 40.0, 25.0, 18.0, 19.0, 50.0, 22.0, 23.0, 24.0, 26.0, 27.0, 28.0, 29.0, 33.0],
            [-95.0, 18.0, 18.5, 60.0, 0.5, -90.0, 2.0, 21.0, 20.0, 19.0, -1.0, 0.0, 44.0, 45.0, 12.0, 3.0]]
    logits, x, wg, sc = _hand_routing(rows, b, V3, k, E)
    sel = eg.selection(sc, b, E)
    G = eg.group_scores(sel, V3)[2]
    picks = eg.route_mid(sel.mid, V3, k, G)
    # token 0: every score 1.0; c = fl(1 + b): group 2 (experts 4, 5; 2 + 2^-9) first, then the groups scoring
    # exactly 2 by the lower index (0, 1, 3; group 6 has 2 - 2^-9); expert 5 (b = 2^-9), then 0, 1, 2 by index (expert 3's
    # 2^-26 is absorbed)
    assert picks[0].tolist() == [5, 0, 1, 2]
    w = ex.f32_to_bf16(np.ones((2, k), np.float32))
    go = ex.f64_to_bf16(sc.s_mid)
    w_ok = ex.f32_to_bf16((0.5 * np.add(*eg.weights_bounds(sc, picks, V3))).astype(np.float32))
    assert eg.check_gated_routing(logits, b, V3, k, picks, go, w_ok, (x, wg)) == 0
    higher = picks.copy()
    higher[0, 1:] = [7, 6, 3]                             # ties broken by the higher index
    with pytest.raises(AssertionError, match="topk_idx"):
        eg.check_gated_routing(logits, b, V3, k, higher, go, w, (x, wg))
    real = 1.0 / (1.0 + np.exp(-logits)) + b              # the bias added to the unrounded score
    bad = eg.route_mid(real, V3, k)
    assert (bad != picks).any()
    with pytest.raises(AssertionError, match="topk_idx"):
        eg.check_gated_routing(logits, b, V3, k, bad, go, w, (x, wg))


def test_llama4_k1_saturated_tie_goes_to_the_lower_index():
    E = 8
    rows = [[5.0, 18.0, 40.0, -100.0, 18.0, 2.0, 60.0, 0.0]]
    logits, x, wg, sc = _hand_routing(rows, None, LLAMA4, 1, E)
    go = ex.f64_to_bf16(sc.s_mid)
    w = ex.f32_to_bf16(np.ones((1, 1), np.float32))
    assert eg.check_gated_routing(logits, None, LLAMA4, 1, np.array([[1]]), go, w, (x, wg)) == 0
    for wrong in (6, 2):   # the largest logit, or another saturated one
        with pytest.raises(AssertionError, match="topk_idx"):
            eg.check_gated_routing(logits, None, LLAMA4, 1, np.array([[wrong]]), go, w, (x, wg))


def test_exact_sums_ignore_zero_products_only():
    a = np.array([[1.0, 2.0 ** -140], [3.0, 0.0]])
    b = np.array([[2.0 ** -5, 0.0]])
    ex.assert_exact_sums(a, b, None, "zero column")          # the tiny value meets a zero weight only
    with pytest.raises(AssertionError, match="not below 2\\^24"):
        ex.assert_exact_sums(a, np.array([[2.0 ** -5, 1.0]]), None, "used column")
