"""CPU checks of tests/test_gpu_subchunks.py: the sub-chunk arithmetic of tests/exact_gated.py is the kernel's, every
case reaches its regime on a 132-SM H100, is exact and rounds, its inputs make the bias and the group limit change the
picks in every sub-chunk position, and the checkers catch the faults that regime can hide."""
import os
import re

import numpy as np
import pytest

from flashmoe_b200.router import RouterSpec
from tests import exact as ex
from tests import exact_gated as eg
from tests import test_gpu_exact as gx
from tests import test_gpu_subchunks as gs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "flashmoe_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _constexpr(src, name):
    m = re.search(rf"constexpr int {name} = ([0-9 *]+);", src)
    assert m, f"constexpr {name} not found"
    return int(np.prod([int(v) for v in m.group(1).split("*")]))


# ----------------------------------------------------------------------------- the kernel's sizing
def test_subchunk_arithmetic_matches_the_kernel():
    src = _src("fm_kernel.cuh")
    assert _constexpr(src, "G_LOGIT_BYTES") == eg.G_LOGIT_BYTES
    assert _constexpr(src, "G_SEL_MAX") == eg.G_SEL_MAX
    assert _constexpr(src, "BLOCK_M") == eg.TC_ROWS
    gate = re.search(r"void gate_phase\(.*?\n}\n", src, re.S)
    assert gate, "gate_phase not found"
    body = re.sub(r"\s+", " ", gate.group(0))
    for line in ("const int ldl = E + 1;", "int TS = G_LOGIT_BYTES / (ldl * 4);", "if (tc) TS = min(TS, BLOCK_M);",
                 "else if (TS > n_tok) TS = n_tok;", "for (int s0 = 0; s0 < n_tok; s0 += TS)",
                 "const int n_sub = min(TS, n_tok - s0);"):
        assert line in body, f"gate_phase no longer has `{line}`: update exact_gated.regime"
    lanes = re.search(r"int softmax_topk_lanes\(int E\) \{(.*?)\n}", src, re.S)
    assert lanes, "softmax_topk_lanes not found"
    m = re.search(r"if \(E > 8\) return E <= (\d+) \? (\d+) : E <= (\d+) \? (\d+) : E <= (\d+) \? (\d+) : (\d+);",
                  lanes.group(1))
    assert m and "while (lpt < E) lpt <<= 1;" in lanes.group(1), "softmax_topk_lanes changed its form"
    t = [int(v) for v in m.groups()]

    def kernel_lanes(E):
        if E > 8:
            return t[1] if E <= t[0] else t[3] if E <= t[2] else t[5] if E <= t[4] else t[6]
        return 1 << (E - 1).bit_length()

    for E in range(1, 1025):
        assert eg.softmax_topk_lanes(E) == kernel_lanes(E) == gx._lpt(E), E
    host = _src("flashmoe_b200.cu")
    assert 'ctx->tc_gate = !ctx->dense && d.E <= 256 && env_int("FM_TC_GATE", d.E > 16 ? 1 : 0) != 0;' in host
    assert "ctx->tpc = ceil_div(d.S, ctx->grid);" in host and "(long long)ctx->tpc * d.k > fm::G_SEL_MAX" in host
    assert [E for E in range(1, 1025) if eg.tc_router(E, {})] == list(range(17, 257))
    assert eg.tc_router(16, {"FM_TC_GATE": "1"}) and not eg.tc_router(64, {"FM_TC_GATE": "0"})
    assert not eg.tc_router(257, {"FM_TC_GATE": "1"})


def test_regime_arithmetic():
    r = eg.regime(16, 2, 131072, 132, False)
    assert (r.tpc, r.TS, r.sub_chunks) == (993, 963, [963, 30])
    r = eg.regime(256, 8, 135168, 132, True)
    assert (r.tpc, r.TS, r.sel_entries, r.s_max, len(r.sub_chunks)) == (1024, 63, 8192, 135168, 17)
    assert r.sub_chunks[-1] == 1024 - 16 * 63
    r = eg.regime(1024, 2, 4096, 132, False)
    assert (r.tpc, r.TS, r.sub_chunks) == (32, 15, [15, 15, 2])
    assert eg.regime(128, 2, 0, 132, True).sub_chunks == []
    assert eg.regime(1024, 2, 1, 132, False).sub_chunks == [1]
    for k in (1, 2, 8):
        s = eg.regime(8, k, 0, 132, False).s_max
        assert s % 128 == 0 and -(-s // 132) * k <= 8192 < -(-(s + 128) // 132) * k


@pytest.mark.parametrize("name", list(gs.CASES))
def test_case_reaches_its_regime(name):
    c = gs.CASES[name]
    rg = gs.case_regime(c, c.cfg.S, env={})
    if c.kind != "routed":
        assert len(rg.sub_chunks) == c.min_sub
    assert (rg.sel_entries == eg.G_SEL_MAX) == c.full_scratch
    ns = gs.token_counts(c, env={})
    assert ns[0] == c.cfg.S and ns[-1] == 1
    if len(ns) == 3:   # every full CTA's second sub-chunk holds one token
        assert gs.case_regime(c, ns[1], env={}).sub_chunks == [rg.TS, 1]


# ----------------------------------------------------------------------------- preconditions and rounding shares
def _shares(st, k):
    hs, os_ = st.d["hidden"], st.d["out"]
    assert hs[1] >= gx.MIN_H_ROUNDED * hs[0], f"only {hs[1]} of {hs[0]} h elements needed rounding"
    if k > 1:
        assert os_[1] >= gx.MIN_OUT_ROUNDED * os_[0], f"only {os_[1]} of {os_[0]} out elements needed rounding"


@pytest.mark.parametrize("name", list(gs.CASES))
def test_case_is_exact_and_rounds(name):
    """assert_exact_sums holds (every reference stage asserts it) and the h / out rounding shares reach
    test_gpu_exact's minimums; the reference device record passes its own checks."""
    c = gs.CASES[name]
    cfg = c.cfg
    inp = gs.case_inputs(c)
    for n in gs.token_counts(c, env={}):
        EC = cfg.EC_of(n)
        if c.kind == "router":
            ex.check_preconditions(inp, EC, gx.MIN_H_ROUNDED if n > 30 else 0, gx.MIN_OUT_ROUNDED, n=n)
            continue
        st = ex.Stats()
        route = dict(routing=gs.case_routing(c) if c.kind == "routed" else None, router=c.router,
                     score_bias=gs.case_bias(c))
        dev, _ = ex.reference_launch(c.kind, inp, EC, n, stats=st, **route)
        if not c.layer:   # (the layer-sized reference is minutes of float64 GEMMs: built once, not re-checked)
            assert ex.check_launch(c.kind, inp, EC, n, dev, **route) <= gs.max_ambiguous(c, n)
        if n > 30:
            _shares(st, cfg.k)


# ----------------------------------------------------------------------------- influence of the bias and the groups
GATED = [n for n, c in gs.CASES.items() if c.kind == "gated"]


def _midpoint_picks(c, inp, router, bias):
    sc = eg.scores(router, c.cfg.k, inp.x64, inp.wg_eff64)
    b = 0.0 if bias is None else bias.astype(np.float64)[None, :]
    return eg.route_mid(sc.s_mid + b, router, c.cfg.k)


def _ungrouped(router):
    return RouterSpec(router.scoring, renormalize=router.renormalize, scale=router.scale)


@pytest.mark.parametrize("name", [n for n in GATED if gs.CASES[n].bias_log2 is not None or gs.CASES[n].router.n_group > 1])
def test_bias_and_groups_change_picks_in_every_subchunk_position(name):
    """In every sub-chunk position of a CTA (not only the first), at least 20 % of the tokens have different picks
    without the bias (rules with a bias), and at least 20 % have a member of their unconstrained top-k outside the kept
    groups (rules with groups)."""
    c = gs.CASES[name]
    inp = gs.case_inputs(c)
    bias = gs.case_bias(c)
    pos = gs.case_regime(c, c.cfg.S, env={}).position(c.cfg.S)
    picks = _midpoint_picks(c, inp, c.router, bias)
    shares = {}
    if bias is not None:
        shares["bias"] = (picks != _midpoint_picks(c, inp, c.router, None)).any(1)
    if c.router.n_group > 1:
        free = np.sort(_midpoint_picks(c, inp, _ungrouped(c.router), bias), 1)
        shares["groups"] = (free != np.sort(picks, 1)).any(1)
    for what, changed in shares.items():
        for p in range(pos.max() + 1):
            share = changed[pos == p].mean()
            assert share >= 0.2, f"{what}: only {share:.1%} of the tokens in sub-chunk position {p} change their picks"
    print(f"\n[{name}] " + "; ".join(f"{w}: {[round(float(ch[pos == p].mean()), 3) for p in range(pos.max() + 1)]}"
                                     for w, ch in shares.items()))


# ----------------------------------------------------------------------------- planted faults
def _gated_base(name):
    c = gs.CASES[name]
    inp = gs.case_inputs(c)
    bias = gs.case_bias(c)
    rg = gs.case_regime(c, c.cfg.S, env={})
    return c, inp, bias, rg, ex.reference_launch("gated", inp, c.cfg.EC, c.cfg.S, router=c.router, score_bias=bias)[0]


def _check_gated(c, inp, dev, bias):
    ex.check_launch("gated", inp, c.cfg.EC, c.cfg.S, dev, router=c.router, score_bias=bias)


def _reroute(c, inp, dev, rows, router, bias):
    """The device record with tokens `rows` routed by `router` / `bias` instead (picks and their midpoint weights)."""
    sc = eg.scores(c.router, c.cfg.k, inp.x64[rows], inp.wg_eff64)
    b = np.zeros(c.cfg.E) if bias is None else bias.astype(np.float64)
    picks = eg.route_mid(sc.s_mid + b, router, c.cfg.k)
    lo, hi = eg.weights_bounds(sc, picks, c.router)
    dev.topk_idx[rows] = picks
    dev.topk_w[rows] = ex.f32_to_bf16((0.5 * (lo + hi)).astype(np.float32))


def test_fault_bias_missing_after_the_first_subchunk():
    c, inp, bias, rg, dev = _gated_base("gated_dsv3")
    later = np.flatnonzero(rg.position(c.cfg.S) > 0)
    _reroute(c, inp, dev, later, c.router, None)
    with pytest.raises(AssertionError, match=r"topk_idx \(gated\): \d+ decided tokens differ; first token (\d+)") as ei:
        _check_gated(c, inp, dev, bias)
    assert int(re.search(r"first token (\d+)", str(ei.value)).group(1)) in set(later)


def test_fault_group_limit_ignored_after_the_first_subchunk():
    c, inp, bias, rg, dev = _gated_base("gated_dsv3")
    later = np.flatnonzero(rg.position(c.cfg.S) > 0)
    _reroute(c, inp, dev, later, _ungrouped(c.router), bias)
    with pytest.raises(AssertionError, match=r"topk_idx \(gated\)"):
        _check_gated(c, inp, dev, bias)


def _second_subchunk_over_first(topk, rg, n):
    """The routing slot_ranks would see if every CTA wrote its second sub-chunk's picks over the first's."""
    seen = topk.copy()
    for t0 in range(0, n, rg.tpc):
        n2 = min(rg.TS, n - t0 - rg.TS)
        if n2 > 0:
            seen[t0:t0 + n2] = topk[t0 + rg.TS:t0 + rg.TS + n2]
    return seen


@pytest.mark.parametrize("name", ["router_E384_k8", "gated_kimi_k2"])
def test_fault_second_subchunk_sel_e_over_the_first(name):
    c = gs.CASES[name]
    cfg = c.cfg
    inp = gs.case_inputs(c)
    rg = gs.case_regime(c, cfg.S, env={})
    bias = gs.case_bias(c)
    dev, _ = ex.reference_launch(c.kind, inp, cfg.EC, cfg.S, router=c.router, score_bias=bias)
    seen = _second_subchunk_over_first(dev.topk_idx, rg, cfg.S)
    assert not np.array_equal(seen, dev.topk_idx)
    dev.slot, dev.counts, dev.recv_cnt, _ = ex.slots_from_topk(seen, cfg.E, cfg.EC)
    with pytest.raises(AssertionError, match=r"^slot: \d+ of \d+ differ; first at token"):
        ex.check_launch(c.kind, inp, cfg.EC, cfg.S, dev, router=c.router, score_bias=bias)


def test_fault_weight_renormalised_by_the_previous_tokens_sum():
    c, inp, bias, rg, dev = _gated_base("gated_kimi_k2")
    assert c.router.renormalize
    sc = eg.scores(c.router, c.cfg.k, inp.x64, inp.wg_eff64)
    W = sc.s_mid[np.arange(c.cfg.S)[:, None], dev.topk_idx].sum(1)
    # the first token of a CTA's second sub-chunk whose previous token's sum differs by more than 1 %
    t = next(t for t in range(rg.TS, c.cfg.S, rg.tpc) if abs(W[t - 1] / W[t] - 1) > 0.01)
    W_prev, picks = W[t - 1], dev.topk_idx[t - 1:t + 1]
    dev.topk_w[t, 0] = ex.f64_to_bf16(np.array([sc.s_mid[t, picks[1, 0]] / W_prev * c.router.scale]))[0]
    with pytest.raises(AssertionError, match=rf"topk_w \(gated\): 1 tokens .*; first token {t} pick 0 "):
        _check_gated(c, inp, dev, bias)


def _aux_from(p, counts, n, rows):
    """gML / gMeC / loss from probabilities p [n, E] summed over the tokens `rows` only."""
    E = counts.shape[0]
    gml = (p[rows].sum(0) / n).astype(np.float32)
    gmec = (counts / n).astype(np.float32)
    loss = np.float32((gml.astype(np.float64) * gmec / E).sum())
    return np.concatenate([gml, gmec, [loss]]).astype(np.float32)


@pytest.mark.parametrize("name", ["training_E1024_k2", "training_E128_k2"])
def test_fault_last_subchunk_column_sums_dropped_from_gml(name):
    c = gs.CASES[name]
    cfg = c.cfg
    inp = gs.case_inputs(c)
    n = cfg.S
    rg = gs.case_regime(c, n, env={})
    ref = ex.router_reference(inp.x64, inp.wg_eff64, cfg.k)
    _, counts, _, _ = ex.slots_from_topk(ref.topk, cfg.E, cfg.EC)
    p = 0.5 * (ref.p_lo + ref.p_hi)
    eg.check_aux(_aux_from(p, counts, n, np.arange(n)), ref, counts, n, rg)
    pos = rg.position(n)
    lost = _aux_from(p, counts, n, np.flatnonzero(pos != pos.max()))
    with pytest.raises(AssertionError, match=r"^gML: \d+ of \d+ experts outside the interval"):
        eg.check_aux(lost, ref, counts, n, rg)
