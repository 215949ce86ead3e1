"""CPU checks of tests/test_gpu_shared_exact.py: the tiling arithmetic of tests/exact_shared.py is the kernel's, every
case reaches its regime on a 132-SM H100, its sums are exact in fp32 and enough of h_s and of the r + s step rounds, and
the checker catches the faults a shared expert can hide, each with a message that names the stage."""
import dataclasses
import os
import re

import numpy as np
import pytest

from tests import exact as ex
from tests import exact_gated as eg
from tests import exact_shared as es
from tests import test_gpu_exact as gx
from tests import test_gpu_shared_exact as gse

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "flashmoe_b200", "csrc")
MIN_RS_ROUNDED = 0.2   # share of out elements whose r + s needs rounding (else an order fault could not show)


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return re.sub(r"\s+", " ", f.read())


# ----------------------------------------------------------------------------- the kernel's tiling and work list
def test_tiling_and_block_placement_match_the_kernel():
    kern, host = _src("fm_kernel.cuh"), _src("flashmoe_b200.cu")
    assert f"constexpr int BLOCK_M = {es.BLOCK_M};" in kern and f"constexpr int BLOCK_N = {es.BLOCK_N};" in kern
    # a block's items: column tiles x row blocks, the shared GEMMs' row blocks being s_rb
    for line in ("L->tpc = (n + G - 1) / G;", "L->s_rb = p.shared ? (n + BLOCK_M - 1) / BLOCK_M : 0;",
                 "return g < GEMM_S_UP ? L.tcm_items : L.s_rb;",
                 "for (int g = 0; g < NUM_GEMMS; ++g) start += b.g[g] * p.gemm[g].tn * gemm_row_blocks(L, g);",
                 "const int local = id - block_start(p, L, w.blk), rbs = gemm_row_blocks(L, w.blk.gemm);",
                 "w.mb = local % rbs;", "w.nt = local / rbs;", "const int t0 = blockIdx.x * L.tpc;",
                 "const int n_tok = max(0, min(L.tpc, L.S - t0));",
                 "for (int rb = t0 / BLOCK_M + (int)threadIdx.x; rb <= (t0 + n_tok - 1) / BLOCK_M; rb += NUM_THREADS)",
                 "while (ld_acquire_gpu_u32(p.s1_done + rb) < (unsigned int)p.TN1)",
                 "int n, tn; // output columns and column tiles, ceil(n / BLOCK_N)"):
        assert line in kern, f"fm_kernel.cuh no longer has `{line}`: update exact_shared.regime"
    # the shared GEMMs' column tiles (GemmOp::tn, the eighth field): TN0s = ceil(Ps / BLOCK_N) and TN1; the shared GEMM1
    # block right after the leading local routed GEMM0 blocks (split_blk), the shared GEMM0 block first
    for line in ("const int ps = (int)Ps;",
                 "p.gemm[fm::GEMM_S_UP] = {fm::TM_XS, fm::TM_WS0, 0, 0, 0, d.H / fm::BLOCK_K, ps, "
                 "ceil_div(ps, fm::BLOCK_N),",
                 "p.gemm[fm::GEMM_S_DOWN] = {fm::TM_HS, fm::TM_WS1, 0, 0, 0, ps / fm::BLOCK_K, d.H, c->TN1,",
                 "ctx->TN1 = ceil_div(d.H, fm::BLOCK_N);",
                 "ctx->grid = d.num_sms;", 'const int lag = env_int("FM_G1_LAG", -1);',
                 "if (lag >= 1 && lag < (int)units.size()) { for (size_t i = 0; i < units.size(); ++i) { push(0, units[i]); "
                 "if ((int)i >= lag) push(1, units[i - lag]); }",
                 "for (const Unit& u : units) push(0, u); for (const Unit& u : g1_units) push(1, u);",
                 "while (split < blocks.size() && blocks[split].gemm == fm::GEMM_UP && blocks[split].pkt / nLx == rank) "
                 "++split;",
                 "blocks.insert(blocks.begin() + split, {{}, fm::GEMM_S_DOWN, rank * nLx}); "
                 "blocks.insert(blocks.begin(), {{}, fm::GEMM_S_UP, rank * nLx});"):
        assert line in host, f"flashmoe_b200.cu no longer has `{line}`: update exact_shared.regime"


def test_regime_arithmetic():
    r = es.regime(320, 320, 301, 132, 16)
    assert (r.TN0s, r.ps_tail, r.TN1, r.h_tail, r.s_rb, r.tpc, r.split_blk) == (2, 64, 2, 64, 3, 3, 16)
    assert r.rb_per_cta == 2   # the CTA at t0 = 126 holds tokens 126..128
    assert es.regime(256, 512, 512, 132, 16).rb_per_cta == 1   # tpc = 4 divides 128
    r = es.regime(320, 320, 132 * 128 + 1, 132, 16)
    assert (r.tpc, r.rb_per_cta, r.s_rb) == (129, 2, 133)
    assert es.regime(1024, 2048, 4096, 132, 16).s_rb == 32
    r = es.regime(192, 1408, 0, 132, 16)
    assert (r.TN0s, r.ps_tail, r.TN1, r.h_tail, r.s_rb, r.rb_per_cta) == (6, 128, 1, 192, 0, 0)
    assert [es.split_blk(16, lag) for lag in (-1, 0, 1, 2, 15, 16)] == [16, 16, 2, 3, 16, 16]


@pytest.mark.parametrize("name", list(gse.CASES))
def test_case_reaches_its_regime(name):
    c = gse.CASES[name]
    missing = set(c.reach) - gse.reached(c)
    assert not missing, f"{name} does not reach {sorted(missing)} on a 132-SM H100"


def test_tile_tails_are_covered():
    """Across the tile-tail cases: every TN0s of Ps in {64, 192, 320, 1408} with and without a partial last tile, and
    H with TN1 = 1 and 2, each partial, on every route and activation."""
    seen = set()
    for name, c in gse.CASES.items():
        if name.startswith("tails_"):
            for ps, n in c.launches:
                r = gse.case_regime(c, ps, n)
                seen.add((c.route, c.act, r.TN0s, r.ps_tail, r.TN1, r.h_tail))
    for route in ("router", "routed", "gated"):
        for act in (0, 1):
            for H in gse.TAIL_H:
                for ps in gse.TAIL_PS:
                    assert (route, act, -(-ps // 256), ps % 256, -(-H // 256), H % 256) in seen


# ----------------------------------------------------------------------------- preconditions and rounding shares
def _route(c):
    return dict(routing=gse.case_routing(c) if c.route == "routed" else None, router=gse.V3,
                score_bias=gse.case_score_bias(c))


def _reference(c, inp, ps, n, st=None):
    se = gse.case_shared(c, ps)
    dev, rec = ex.reference_launch(c.route, inp, c.cfg.EC_of(n), n, shared=se, stats=st, **_route(c))
    return se, dev, rec


@pytest.mark.parametrize("name", list(gse.CASES))
def test_case_is_exact_and_rounds(name):
    """For every Ps of the case, at its largest n: every reference sum is fp32-exact (the references assert it), the
    reference record passes the checker, at least 2 % of h_s rounds and at least 20 % of out rounds in the r + s step."""
    c = gse.CASES[name]
    inp = gse.case_inputs(c)
    for ps in sorted({ps for ps, _ in c.launches}):
        n = max(n for p, n in gse.launch_ns(c, 132) if p == ps)
        st = ex.Stats()
        se, dev, rec = _reference(c, inp, ps, n, st)
        ex.check_launch(c.route, inp, c.cfg.EC_of(n), n, dev, rec, shared=se, **_route(c))
        h, o = st.d["h_s"], st.d["out = rne(r + s)"]
        assert h[1] >= gx.MIN_H_ROUNDED * h[0], f"Ps={ps}: only {h[1]} of {h[0]} h_s elements round"
        assert o[1] >= MIN_RS_ROUNDED * o[0], f"Ps={ps}: only {o[1]} of {o[0]} out elements round in r + s"


@pytest.mark.parametrize("name", list(gse.LAYERS))
def test_model_shape_shared_sums_exact(name):
    """The model-shape shared experts: GEMM0 and GEMM1 sums exact in fp32 on 128 tokens drawn as the layer's (the
    bound is per row; the GPU test checks every row), and h_s on the 2^-3 grid with most of it nonzero."""
    cfg, _, ps = gse.LAYERS[name]
    li_x = eg.layer_inputs(cfg.replace(sequence_len=128), seed=8100 + len(name)).x64
    rec = ex.shared_stage(li_x, gse.layer_shared(name))
    h = ex.bits_to_f64(rec.h_s)
    assert (h != 0).mean() > 0.3 and ex.grid_log2(h) == ex.WUP_GRID


# ----------------------------------------------------------------------------- planted faults
S = 512


def _base(route="routed", k=2, H=320, ps=320, n=S, act=0):
    c = gse.Case(route, gse._cfg(k=k, H=H, hidden_act=act), ((ps, n),))
    inp = gse.case_inputs(c)
    se, dev, rec = _reference(c, inp, ps, n)

    def check(d=dev, r=rec):
        ex.check_launch(route, inp, c.cfg.EC_of(n), n, d, r, shared=se, **_route(c))

    check()   # the reference record itself passes
    return c, inp, se, dev, rec, check


def _routed_r(inp, c, n):
    """The routed result r (bf16 bits) of the routed base case, and its per-pick terms (kept, terms [n, k, H])."""
    dev, _ = ex.reference_launch("routed", inp, c.cfg.EC_of(n), n, routing=gse.case_routing(c))
    kept = dev.slot < c.cfg.EC_of(n)
    y_of = dev.ret_y[np.where(kept, dev.topk_idx, 0), np.where(kept, dev.slot, 0)]
    terms = ex.bits_to_f64(ex.f64_to_bf16(ex.bits_to_f64(dev.topk_w)[:, :, None] * ex.bits_to_f64(y_of)))
    return dev.out, kept, terms


def _accumulate(kept, terms, s, at):
    """The bf16 accumulation of the kept terms in pick order from +0, with s added as an extra term before pick `at`."""
    acc = np.zeros(terms.shape[::2])
    for j in range(terms.shape[1]):
        if j == at:
            acc = ex.bits_to_f64(ex.f64_to_bf16(acc + s))
        acc = np.where(kept[:, j][:, None], ex.bits_to_f64(ex.f64_to_bf16(acc + terms[:, j])), acc)
    return ex.f64_to_bf16(acc)


@pytest.mark.parametrize("k,at", [(2, 0), (4, 0), (4, 2)])
def test_fault_s_inside_the_combine(k, at):
    """s added as the first combine term (at = 0) or between the terms, instead of after r is rounded."""
    c, inp, se, dev, rec, check = _base(k=k)
    r, kept, terms = _routed_r(inp, c, S)
    dev.out = _accumulate(kept, terms, ex.bits_to_f64(rec.y_s), at)
    with pytest.raises(AssertionError, match=r"^out = rne\(r \+ s\): \d+ of \d+ elements outside the reference; first at token"):
        check()


def test_fault_s_missing_on_the_last_partial_row_block():
    c, inp, se, dev, rec, check = _base(n=301)
    r, _, _ = _routed_r(inp, c, 301)
    dev.out[256:] = r[256:]
    with pytest.raises(AssertionError, match=r"^out = rne\(r \+ s\): \d+ of \d+ elements outside the reference; first at token 2(5[6-9]|[6-9]\d)"):
        check()


def test_fault_y_s_rows_of_the_previous_row_block():
    c, inp, se, dev, rec, check = _base()
    rec.y_s[256:384] = rec.y_s[128:256]
    dev.out[256:384] = ex.add_shared(ex.Rounded(*(_routed_r(inp, c, S)[0][256:384],) * 2, 0), rec.y_s[256:384]).lo
    with pytest.raises(AssertionError, match=r"^y_s \(shared expert\): \d+ of \d+ differ; first at token 256"):
        check()


@pytest.mark.parametrize("which", ["dropped", "routed_expert_0"])
def test_fault_shared_bias_down(which):
    c, inp, se, dev, rec, check = _base()
    w_down, bd_s = se.down(0)
    bd = None if which == "dropped" else inp.experts.down(0)[1]
    assert bd_s is not None and (bd is None or not np.array_equal(bd, bd_s))
    rec.y_s = ex.gemm1_reference(rec.h_s, w_down, bd, "GEMM1").lo
    with pytest.raises(AssertionError, match=r"^y_s \(shared expert\)"):
        check()


def test_fault_partial_ps_tile_of_h_s_from_the_previous_launch():
    """Columns 256..319 of h_s (the last, partial Ps tile at Ps = 320) left from a launch on other tokens; y_s and out
    follow the stale h_s, as a kernel that skipped the tile would produce them."""
    c, inp, se, dev, rec, check = _base()
    stale = ex.shared_stage(inp.x64[::-1][:S], se)
    rec.h_s[:, 256:] = stale.h_s[:, 256:]
    rec.y_s = se.y(0, rec.h_s).lo
    with pytest.raises(AssertionError, match=r"^h_s \(shared expert\): \d+ of \d+ elements outside the reference; first at token \d+, column (2[5-9]\d|3[01]\d)"):
        check()


def test_fault_partial_h_tile_of_y_s_from_the_previous_launch():
    c, inp, se, dev, rec, check = _base()
    stale = ex.shared_stage(inp.x64[::-1][:S], se)
    rec.y_s[:, 256:] = stale.y_s[:, 256:]
    with pytest.raises(AssertionError, match=r"^y_s \(shared expert\): \d+ of \d+ differ; first at token \d+, column (2[5-9]\d|3[01]\d)"):
        check()


def test_fault_gelu_replaced_by_relu_in_h_s():
    c, inp, se, dev, rec, check = _base(route="router", act=1)
    relu = ex.shared_stage(inp.x64[:S], dataclasses.replace(se, act=0))
    rec.h_s, rec.y_s = relu.h_s, relu.y_s
    with pytest.raises(AssertionError, match=r"^h_s \(shared expert\): \d+ of \d+ elements outside the reference"):
        check()


@pytest.mark.parametrize("route", ["router", "routed", "gated"])
def test_fault_s_added_twice(route):
    c, inp, se, dev, rec, check = _base(route=route)
    dev.out = ex.add_shared(ex.Rounded(dev.out, dev.out, 0), rec.y_s).lo
    with pytest.raises(AssertionError, match=r"^out = rne\(r \+ s\)"):
        check()


def test_fault_all_dropped_rows_without_s():
    """Rows whose picks were all skipped or dropped must be rne(+0 + s), not +0."""
    c, inp, se, dev, rec, check = _base(k=1)
    none = ~(dev.slot < c.cfg.EC).any(1)
    assert none.sum() >= 8
    dev.out[none] = 0
    with pytest.raises(AssertionError, match=r"^out = rne\(r \+ s\)"):
        check()
