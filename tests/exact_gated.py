"""The exact-input reference (tests/exact.py) for gated forwards (fm_moe_forward_gated), and the router's sub-chunk
arithmetic.

A CTA's ceil(n / grid) tokens go through the router in sub-chunks of TS tokens, as many as fit one padded fp32 logits
row each in the logits scratch (gate_phase in fm_kernel.cuh); the tensor-core router caps TS at one 128-row tile.
`regime` states that arithmetic, and tests/test_subchunk_cases.py pins its constants to the kernel's source.

`check_gated_routing` checks a gated launch's gate_out, picks and weights against intervals: the scores are those of the
softmax reference (exact.router_reference) or of the kernel's sigmoid, the selection value adds the fp32 score bias, the
kept groups and the picks are decided from the intervals, and a token whose picks the intervals cannot decide is counted
as ambiguous instead of checked.  The rest of a gated launch is a routed launch on its own routing (exact.check_launch).
No pytest in here.
"""
from __future__ import annotations

import dataclasses
import os
from typing import List

import numpy as np
import torch

from tests import exact as ex

# ----------------------------------------------------------------------------- sub-chunk arithmetic (fm_kernel.cuh)
G_LOGIT_BYTES = 64 * 1024   # the logits scratch
G_SEL_MAX = 8192            # tokens per CTA * k: sel_e / rank scratch, the largest the host accepts
TC_ROWS = 128               # BLOCK_M: the tensor-core router's sub-chunk cap (two wgmma warpgroups of 64 rows)
H100_SMS = 132              # the grid of an H100 SXM (one CTA per SM); GPU tests use the context's own grid


def softmax_topk_lanes(E: int) -> int:
    """Lanes per token of the router's softmax / top-k (fm_kernel.cuh softmax_topk_lanes)."""
    if E > 8:
        return 4 if E <= 128 else 8 if E <= 256 else 16 if E <= 512 else 32
    p = 1
    while p < E:
        p <<= 1
    return p


def tc_router(E: int, env=None) -> bool:
    """The router path fm_create picks: tensor cores for 17 <= E <= 256 unless FM_TC_GATE says otherwise (E = 1
    takes the dense path and no router)."""
    v = (os.environ if env is None else env).get("FM_TC_GATE", "")
    want = int(v) != 0 if v else E > 16
    return E != 1 and E <= 256 and want


@dataclasses.dataclass(frozen=True)
class Regime:
    grid: int
    tpc: int                 # tokens per CTA, ceil(n / grid)
    TS: int                  # tokens per sub-chunk
    sub_chunks: List[int]    # sub-chunk sizes of the fullest CTA
    sel_entries: int         # tpc * k: entries of the sel_e / rank scratch
    s_max: int               # the largest S, a multiple of 128, with ceil(S / grid) * k <= G_SEL_MAX

    def position(self, n: int) -> np.ndarray:
        """Sub-chunk index of each of the first n tokens inside its CTA."""
        return (np.arange(n) % self.tpc) // self.TS if self.tpc else np.zeros(0, np.int64)


def regime(E: int, k: int, n: int, grid: int, tc: bool) -> Regime:
    tpc = -(-n // grid)
    ts = G_LOGIT_BYTES // (4 * (E + 1))
    if tc:
        ts = min(ts, TC_ROWS)
    elif tpc:
        ts = min(ts, tpc)   # (the GEMV path trims TS to the CTA's tokens; the sizes are the same)
    subs = [min(ts, tpc - s0) for s0 in range(0, tpc, ts)]
    s_max = (grid * (G_SEL_MAX // k)) // 128 * 128
    return Regime(grid, tpc, ts, subs, tpc * k, s_max)


# ----------------------------------------------------------------------------- inputs at a model's layer size
def layer_inputs(cfg, seed: int, *, x_range: int = 4, wg_density: float = 1 / 16, up_range: int = 2,
                 down_range: int = 2) -> ex.ExactInputs:
    """Exact inputs at a model's layer size (e.g. DeepSeek-V3: H = 7168, P = 2048, E = 256): the expert weights are
    drawn one block at a time from a seed per (expert, block) (exact.PerExpert), so neither the reference nor the upload
    holds all E experts at once (60 GB in float64 at DeepSeek-V3's size).  x: integers in [-x_range, x_range]; Wg_eff:
    sparse (density `wg_density`) entries +-2^-6, so the logits of H-term sums stay near unit scale; W_up: integers in
    [-up_range, up_range] * 2^-3; W_down: integers in [-down_range, down_range] * 2^-5.  No biases."""
    S, H, E, P = cfg.S, cfg.H, cfg.E, cfg.P
    g = np.random.default_rng(seed)
    x = g.integers(-x_range, x_range + 1, size=(S, H), dtype=np.int8)
    wg = (g.integers(0, 2, size=(E, H), dtype=np.int8) * 2 - 1) * (g.random((E, H)) < wg_density)

    def block(e, i):   # W_up [P, H] (block 0), or W_down_eff [H, P] viewed flat as [P, H] (block 1)
        r, grid = (up_range, ex.WUP_GRID) if i == 0 else (down_range, ex.WDOWN_GRID)
        ints = np.random.default_rng((seed, e, i)).integers(-r, r + 1, size=(P, H) if i == 0 else (H, P), dtype=np.int8)
        return (torch.from_numpy(ints).bfloat16() * 2.0 ** grid).reshape(P, H)

    none = np.zeros(0, np.int64)
    return ex.ExactInputs(cfg, torch.from_numpy(x).bfloat16().reshape(cfg.mini_batch, cfg.sequence_len, H),
                          (torch.from_numpy(wg.astype(np.float32)) * 2.0 ** ex.WG_GRID).bfloat16().reshape(-1).reshape(H, E),
                          ex.Experts(ex.PerExpert(block, (E, 2, P, H)), None, None, cfg.hidden_act), none, none)


# ----------------------------------------------------------------------------- gated routing reference
SAT_A = -25.0   # power arguments at or below this give a score of exactly 1.0


def sigmoid_bounds(logits):
    """Interval (lo, hi, mid) of the kernel's sigmoid_score(l) = rcp_rn(fl(1 + ex2.approx.ftz(a))), a = fl(-l log2e),
    for exact fp32 logits; lo == hi where the device value is known exactly.
      a <= SAT_A (l >= 17.33; on the 2^-6 logit grid l >= 17.34): the power is at most 2^-25 (1 + 2^-21) < 2^-24, half
        an ulp of 1, so 1 + p rounds to 1 and the score is exactly 1.0 -- every such expert ties;
      a > exact.NORMAL_A (l below about -86.6): the kernel's steps from ex2's ends (exact.sigmoid_f32_ends): a
        subnormal score for a in (126, 128), exactly +0 once the power overflows (a >= 128, l <= -88.73);
      elsewhere relative 2^-21 + 2^-24 (1.25 |l| + 3) (flashmoe_b200.h): ex2's 2^-21, the rounded argument (|l| 2^-24),
        fl32(log2 e)'s own error (under 2^-26, so |l| 2^-26), the sum and the reciprocal, and one 2^-24 for the
        second-order terms.  (Without the constant's error the bound is exceeded near |l| = 50 when ex2 errs by its
        full 2^-21; tests/test_exact_tails.py emulates that.)"""
    logits = np.asarray(logits, dtype=np.float64)
    with np.errstate(over="ignore"):
        s = 1.0 / (1.0 + np.exp(-logits))
    eps = 2.0 ** -21 + 2.0 ** -24 * (1.25 * np.abs(logits) + 3)
    lo, hi, mid = s * (1 - eps), s * (1 + eps), s.copy()
    a = (-logits * float(ex.LOG2E_F32)).astype(np.float32).astype(np.float64)
    sat = a <= SAT_A
    lo[sat] = hi[sat] = mid[sat] = 1.0
    tail = a > ex.NORMAL_A
    if tail.any():
        t_lo, t_hi = ex.sigmoid_f32_ends(a[tail])
        lo[tail], hi[tail] = t_lo, t_hi
        mid[tail] = np.where(t_lo == t_hi, t_lo, s[tail])
    return lo, hi, mid


@dataclasses.dataclass
class Scores:
    s_lo: np.ndarray       # [n, E] bounds of the device's fp32 score
    s_hi: np.ndarray
    s_mid: np.ndarray
    go_lo: np.ndarray      # bf16 bits [n, E] bounds of gate_out
    go_hi: np.ndarray


def scores(router, k, x, wg_eff) -> Scores:
    if router.scoring == "softmax":
        ref = ex.router_reference(x, wg_eff, k)
        return Scores(ref.p_lo, ref.p_hi, 0.5 * (ref.p_lo + ref.p_hi), ref.go_lo, ref.go_hi)
    ex.assert_exact_sums(x, wg_eff, None, "router logits")
    lo, hi, mid = sigmoid_bounds(x @ wg_eff.T)
    return Scores(lo, hi, mid, ex.f64_to_bf16(lo), ex.f64_to_bf16(hi))


def _group_scores(c, router, f32=False):
    """[n, n_group] group scores of the selection values c [n, E]: the largest, or the sum of the two largest (rounded
    to fp32 as the kernel does with `f32`, for exact c)."""
    n, E = c.shape
    g = -np.sort(-c.reshape(n, router.n_group, E // router.n_group), axis=2)
    if router.group_top == 1:
        return g[:, :, 0]
    s = g[:, :, 0] + g[:, :, 1]
    return s.astype(np.float32).astype(np.float64) if f32 else s


@dataclasses.dataclass
class Selection:
    """The selection values c = fl(s + b) [n, E] as intervals, and where they are known exactly (an exact score:
    saturated at 1.0, +0, or a flushed softmax probability; fl(s + b) of exact fp32 operands is then exact too)."""
    lo: np.ndarray
    hi: np.ndarray
    mid: np.ndarray
    exact: np.ndarray


def selection(sc: "Scores", bias, E: int) -> Selection:
    bv = np.zeros(E) if bias is None else np.asarray(bias, dtype=np.float64)
    m = 2.0 ** -23 * (np.abs(sc.s_hi) + np.abs(bv)) + 1e-300        # the fp32 rounding of s + b
    exact = sc.s_lo == sc.s_hi
    c_ex = (sc.s_lo.astype(np.float32) + bv.astype(np.float32)).astype(np.float32).astype(np.float64)
    lo = ex.f32_up(np.where(exact, c_ex, sc.s_lo + bv - m)).astype(np.float64)   # (the device's c is an fp32 number)
    hi = ex.f32_down(np.where(exact, c_ex, sc.s_hi + bv + m)).astype(np.float64)
    return Selection(lo, hi, np.where(exact, c_ex, sc.s_mid + bv), exact)


def group_scores(sel: Selection, router):
    """(G_lo, G_hi, G_mid, exact) [n, n_group]: bounds of the device's group scores and where they are one value.  The
    largest c, or the sum of the two largest, is increasing in every c, and the kernel's fp32 sum rounds monotonically,
    so the kernel's sum of the bounds' two largest bounds it (a float64 sum of two fp32 numbers rounds to fp32 as
    their exact sum does); equal bounds give the device's value exactly (fl(1 + 1) = 2, or fl(1 + 2^-93) = 1)."""
    G_lo, G_hi = _group_scores(sel.lo, router, f32=True), _group_scores(sel.hi, router, f32=True)
    ex_g = G_lo == G_hi
    return G_lo, G_hi, np.where(ex_g, G_lo, _group_scores(sel.mid, router)), ex_g


def kept_groups(c, router, G=None):
    """bool [n, n_group]: the topk_group groups of the largest group score (of c, or the scores G), the lower group
    on equal scores."""
    G = _group_scores(np.atleast_2d(c), router) if G is None else G
    rows = np.arange(G.shape[0])
    kept = np.zeros(G.shape, bool)
    for _ in range(router.topk_group):
        kept[rows, np.argmax(np.where(kept, -np.inf, G), axis=1)] = True
    return kept


def route_mid(c, router, k, G=None):
    """The reference's picks [n, k] on the selection values c [n, E] (interval midpoints): larger c first, the lower
    index on equal values, only experts of the kept groups (of the group scores G when given)."""
    c = np.atleast_2d(c)
    if router.n_group > 1:
        allowed = np.repeat(kept_groups(c, router, G), c.shape[1] // router.n_group, axis=1)
        c = np.where(allowed, c, -np.inf)
    return np.argsort(-c, axis=1, kind="stable")[:, :k].astype(np.int32)


def weights_bounds(sc: Scores, picks, router):
    """Bounds [n, k] of the device's fp32 weight before its bf16 rounding."""
    rows = np.arange(picks.shape[0])[:, None]
    k = picks.shape[1]
    w_lo, w_hi = sc.s_lo[rows, picks], sc.s_hi[rows, picks]
    if router.renormalize:
        W_lo = w_lo.sum(1, keepdims=True) * (1 - k * 2.0 ** -24)
        W_hi = w_hi.sum(1, keepdims=True) * (1 + k * 2.0 ** -24)
        w_lo, w_hi = w_lo / W_hi, w_hi / W_lo
    return w_lo * router.scale * (1 - 3 * 2.0 ** -24), w_hi * router.scale * (1 + 3 * 2.0 ** -24)


def check_gated_routing(logits, bias, router, k, dev_idx, dev_go, dev_w, wg_x):
    """`logits` [n, E] are the exact logits x . Wg_eff^T of wg_x = (x, Wg_eff); they serve only to recognise exact ties
    (equal logits and equal bias give identical device values), the score intervals come from wg_x.  Selection values
    known exactly (a saturated 1.0 or +0 score plus the bias, rounded as the kernel rounds fl(s + b)) that are equal
    are identical device values too, and so are equal exact group scores: the kernel's strict '>' then decides by the
    lower index or the lower group, and such a token is decided, not ambiguous.
    gate_out inside its interval; every decided token's picks equal the reference's and its weights lie inside
    their interval; returns the number of ambiguous tokens.  A failure names the stage (gate_out, topk_idx or topk_w),
    the first failing token and pick, and the experts involved."""
    n, E = logits.shape
    if n == 0:
        return 0
    sc = scores(router, k, *wg_x)
    g = ex.order_key(dev_go)
    ok = (g >= ex.order_key(sc.go_lo)) & (g <= ex.order_key(sc.go_hi))
    if not ok.all():
        t, e = (int(v) for v in np.argwhere(~ok)[0])
        raise AssertionError(f"gate_out (gated): {int((~ok).sum())} elements outside their interval; first at token "
                             f"{t}, expert {e}: device {ex._fmt(dev_go[t, e])}, reference "
                             f"[{ex._fmt(sc.go_lo[t, e])}, {ex._fmt(sc.go_hi[t, e])}]")
    bv = np.zeros(E) if bias is None else np.asarray(bias, dtype=np.float64)
    sel = selection(sc, bias, E)
    c_lo, c_hi, c_mid = sel.lo, sel.hi, sel.mid
    G = group_scores(sel, router) if router.n_group > 1 else None
    picks = route_mid(c_mid, router, k, None if G is None else G[2])
    rows = np.arange(n)
    decided = np.ones(n, bool)
    allowed = np.ones((n, E), bool)
    if router.n_group > 1:   # the kept groups must be certain: every kept group's score above every other group's, or
        G_lo, G_hi, G_mid, G_ex = G   # identical to it (known exactly, or of the same inputs) and the lower group
        kept = kept_groups(c_mid, router, G_mid)
        gi = np.arange(router.n_group)
        GS = E // router.n_group   # groups whose (logit, bias) pairs are the same multiset have identical scores
        order = np.lexsort((np.broadcast_to(bv.reshape(router.n_group, GS), (n, router.n_group, GS)),
                            logits.reshape(n, router.n_group, GS)), axis=-1)
        Ls = np.take_along_axis(logits.reshape(n, router.n_group, GS), order, -1)
        Bs = np.take_along_axis(np.broadcast_to(bv.reshape(router.n_group, GS), Ls.shape), order, -1)
        same = ((Ls[:, :, None] == Ls[:, None, :]) & (Bs[:, :, None] == Bs[:, None, :])).all(-1)
        same |= G_ex[:, :, None] & G_ex[:, None, :] & (G_mid[:, :, None] == G_mid[:, None, :])
        tie = same & (gi[:, None] < gi[None, :])
        first = (G_lo[:, :, None] > G_hi[:, None, :]) | tie   # [n, g, h]: group g certainly ranks before group h
        decided &= (first | ~(kept[:, :, None] & ~kept[:, None, :])).all(axis=(1, 2))
        allowed = np.repeat(kept, E // router.n_group, axis=1)

    def precedes(r, a, b):   # the device's c[r, a] certainly ranks before c[r, b]: disjoint intervals, or identical
        same = (logits[r, a] == logits[r, b]) & (bv[a] == bv[b])   # inputs (identical device values) or c values
        same |= sel.exact[r, a] & sel.exact[r, b] & (c_mid[r, a] == c_mid[r, b])   # known exactly, with a < b
        return (c_lo[r, a] > c_hi[r, b]) | (same & (a < b))

    for j in range(k - 1):
        decided &= precedes(rows, picks[:, j], picks[:, j + 1])
    rest = allowed.copy()
    rest[rows[:, None], picks] = False
    decided &= (precedes(rows[:, None], picks[:, -1:], np.arange(E)[None, :]) | ~rest).all(1)
    ambiguous = int((~decided).sum())
    bad = decided & (np.asarray(dev_idx) != picks).any(1)
    if bad.any():
        t = int(np.flatnonzero(bad)[0])
        j = int(np.flatnonzero(dev_idx[t] != picks[t])[0])
        raise AssertionError(f"topk_idx (gated): {int(bad.sum())} decided tokens differ; first token {t} pick {j}: "
                             f"device {list(map(int, dev_idx[t]))}, reference {picks[t].tolist()} (selection values "
                             f"of those experts: {c_mid[t, dev_idx[t]].tolist()} vs {c_mid[t, picks[t]].tolist()})")
    w_lo, w_hi = weights_bounds(sc, picks, router)
    kk = ex.order_key(dev_w)
    wok = (kk >= ex.order_key(ex.f64_to_bf16(w_lo))) & (kk <= ex.order_key(ex.f64_to_bf16(w_hi)))
    wbad = decided[:, None] & ~wok
    if wbad.any():
        t, j = (int(v) for v in np.argwhere(wbad)[0])
        raise AssertionError(f"topk_w (gated): {int(wbad.any(1).sum())} tokens with a weight outside its interval; "
                             f"first token {t} pick {j} (expert {int(picks[t, j])}): device {ex._fmt(dev_w[t, j])}, "
                             f"reference [{w_lo[t, j]!r}, {w_hi[t, j]!r}]")
    return ambiguous


def reference_routing(router, bias, k: int, x: np.ndarray, wg_eff: np.ndarray):
    """A gated launch's routing computed from the interval midpoints (scores, selection values, picks, weights), what
    a correct kernel could have produced: (picks int32 [n, k], fp32 weights [n, k], gate_out bf16 bits [n, E])."""
    n, E = x.shape[0], wg_eff.shape[0]
    sc = scores(router, k, x, wg_eff)
    sel = selection(sc, bias, E)
    G = group_scores(sel, router)[2] if router.n_group > 1 and n else None
    picks = route_mid(sel.mid, router, k, G) if n else np.zeros((0, k), np.int32)
    w_lo, w_hi = weights_bounds(sc, picks, router)
    return picks, (0.5 * (w_lo + w_hi)).astype(np.float32), ex.f64_to_bf16(sc.s_mid)


# ----------------------------------------------------------------------------- training-mode auxiliary loss
def check_aux(aux: np.ndarray, ref: ex.RouterRef, counts: np.ndarray, n: int, rg: Regime) -> None:
    """gML, gMeC and the loss of a training launch over n tokens (aux = [gML E | gMeC E | loss]).
    gML[e] = sum_t p[t, e] / n: an interval from p_lo / p_hi, widened by a first-order bound of the kernel's fp32
    sums (a term passes at most ceil(TS / 32) lane adds, 5 shuffle adds, one add per sub-chunk, the division and one
    atomic add per CTA).  gMeC[e] = __fdividef(counts[e], n): within the division's bound of counts / n, and equal to it
    when n is a power of two.  The loss sum_e gML gMeC / E: an interval from those of gML and gMeC."""
    E = counts.shape[0]
    gml, gmec, loss = aux[:E].astype(np.float64), aux[E:2 * E].astype(np.float64), float(aux[2 * E])
    if n == 0:
        ex.check_equal(aux, np.zeros_like(aux), "aux (no tokens: all zero)", ("entry",))
        return
    depth = -(-rg.TS // 32) + 5 + len(rg.sub_chunks) + rg.grid + 4
    tot_hi = ref.p_hi.sum(0)
    slack = depth * ex.U32 * tot_hi / n + ex.EPS_DIV * tot_hi / n
    lo, hi = ref.p_lo.sum(0) / n - slack, tot_hi / n + slack
    bad = (gml < lo) | (gml > hi)
    if bad.any():
        e = int(np.flatnonzero(bad)[0])
        raise AssertionError(f"gML: {int(bad.sum())} of {E} experts outside the interval; first expert {e}: device "
                             f"{gml[e]!r}, reference [{lo[e]!r}, {hi[e]!r}]")
    ce = counts.astype(np.float64) / n
    if n & (n - 1) == 0:
        ex.check_equal(aux[E:2 * E], ce.astype(np.float32), "gMeC = counts / n", ("expert",))
    else:
        bad = np.abs(gmec - ce) > ex.EPS_DIV * ce
        assert not bad.any(), (f"gMeC: expert {int(np.flatnonzero(bad)[0])}: device "
                               f"{gmec[bad][0]!r}, counts / n {ce[bad][0]!r}")
    t_lo, t_hi = np.maximum(lo, 0) * gmec / E, hi * gmec / E
    l_lo = t_lo.sum() * (1 - (E + 6) * ex.U32)   # per term: the product, __fdividef (4 roundings' worth), E adds
    l_hi = t_hi.sum() * (1 + (E + 6) * ex.U32)
    assert l_lo <= loss <= l_hi, f"aux loss: device {loss!r} outside [{l_lo!r}, {l_hi!r}]"
