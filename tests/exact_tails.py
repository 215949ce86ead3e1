"""Exact inputs that reach the tails of the forward's nonlinear steps, and counts of the tail regions a launch covered.

The exact-input generators (tests/exact.py, exact_swiglu.py) keep GELU pre-activations >= 0, SwiGLU gates in [-4, 4]
and router logits small, where the kernel's fp32 formulas track the real functions to a relative bound.  These inputs
go where they do not:
  GELU     pre-activations v on the 2^-3 grid over about [-10, 6], negative biases included: 1 + erff cancels below
           zero, and below about v = -5.8 erff may return -1 and h is -0 (exact.gelu_neg_f32);
  SwiGLU   gates g on the 1/2 grid over about [-136, 136]: the subnormal sigma band (g in [-88.5, -87.5]) and the
           overflow cliff below g = -88.72, where h is exactly +-0 (exact_swiglu.silu_mul_rounded);
  sigmoid  router logits >= 64 on blocks of experts (score exactly 1.0: ties decided by the bias and the lower index,
           group scores fl(1 + 1) that tie), logits <= -124 (score +0), and biases below 2^-25 that fl(1 + b) absorbs
           (exact_gated.sigmoid_bounds, check_gated_routing).
GEMM0 stays exact: x column H - 1 is a constant 1 whose gate weights are zero (the router ignores it), so a W_up or
W_gate entry there acts as a per-row offset.  GEMM1 stays exact: the tail pre-activations sit in every fourth
intermediate column, whose W_down column is all zero (exact.assert_exact_sums ignores products that are zero); the
other columns keep the generators' coarse h.  No pytest in here.
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from tests import exact as ex
from tests import exact_gated as eg
from tests import exact_shared as es
from tests import exact_swiglu as sw

SAT_W, NEG_W = 64.0, -128.0   # router weights of x columns 0 and 1 on the saturated and the +0 blocks
SAT_BLOCK = (0, 1, 2, 4, 5, 7, 8, 9, 10, 11, 13, 14)   # experts (mod 16) whose logit is >= 64 - 6 when x[:, 0] = 1
NEG_BLOCK = (2, 6, 9, 12, 15)                            # experts whose logit is <= -124 when x[:, 1] = 1
ALWAYS_SAT = (8, 10)                                     # experts saturated on every token (the tiny biases sit there)
SWIGLU_OFFSETS = (-120, -104, -96, -92, -88, -88, -88, -84, -72, -48, -24, -12, 12, 24, 48, 72, 88, 96, 120)


def tail_columns(P: int) -> np.ndarray:
    """bool [P]: the intermediate columns that carry tail pre-activations (every fourth; W_down zero there)."""
    return np.arange(P) % 4 == 3


def _bf(a) -> torch.Tensor:
    t = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).bfloat16()
    assert np.array_equal(t.double().numpy(), a), "generator produced a value that is not a bf16 number"
    return t


def _free_cols(H: int, rng, size: int) -> np.ndarray:
    """Columns of x for tail entries: clear of the routing columns at the front and of the constant column H - 1."""
    return rng.choice(np.arange(H // 2, H - 1), size=size, replace=False)


def constant_column(base: ex.ExactInputs) -> None:
    """x[:, H-1] = 1 for every token, Wg_eff[:, H-1] = 0 (in place; the router's logits do not change)."""
    cfg = base.cfg
    H, E = cfg.H, cfg.E
    x = base.x.reshape(-1, H).double().numpy().copy()
    wg = base.wg.reshape(-1).reshape(E, H).double().numpy().copy()
    x[:, H - 1] = 1
    wg[:, H - 1] = 0
    base.x = _bf(x).reshape(base.x.shape)
    base.wg = _bf(wg.reshape(-1).reshape(H, E))
    base.__dict__.pop("x64", None)
    base.__dict__.pop("wg_eff64", None)


def saturating_router(base: ex.ExactInputs, seed: int, sat_frac: float = 0.7, neg_frac: float = 0.3) -> None:
    """Logit blocks on x columns 0 and 1 (in place): a `sat_frac` share of tokens gets x[:, 0] = 1, lifting the experts
    of SAT_BLOCK by SAT_W (every other logit term stays within +-6, so those logits are >= 58 and their scores exactly
    1.0); a `neg_frac` share gets x[:, 1] = 1, lowering NEG_BLOCK by 128 (scores +0); ALWAYS_SAT is lifted on every
    token through the constant column (call constant_column first).  The rest of each logit comes from x columns 2 .. 9
    alone and is >= 0: sigmoid(l) + sigmoid(-l) = 1 would otherwise make group scores of different experts agree to
    the last bit in real arithmetic, which no interval can order."""
    cfg = base.cfg
    H, E, S = cfg.H, cfg.E, cfg.S
    g = np.random.default_rng(seed)
    x = base.x.reshape(-1, H).double().numpy().copy()
    wg = base.wg.reshape(-1).reshape(E, H).double().numpy().copy()
    x[:, :2] = 0
    wg[:, :2] = 0
    wg[:, 10:] = 0   # the other logit terms from x columns 2 .. 9 only: |x| <= 8, |Wg_eff| <= 2^-4 -> at most 4
    x[:, 2:10], wg[:, 2:10] = np.abs(x[:, 2:10]), np.abs(wg[:, 2:10])
    x[:, 0] = g.random(S) < sat_frac
    x[:, 1] = g.random(S) < neg_frac
    e = np.arange(E)
    wg[np.isin(e % 16, SAT_BLOCK), 0] = SAT_W
    wg[np.isin(e % 16, NEG_BLOCK), 1] = NEG_W
    wg[np.isin(e % 16, ALWAYS_SAT), H - 1] = SAT_W   # (x[:, H-1] = 1: constant_column)
    rest = x[:, 2:10] @ wg[:, 2:10].T
    assert rest.max() <= 6, f"logit terms outside the blocks reach {rest.max()}"
    base.x = _bf(x).reshape(base.x.shape)
    base.wg = _bf(wg.reshape(-1).reshape(H, E))
    base.__dict__.pop("x64", None)
    base.__dict__.pop("wg_eff64", None)


def score_bias(E: int) -> np.ndarray:
    """fp32 [E]: zeros (equal biases), 2^-26 on the two ALWAYS_SAT experts (below half an ulp of 1: fl(1 + b) = 1;
    on an unsaturated score fl(s + b) would be undecidable), 2^-9 on two
    (equal, unequal to the rest), -2^-8 on one."""
    b = np.zeros(E, np.float32)
    for e, v in ((10, 2.0 ** -26), (8, 2.0 ** -26), (5, 2.0 ** -9), (13, 2.0 ** -9), (12, -2.0 ** -8)):
        if e < E:
            b[e] = v
    return b


# ----------------------------------------------------------------------------- the tail columns
def gelu_tail_rows(w, down, b, rng) -> None:
    """In place, for one GELU expert (w [2, P, H], W_down [H, P], b_up [P] or None): the tail columns get an offset in
    [-7, 3] on 2^-3 at the constant column, two entries +-2^-3 (x in [0, 8]: +-2 more), a signed bias in [-1, 1] on
    2^-3 and a zero W_down column."""
    w_up = w[0]
    P, H = w_up.shape
    cols = np.flatnonzero(tail_columns(P))
    w_up[cols] = 0
    w_up[cols, H - 1] = rng.integers(-56, 25, size=cols.size) * 2.0 ** ex.WUP_GRID
    for p in cols:
        w_up[p, _free_cols(H, rng, 2)] = rng.choice([-1.0, 1.0], size=2) * 2.0 ** ex.WUP_GRID
    down[:, cols] = 0
    if b is not None:
        b[cols] = rng.integers(-8, 9, size=cols.size) * 2.0 ** ex.WUP_GRID


def swiglu_tail_rows(w, down, b, rng) -> None:
    """In place, for one SwiGLU expert (w [3, P, H], W_down [H, P], b_up [2, P] or None; x in {-1, 0, 1}): the tail
    columns get a gate offset from SWIGLU_OFFSETS at the constant column plus three entries in [-4, 4] on 1/2 (g within
    +-12 of it, +-4 more from the bias), an up offset in +-[1, 4] and one entry +-1, and a zero W_down column."""
    gate, up = w[0], w[1]
    P, H = gate.shape
    cols = np.flatnonzero(tail_columns(P))
    gate[cols] = 0
    up[cols] = 0
    gate[cols, H - 1] = [SWIGLU_OFFSETS[int(i)] for i in rng.integers(0, len(SWIGLU_OFFSETS), size=cols.size)]
    up[cols, H - 1] = rng.choice([-4.0, -3.0, -2.0, -1.0, 1.0, 2.0, 3.0, 4.0], size=cols.size)
    for p in cols:
        gate[p, _free_cols(H, rng, 3)] = rng.choice([v / 2 for v in range(-8, 9) if v], size=3)
        up[p, _free_cols(H, rng, 1)] = rng.choice([-1.0, 1.0])
    down[:, cols] = 0
    if b is not None:
        b[0, cols] = rng.integers(-8, 9, size=cols.size) * 0.5
        b[1, cols] = rng.integers(-2, 3, size=cols.size)


def with_tails(experts: ex.Experts, rng) -> ex.Experts:
    """The record with the activation's tail columns (gelu_tail_rows, swiglu_tail_rows) in every expert, in order."""
    tail_rows = gelu_tail_rows if experts.act == 1 else swiglu_tail_rows
    w = experts.w.double().numpy().copy()
    bu = None if experts.bu is None else experts.bu.double().numpy().copy()
    E, m, P, H = w.shape
    for e in range(E):
        down = w[e, m - 1].reshape(-1).reshape(H, P).copy()
        tail_rows(w[e], down, None if bu is None else bu[e], rng)
        w[e, m - 1] = down.reshape(-1).reshape(P, H)
    return ex.Experts(_bf(w), None if bu is None else _bf(bu), experts.bd, experts.act)


def tail_inputs(cfg, seed: int, bias: bool, saturate: bool = False, **router_kw) -> ex.ExactInputs:
    """Exact inputs with the tail columns of the context's activation (GELU: exact.exact_inputs(gelu_friendly);
    SwiGLU: exact_swiglu.swiglu_inputs) in every expert, and saturated router blocks with `saturate`."""
    if cfg.hidden_act == 1:
        inp = ex.exact_inputs(cfg, seed, bias=bias, gelu_friendly=True, **router_kw)
    else:
        inp = sw.swiglu_inputs(cfg, seed, bias, **router_kw)
    inp.experts = with_tails(inp.experts, np.random.default_rng(seed + 7))
    constant_column(inp)
    if saturate:
        saturating_router(inp, seed + 11)
    return inp


def tail_shared(H: int, Ps: int, seed: int, act: int, bias: bool) -> ex.Experts:
    """A shared expert of activation `act` with the tail columns."""
    if act == 1:
        se = es.shared_inputs(H, Ps, seed, act=1, bias=bias, gelu_friendly=True)
    else:
        se = sw.shared_swiglu(H, Ps, seed, bias)
    return with_tails(se, np.random.default_rng(seed + 5))


def activation_regions(experts: ex.Experts, e: int, rows: np.ndarray) -> Dict[str, int]:
    """The region counts (gelu_regions, swiglu_regions) of expert e's pre-activations for the rows."""
    return (gelu_regions if experts.act == 1 else swiglu_regions)(*experts.pre(e, rows))


# ----------------------------------------------------------------------------- regions
def gelu_regions(v: np.ndarray) -> Dict[str, int]:
    """Counts of GELU pre-activations below zero, and of those whose interval admits the kernel's -0."""
    v = np.asarray(v, np.float64).ravel()
    neg = v < 0
    r = ex.gelu_rounded(v[neg])
    return {"GELU v < 0": int(neg.sum()), "GELU -0 tail": int((ex.order_key(r.hi) == 0).sum())}


def swiglu_regions(g: np.ndarray, u: np.ndarray) -> Dict[str, int]:
    """Counts of (g, u != 0) pairs with |g| > 4, in the subnormal sigma band (126 < a < 128) and past the cliff."""
    g, u = np.asarray(g, np.float64).ravel(), np.asarray(u, np.float64).ravel()
    a = sw.power_arg(g)
    nz = u != 0
    return {"SwiGLU |g| > 4": int((nz & (np.abs(g) > 4)).sum()),
            "SwiGLU subnormal sigma": int((nz & (a > 126) & (a < ex.EX2_OVERFLOW)).sum()),
            "SwiGLU cliff": int((nz & (a >= ex.EX2_OVERFLOW)).sum())}


def router_regions(logits: np.ndarray, bias, router) -> Dict[str, int]:
    """Tokens with two experts whose selection values are exactly equal saturated scores, (token, expert) pairs whose
    nonzero bias fl(1 + b) absorbs, tokens with +0 scores, and tokens with two equal exact group scores."""
    E = logits.shape[1]
    lo, hi, mid = eg.sigmoid_bounds(logits)
    sc = eg.Scores(lo, hi, mid, ex.f64_to_bf16(lo), ex.f64_to_bf16(hi))
    sel = eg.selection(sc, bias, E)
    sat = sel.exact & (lo == 1.0)
    c = np.where(sat, sel.mid, np.nan)
    ties = (c[:, :, None] == c[:, None, :]) & ~np.eye(E, dtype=bool)[None]
    b = np.zeros(E) if bias is None else np.asarray(bias, np.float64)
    out = {"saturated score ties": int(ties.any(axis=(1, 2)).sum()),
           "absorbed biases": int((sat & (b != 0)[None, :] & (sel.mid == 1.0)).sum()),
           "+0 scores": int((sel.exact & (hi == 0)).any(axis=1).sum())}
    if router.n_group > 1:
        _, _, G, G_ex = eg.group_scores(sel, router)
        Gc = np.where(G_ex, G, np.nan)
        NG = Gc.shape[1]
        out["tied group scores"] = int(((Gc[:, :, None] == Gc[:, None, :]) & ~np.eye(NG, dtype=bool)[None])
                                       .any(axis=(1, 2)).sum())
    return out


def add_regions(acc: Dict[str, int], new: Dict[str, int]) -> None:
    for k, v in new.items():
        acc[k] = acc.get(k, 0) + v
