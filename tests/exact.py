"""Inputs on which fp32 arithmetic is exact, a float64 reference of every stage of the forward, and per-stage checkers.

Every input is a small integer times a power of two: x on a grid of 1, the gate weights on 2^-6, W_up on 2^-3, W_down on
2^-5, the biases on the grid of the product they are added to.  When, for every output element, sum |a_i * b_i| stays
below 2^24 grid units, every partial sum in any order is an fp32 number, so the router logits and the pre-rounding values
of `h` and `y` are exact whatever the tile shape, k-block order or wgmma reduction tree.  On such inputs float64 numpy
computes the exact answer, and a correct kernel has freedom only in three documented approximations:

  1. the softmax: ex2.approx.ftz on fl(z * log2e), the fma recurrence of the denominator and __fdividef
     (gate_out, topk_w, mcw);
  2. GELU: erff and three fp32 operations (relative EPS_GELU for v >= 0, the kernel's steps from erff's ends below);
  3. the combine's __fdividef(y, mcw).

For those the reference is an interval: each rounding step is monotone, so the ends run through the kernel's own sequence
of roundings, and the device value must lie inside.  Everything else (ReLU, bias adds, the RNE conversions, the bf16
products and the bf16 accumulation of the combine) is checked bit for bit.  Top-k is decided exactly: distinct logits
differ by at least one grid step, ties are exact, and an expert whose probability flushes to zero is picked in index
order behind the others.

One launch of any route, activation (the expert record `Experts`) and shared expert is checked by check_launch, and
reference_launch builds a correct launch record by the same walk.  The checkers raise AssertionError naming the stage,
the first failing (token, pick) or (packet, row, column), and the device and reference bits.  `Launcher` runs a route
on a GPU context and reads the launch back.  No pytest in here.
"""
from __future__ import annotations

import dataclasses
import functools
import os
from typing import Dict, Optional, Sequence

import numpy as np
import torch

from flashmoe_b200.config import MoEConfig

# ----------------------------------------------------------------------------- grids and fp32 limits
X_GRID, WG_GRID, WUP_GRID, WDOWN_GRID = 0, -6, -3, -5   # log2 of the grid step of each operand
EXACT_UNITS = 2 ** 24                                   # sum |a b| below this many product-grid units: fp32-exact sums

LOG2E_F32 = np.float32(1.4426950408889634)              # the constant fast_expf multiplies by (fm_ptx.cuh)
FLUSH_T = -126.0                                        # ex2.approx.ftz: a result below 2^-126 is flushed to +0
FLUSH_MARGIN = 0.01                                     # no logit gap within this of the flush threshold
MIN_PROB = 2.0 ** -120                                  # non-flushed probabilities stay well inside the normal range

# Error bounds of the three approximations (relative, for normal fp32 values).
#   ex2.approx.ftz.f32: the PTX ISA documents a maximum relative error of about 2 ulp (2^-22) over the normal range;
#     taken as 2^-21.
EPS_EX2 = 2.0 ** -21
#   __fdividef(x, y): 2 ulp for 2^-126 <= |y| <= 2^126 (CUDA C++ Programming Guide, intrinsic functions) -> 2^-22.
EPS_DIV = 2.0 ** -22
#   GELU 0.5f * v * (1.0f + erff(v * 0.70710678f)) for v >= 0 (below zero 1 + erff cancels; gelu_neg_f32 there):
#     fl(v * c) with c = fl32(1/sqrt 2): 2^-24 + 2^-24; erf is concave on [0, inf), so a relative error d of its
#     argument moves erf by at most d relative -> 2^-23; erff itself 2 ulp (Programming Guide, standard functions)
#     -> 2^-22; 1 + e rounds once (2^-24) and does not amplify e's relative error since e >= 0; the final product
#     rounds once (2^-24; 0.5f * v is exact).  Total 7 * 2^-24, taken as 8 * 2^-24.
EPS_GELU = 8 * 2.0 ** -24
U32 = 2.0 ** -24                                        # one fp32 rounding (RNE)


# ----------------------------------------------------------------------------- bf16 bit helpers
def to_bits(t: torch.Tensor) -> np.ndarray:
    assert t.dtype == torch.bfloat16
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16).copy()


def from_bits(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16).copy()).view(torch.bfloat16)


def bits_to_f64(a: np.ndarray) -> np.ndarray:
    return (np.asarray(a, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def f32_to_bf16(a32: np.ndarray) -> np.ndarray:
    """fp32 -> bf16 bits, round to nearest even (no NaNs occur here)."""
    u = np.ascontiguousarray(a32, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def f64_to_bf16(a: np.ndarray) -> np.ndarray:
    """float64 -> fp32 (RNE) -> bf16 (RNE): a single rounding for values that are fp32 numbers, and monotone always."""
    return f32_to_bf16(np.asarray(a, dtype=np.float64).astype(np.float32))


def f64_to_bf16_trunc(a: np.ndarray) -> np.ndarray:
    """Round toward zero instead of to nearest even (planted fault)."""
    u = np.ascontiguousarray(np.asarray(a, dtype=np.float64).astype(np.float32)).view(np.uint32)
    return (u >> 16).astype(np.uint16)


def order_key(bits: np.ndarray) -> np.ndarray:
    """Integer key monotone in the bf16 value (+0 and -0 share key 0); one bf16 ulp = 1."""
    b = np.asarray(bits, dtype=np.uint16).astype(np.int32)
    mag = b & 0x7FFF
    return np.where(b & 0x8000, -mag, mag)


def grid_log2(a: np.ndarray) -> int:
    """Largest q such that every element of `a` (bf16 values as float64) is a multiple of 2^q (0 for an all-zero array)."""
    v = np.abs(np.asarray(a, dtype=np.float64)).ravel()
    hi = float(v.max(initial=0.0))
    if hi == 0:
        return 0
    lo = float(v.min(where=v > 0, initial=np.inf))
    if 2.0 ** -126 <= lo and hi < 2.0 ** 127 and hi < lo * 2.0 ** 50:
        # fast path (a weight matrix of a model-sized layer): every element is a multiple of 2^Q, Q = the exponent of
        # the smallest one less bf16's 7 fraction bits; the lowest set bit of the OR of all of them in units of 2^Q
        # is the grid
        f = v.astype(np.float32)
        assert np.array_equal(f, v) and not (f.view(np.uint32) & 0xFFFF).any(), "not a bf16 value"
        Q = int(np.frexp(lo)[1]) - 8
        acc = int(np.bitwise_or.reduce((v * 2.0 ** -Q).astype(np.int64)))
        return Q + (acc & -acc).bit_length() - 1
    v = v[v != 0]
    # from the float64 bits: the significand (implicit bit included for normals) over its lowest set bit is the odd
    # part, which has at most bf16's 8 significant bits; the lowest set bit gives the element's grid
    u = v.view(np.uint64)
    e = (u >> np.uint64(52)).astype(np.int64)
    m = (u & np.uint64((1 << 52) - 1)) | np.where(e > 0, 1 << 52, 0).astype(np.uint64)
    low = m & (~m + np.uint64(1))
    assert (m < (low << np.uint64(8))).all(), "not a bf16 value"
    return int((np.maximum(e, 1) - 1075 + np.log2(low).astype(np.int64)).min())


def _fmt(bits) -> str:
    b = int(bits)
    return f"0x{b:04x} ({float(bits_to_f64(np.array([b]))[0]):.9g})"


# ----------------------------------------------------------------------------- experts
class PerExpert:
    """Expert weights drawn on demand: w[e, i] = fn(e, i), block i of expert e (bf16 [P, H]), of a [E, m, P, H] whole
    that is never built on the host."""

    def __init__(self, fn, shape):
        self.fn, self.shape = fn, tuple(shape)

    def __getitem__(self, key):
        e, i = key
        return self.fn(int(e), int(i))


@dataclasses.dataclass
class Experts:
    """E experts of one activation `act` (hidden_act): bf16 weights w [E, m, P, H] -- m = 2, W_up then the P*H block
    flat-viewed as W_down [H, P]; m = 3 for SwiGLU, W_gate, W_up, W_down -- and biases bu [E, P] ([E, 2, P]: gate, up)
    and bd [E, H], or None.  `w` may be a PerExpert: the reference reads one expert block at a time, so a model-sized
    layer is never held in float64 whole.  A shared expert is a record with E = 1."""
    w: object
    bu: Optional[torch.Tensor]
    bd: Optional[torch.Tensor]
    act: int

    def _block64(self, e: int, i: int) -> np.ndarray:
        return self.w[e, i].double().numpy()

    def pre(self, e: int, rows: np.ndarray, what: str = "GEMM0"):
        """The pre-activations of expert e for the rows (float64 [M, H]): [v] or, for SwiGLU, [g, u], each [M, P] and
        exact (the sums are asserted exact in fp32)."""
        n_pre = self.w.shape[1] - 1
        b = None if self.bu is None else self.bu[e].double().numpy().reshape(n_pre, -1)
        names = ("",) if n_pre == 1 else (" (gate)", " (up)")
        out = []
        for i in range(n_pre):
            w, bi = self._block64(e, i), None if b is None else b[i]
            assert_exact_sums(rows, w, bi, what + names[i])
            v = rows @ w.T
            out.append(v if bi is None else v + bi[None, :])
        return out

    def h(self, e: int, rows: np.ndarray, what: str = "GEMM0") -> Rounded:
        """h = RNE(act(pre-activations)) of expert e for the rows: ReLU exact, GELU's interval (gelu_rounded), SwiGLU's
        (exact_swiglu.silu_mul_rounded)."""
        pre = self.pre(e, rows, what)
        if self.act == 0:
            a = np.maximum(pre[0], 0.0)
            b = f64_to_bf16(a)
            return Rounded(b, b, a)
        if self.act == 1:
            return gelu_rounded(pre[0])
        from tests.exact_swiglu import silu_mul_rounded

        return silu_mul_rounded(*pre)

    def down(self, e: int):
        """(W_down [H, P], b_down [H] or None) of expert e in float64."""
        _, m, P, H = self.w.shape
        return (self._block64(e, m - 1).reshape(-1).reshape(H, P),
                None if self.bd is None else self.bd[e].double().numpy())

    def y(self, e: int, h_bits: np.ndarray, what: str = "GEMM1") -> Rounded:
        return gemm1_reference(h_bits, *self.down(e), what)

    def device(self, dev):
        """(w, bu, bd) on `dev`, the weights uploaded one block at a time."""
        w = torch.empty(self.w.shape, dtype=torch.bfloat16, device=dev)
        for e in range(w.shape[0]):
            for i in range(w.shape[1]):
                w[e, i] = self.w[e, i].to(dev)
        return (w, *(None if b is None else b.to(dev) for b in (self.bu, self.bd)))


def shared_expert(se: Experts, dev):
    """The runtime.SharedExpert of a one-expert record, on `dev`."""
    from flashmoe_b200.runtime import SharedExpert

    w, bu, bd = se.device(dev)
    return SharedExpert(w[0], None if bu is None else bu[0], None if bd is None else bd[0])


# ----------------------------------------------------------------------------- inputs
@dataclasses.dataclass
class ExactInputs:
    cfg: MoEConfig
    x: torch.Tensor                 # [mini_batch, seq, H] bf16 (CPU)
    wg: torch.Tensor                # [H, E] bf16, flat view = Wg_eff [E, H]
    experts: Experts
    underflow_tokens: np.ndarray    # token indices built to flush all but one expert
    zero_tokens: np.ndarray         # token indices with x = 0 (all logits tie)

    @functools.cached_property
    def x64(self) -> np.ndarray:
        return self.x.reshape(-1, self.cfg.H).double().numpy()

    @functools.cached_property
    def wg_eff64(self) -> np.ndarray:
        return self.wg.reshape(-1).reshape(self.cfg.E, self.cfg.H).double().numpy()

    def device(self, dev):
        """(x, gate weights, expert weights, bias_up, bias_down) on `dev`."""
        return (self.x.to(dev), self.wg.to(dev), *self.experts.device(dev))


def exact_inputs(cfg: MoEConfig, seed: int, *, x_range: int = 8, wg_range: int = 4, up_range: int = 8,
                 down_range: int = 4, bias: bool = False, gelu_friendly: bool = False,
                 ties: Sequence[Sequence[int]] = (), boost_frac: float = 0.3, tie_boost: int = 16,
                 zero_tokens: int = 0, underflow_tokens: int = 0, first_choice: Optional[np.ndarray] = None,
                 route_gain: int = 32) -> ExactInputs:
    """Seeded exact inputs for `cfg` (CPU bf16 tensors).

    x: integers in [-x_range, x_range]; Wg_eff: integers in [-wg_range, wg_range] * 2^-6; W_up: integers in
    [-up_range, up_range] * 2^-3; W_down: integers in [-down_range, down_range] * 2^-5; b_up on 2^-3, b_down on 2^-8.

    Routing controls (x columns 0, 1 and 2 .. 2 + E are reserved for them when used):
      ties         expert groups whose Wg_eff rows are made identical (exact logit ties for every token); a
                   `boost_frac` share of the tokens gets x[:, 0] in {1, 2} and the tied experts a weight of
                   `tie_boost` there, which lifts the tied groups into those tokens' top-k.
      zero_tokens  tokens with x = 0: every logit is 0, p = 1/E, picks 0 .. k-1.
      underflow_tokens  tokens with x[:, 1] = 1; expert E-1 weighs 192 there and leads by more than 88 logit units,
                   so every other probability flushes to 0 and the rest of the top-k is picked in index order.
      first_choice planned routing: token t has x[t, 2 + first_choice[t]] = 1, and expert e weighs `route_gain` in
                   column 2 + e, so first_choice[t] leads every other expert (exact packet sizes for k = 1).
    gelu_friendly: x >= 0, sparse W_up >= 0 and b_up >= 0, so GELU pre-activations are >= 0 and the GELU error bound
    applies, and h keeps a grid coarse enough for GEMM1 to stay exact."""
    g = np.random.default_rng(seed)
    S, H, P, E = cfg.S, cfg.H, cfg.P, cfg.E
    if gelu_friendly:
        x = g.integers(0, x_range + 1, size=(S, H)).astype(np.float64)
        up = g.integers(1, up_range + 1, size=(E, P, H)) * (g.random((E, P, H)) < 4.0 / H)
    else:
        x = g.integers(-x_range, x_range + 1, size=(S, H)).astype(np.float64)
        up = g.integers(-up_range, up_range + 1, size=(E, P, H))
    wg = g.integers(-wg_range, wg_range + 1, size=(E, H)).astype(np.float64) * 2.0 ** WG_GRID
    up = up.astype(np.float64) * 2.0 ** WUP_GRID
    down = g.integers(-down_range, down_range + 1, size=(E, H, P)).astype(np.float64) * 2.0 ** WDOWN_GRID
    bu = bd = None
    if bias:
        lo = 0 if gelu_friendly else -16
        bu = g.integers(lo, 17, size=(E, P)).astype(np.float64) * 2.0 ** WUP_GRID
        bd = g.integers(-256, 257, size=(E, H)).astype(np.float64) * 2.0 ** (WUP_GRID + WDOWN_GRID)

    reserved = 2 + (E if first_choice is not None else 0)
    if ties or underflow_tokens or first_choice is not None:
        assert H > reserved, f"H={H} leaves no room for the routing columns"
        x[:, :reserved] = 0
        wg[:, :reserved] = 0
    if first_choice is not None:
        fc = np.asarray(first_choice)
        assert fc.shape == (S,)
        x[np.arange(S), 2 + fc] = 1
        wg[np.arange(E), 2 + np.arange(E)] = route_gain
    tied = sorted({e for grp in ties for e in grp})
    for grp in ties:
        for e in grp[1:]:
            wg[e] = wg[grp[0]]
    if ties:
        boosted = g.random(S) < boost_frac
        x[boosted, 0] = g.integers(1, 3, size=int(boosted.sum()))
        wg[tied, 0] = tie_boost
    under = np.sort(g.choice(S, size=underflow_tokens, replace=False)) if underflow_tokens else np.zeros(0, np.int64)
    if underflow_tokens:
        x[under, 0] = 0
        x[under, 1] = 1
        wg[E - 1, 1] = 192
    zeros = np.setdiff1d(np.arange(S), under)
    zeros = np.sort(g.choice(zeros, size=zero_tokens, replace=False)) if zero_tokens else np.zeros(0, np.int64)
    x[zeros] = 0

    def bf(a):
        t = torch.from_numpy(np.ascontiguousarray(a)).bfloat16()
        assert np.array_equal(t.double().numpy(), a), "generator produced a value that is not a bf16 number"
        return t

    we = np.stack([up, down.reshape(E, -1).reshape(E, P, H)], axis=1)
    experts = Experts(bf(we), None if bu is None else bf(bu), None if bd is None else bf(bd), cfg.hidden_act)
    return ExactInputs(cfg, bf(x).reshape(cfg.mini_batch, cfg.sequence_len, H), bf(wg.reshape(-1).reshape(H, E)),
                       experts, under, zeros)


# ----------------------------------------------------------------------------- preconditions
def assert_exact_sums(a: np.ndarray, b: np.ndarray, bias: Optional[np.ndarray], what: str) -> None:
    """a [M, K] @ b[N, K]^T (+ bias [N]) has every partial sum exact in fp32: all values on a common product grid and
    sum |a b| + |bias| below 2^24 grid units for every output element.  A column k of `a` whose column of `b` is all
    zero (and the other way round) only forms products that are zero, which are exact whatever its grid, so its grid
    does not count (the tail tests put tiny h values in intermediate columns whose W_down column is zero)."""
    if a.size == 0 or b.size == 0:
        return
    q = grid_log2(a) + grid_log2(b)
    tot = np.abs(a) @ np.abs(b).T
    if bias is not None:
        assert grid_log2(bias) >= q or not np.any(bias), f"{what}: bias is off the product grid 2^{q}"
        tot = tot + np.abs(bias)[None, :]
    worst = float(tot.max())
    if worst >= EXACT_UNITS * 2.0 ** q:   # the grid of the nonzero products alone (the zero ones add nothing to tot)
        a = np.where(np.any(b != 0, axis=0)[None, :], a, 0.0)
        b = np.where(np.any(a != 0, axis=0)[None, :], b, 0.0)
        q = grid_log2(a) + grid_log2(b)
        if bias is not None and np.any(bias):   # (that grid may be coarser than the bias's)
            q = min(q, grid_log2(bias))
    assert worst < EXACT_UNITS * 2.0 ** q, (f"{what}: sum |ab| reaches {worst:.6g} = {worst / 2.0 ** q:.4g} units of "
                                            f"2^{q}, not below 2^24: fp32 partial sums would not be exact")


# ----------------------------------------------------------------------------- router reference
@dataclasses.dataclass
class RouterRef:
    logits: np.ndarray     # float64 [n, E], exact
    flushed: np.ndarray    # bool [n, E]: probability exactly +0
    topk: np.ndarray       # int32 [n, k]
    p_lo: np.ndarray       # float64 [n, E] bounds of the device's fp32 probability
    p_hi: np.ndarray
    go_lo: np.ndarray      # bf16 bits [n, E] bounds of gate_out
    go_hi: np.ndarray

    def mcw_bounds(self):
        k = self.topk.shape[1]
        rows = np.arange(self.topk.shape[0])[:, None]
        lo = self.p_lo[rows, self.topk].sum(1) * (1 - U32) ** k
        hi = self.p_hi[rows, self.topk].sum(1) * (1 + U32) ** k
        return lo, hi


def router_reference(x: np.ndarray, wg_eff: np.ndarray, k: int) -> RouterRef:
    n, E = x.shape[0], wg_eff.shape[0]
    assert_exact_sums(x, wg_eff, None, "router logits")
    logits = x @ wg_eff.T
    if n == 0:
        z = np.zeros((0, E))
        return RouterRef(z, z.astype(bool), np.zeros((0, k), np.int32), z, z, z.astype(np.uint16), z.astype(np.uint16))
    m = logits.max(axis=1, keepdims=True)
    d32 = (logits - m).astype(np.float32)                       # exact: both on the 2^-6 grid, far below 2^24 units
    t32 = (d32 * LOG2E_F32).astype(np.float64)                 # fl(z * log2e), the argument of ex2 in the final pass
    near = np.abs(t32 - FLUSH_T) < FLUSH_MARGIN * float(LOG2E_F32)
    assert not near.any(), f"token {int(np.argwhere(near)[0][0])}: a logit gap lies within {FLUSH_MARGIN} of the flush threshold"
    flushed = t32 < FLUSH_T
    # denominator: the recurrence dI = fma(dI, ex2(t(pM - mI)), ex2(t(l_e - mI))) against D = sum 2^((l_e - m) c):
    #   every ex2 call is within EPS_EX2 and a term passes through at most E of them, every fma rounds once (E * U32);
    #   the t() roundings along a term's path add exponent errors that telescope to at most U32 * c * (m - l_e), i.e.
    #   a relative 2^-24 * (m - l_e); terms and rescale factors that flush in the recurrence change dI by < 2^-126 * E.
    c = float(LOG2E_F32)
    D = np.where(flushed, 0.0, np.exp2(d32.astype(np.float64) * c)).sum(axis=1)
    spread = np.where(flushed, 0.0, -d32.astype(np.float64)).max(axis=1)
    dD = (E + 1) * (EPS_EX2 + U32) + U32 * spread + E * 2.0 ** -126
    D_lo, D_hi = D * (1 - dD), D * (1 + dD)
    num = np.exp2(t32)
    p_lo = np.where(flushed, 0.0, num * (1 - EPS_EX2) / D_hi[:, None] * (1 - EPS_DIV))
    p_hi = np.where(flushed, 0.0, num * (1 + EPS_EX2) / D_lo[:, None] * (1 + EPS_DIV))
    small = ~flushed & (p_lo < MIN_PROB)
    assert not small.any(), f"token {int(np.argwhere(small)[0][0])}: a probability leaves the normal fp32 range"
    # top-k: strict '>' in ascending expert order, i.e. larger p first and the lower index on equal p.  Distinct
    # logits give distinct p (they differ by >= 2^-6 in the exponent's argument, 1.6 %, far beyond the error bounds),
    # equal logits give identical device p, and flushed experts all have p = +0.
    key = np.where(flushed, -np.inf, logits)
    topk = np.argsort(-key, axis=1, kind="stable")[:, :k].astype(np.int32)
    return RouterRef(logits, flushed, topk, p_lo, p_hi, f64_to_bf16(p_lo), f64_to_bf16(p_hi))


# ----------------------------------------------------------------------------- bookkeeping
def slots_from_topk(topk: np.ndarray, E: int, EC: int):
    """slot [n, k]: position of (t, j) among all selections of its expert in ascending (token, pick) order, dropped ones
    counted; counts [E]: all selections; recv_cnt [E] = min(counts, EC); kept = slot < EC."""
    flat = np.asarray(topk, dtype=np.int64).reshape(-1)
    assert flat.size == 0 or (flat.min() >= 0 and flat.max() < E), "expert index out of range"
    counts = np.bincount(flat, minlength=E).astype(np.int32)
    order = np.argsort(flat, kind="stable")
    start = np.concatenate([[0], np.cumsum(counts)[:-1]])
    slot = np.empty(flat.size, dtype=np.int32)
    slot[order] = np.arange(flat.size) - start[flat[order]]
    slot = slot.reshape(topk.shape)
    return slot, counts, np.minimum(counts, EC).astype(np.int32), slot < EC


INT32_MAX = 2 ** 31 - 1


def slots_from_routing(topk: np.ndarray, E: int, EC: int):
    """slots_from_topk for routing that may hold -1 (no expert, the caller's routing): slot [n, k] (INT32_MAX for -1),
    counts [E], recv_cnt [E] = min(counts, EC), kept [n, k] = slot < EC."""
    topk = np.asarray(topk, dtype=np.int64)
    valid = topk >= 0
    assert (topk[valid] < E).all() and (topk[~valid] == -1).all(), "expert index outside [-1, E)"
    flat, vflat = topk.reshape(-1), valid.reshape(-1)
    slot = np.full(flat.size, INT32_MAX, dtype=np.int64)
    sub = flat[vflat]
    s, counts, recv_cnt, _ = slots_from_topk(sub.reshape(-1, 1), E, EC)   # ascending (token, pick) order kept
    slot[vflat] = s[:, 0]
    slot = slot.reshape(topk.shape).astype(np.int32)
    return slot, counts, recv_cnt, slot < EC


def sanitize(topk: np.ndarray, E: int) -> np.ndarray:
    """The caller's routing the kernel runs: indices outside [0, E) become -1."""
    t = np.asarray(topk, dtype=np.int32)
    return np.where((t >= 0) & (t < E), t, -1).astype(np.int32)


def routing_case(n: int, E: int, k: int, seed: int, *, skip_frac: float = 0.1, dup_frac: float = 0.1,
                 hot: int = 0, hot_frac: float = 0.5, empty=(), bad=()):
    """Seeded caller routing for n tokens: picks drawn from the experts not in `empty`, a `hot_frac` share of them sent
    to expert `hot` (skew that overflows its capacity), a `dup_frac` share of tokens naming one expert twice, a
    `skip_frac` share of picks set to -1, and `bad` (token, pick, value) entries written last.  Weights are fp32 in
    [-1, 2), with some exact zeros.  Returns (topk_idx int32 [n, k], topk_w float32 [n, k])."""
    g = np.random.default_rng(seed)
    allowed = np.array([e for e in range(E) if e not in set(empty)])
    idx = allowed[g.integers(0, len(allowed), size=(n, k))].astype(np.int32)
    if hot not in set(empty):
        idx[g.random((n, k)) < hot_frac] = hot
    if k > 1:
        dup = g.random(n) < dup_frac
        idx[dup, 1] = idx[dup, 0]
    idx[g.random((n, k)) < skip_frac] = -1
    for t, j, v in bad:
        if t < n:
            idx[t, j] = v
    w = (g.random((n, k)) * 3 - 1).astype(np.float32)
    w[g.random((n, k)) < 0.05] = 0.0
    return idx, w


def weights_f32(w_bits: np.ndarray) -> np.ndarray:
    """bf16 bits as the fp32 weights a routed replay takes (the same bits after rne_bf16)."""
    return (np.asarray(w_bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def packet_tokens(topk: np.ndarray, slot: np.ndarray, E: int, EC: int):
    """For every expert, the token of each kept slot in slot order (rows of its packet)."""
    out = []
    for e in range(E):
        t, j = np.nonzero((topk == e) & (slot < EC))
        out.append(t[np.argsort(slot[t, j])])
    return out


# ----------------------------------------------------------------------------- expert FFN reference
@dataclasses.dataclass
class Rounded:
    lo: np.ndarray          # bf16 bits
    hi: np.ndarray
    exact: np.ndarray       # float64 value before the final rounding (the midpoint for intervals)
    wide_ok: Optional[np.ndarray] = None   # bool: elements whose interval may span several bf16 ulps (GELU below zero)


def gelu_rounded(v: np.ndarray) -> Rounded:
    """The interval of the kernel's bf16 GELU of the exact pre-activations v (float64, fp32 values), over the whole
    real line: v >= 0 by EPS_GELU, v < 0 by gelu_neg_f32 (whose intervals may span several bf16 ulps: `wide_ok`)."""
    from scipy.special import erf, erfc

    v = np.asarray(v, dtype=np.float64)
    gl = np.where(v >= 0, 0.5 * v * (1.0 + erf(v / np.sqrt(2.0))),
                  0.5 * v * erfc(-v / np.sqrt(2.0)))   # 1 + erf(x) = erfc(-x), without the cancellation below zero
    lo, hi = f64_to_bf16(gl * (1 - EPS_GELU)), f64_to_bf16(gl * (1 + EPS_GELU))
    neg = v < 0
    if neg.any():
        nlo, nhi = gelu_neg_f32(v[neg])
        lo[neg], hi[neg] = f32_to_bf16(nlo), f32_to_bf16(nhi)
    return Rounded(lo, hi, gl, neg)


def f32_down(a: np.ndarray) -> np.ndarray:
    """The largest fp32 value <= a (float64 in, float32 out; +-inf kept)."""
    a = np.asarray(a, dtype=np.float64)
    with np.errstate(over="ignore"):
        f = a.astype(np.float32)
    return np.where(f.astype(np.float64) > a, np.nextafter(f, np.float32(-np.inf)), f).astype(np.float32)


def f32_up(a: np.ndarray) -> np.ndarray:
    """The smallest fp32 value >= a."""
    return -f32_down(-np.asarray(a, dtype=np.float64))


def ulp32(y: np.ndarray) -> np.ndarray:
    """One fp32 ulp at the real value y: 2^(floor(log2 |y|) - 23), at least 2^-149."""
    _, e = np.frexp(np.abs(np.asarray(y, dtype=np.float64)))
    return np.ldexp(1.0, np.maximum(e - 1, -126) - 23)


FLT_MAX = float(np.finfo(np.float32).max)
EX2_OVERFLOW = 128.0   # ex2.approx of an argument >= 128 is +inf (2^128 is past the fp32 range)
NORMAL_A = 125.0       # below this power argument 1 / (1 + 2^a) stays a normal fp32 number: the relative bounds hold


def ex2_ends(a: np.ndarray):
    """Bounds (float32 lo, hi) of ex2.approx.ftz(a) for fp32 arguments a (float64 in): within EPS_EX2 of 2^a and an
    fp32 number, +inf for a >= EX2_OVERFLOW or where the value passes the fp32 range, +0 where it is below 2^-126
    (the .ftz flush).  Both ends are monotone in the result, so they bound every value the instruction may return."""
    a = np.asarray(a, dtype=np.float64)
    p = np.exp2(np.minimum(a, 1000.0))
    lo_v, hi_v = p * (1 - EPS_EX2), p * (1 + EPS_EX2)
    over = a >= EX2_OVERFLOW
    lo = np.where(over | (lo_v > FLT_MAX), np.float32(np.inf), f32_down(np.minimum(lo_v, FLT_MAX)))
    hi = np.where(over, np.float32(np.inf), f32_up(hi_v))
    tiny = np.float32(2.0 ** -126)
    return np.where(lo < tiny, np.float32(0), lo).astype(np.float32), np.where(hi < tiny, np.float32(0), hi).astype(np.float32)


def sigmoid_f32_ends(a: np.ndarray):
    """Bounds (float32 lo, hi) of sigmoid_score's __frcp_rn(__fadd_rn(1, ex2.approx.ftz(a))) for its power argument
    a = fl(-l * fl32(log2 e)): the sum and the reciprocal are correctly rounded (the build keeps denormals, so a
    reciprocal below 2^-126 is a subnormal, not +0) and decreasing in the power, so ex2_ends' ends give the ends.
    An infinite power gives +0."""
    p_lo, p_hi = ex2_ends(a)

    def s_of(p):
        with np.errstate(over="ignore"):
            return (np.float32(1) / (np.float32(1) + p).astype(np.float32)).astype(np.float32)

    return s_of(p_hi), s_of(p_lo)


SQRT1_2_F32 = np.float32(0.70710678118654752)   # the constant gelu_erf multiplies by (fm_kernel.cuh)
ERFF_ULP = 2                                    # erff: 2 ulp (CUDA C++ Programming Guide, standard functions)


def gelu_neg_f32(v: np.ndarray):
    """Bounds (float32 lo, hi) of the kernel's fp32 GELU 0.5f * v * (1.0f + erff(v * 0.70710678f)) before its bf16
    rounding, for v < 0 (fp32 values; float64 in).

    Below zero a relative bound cannot hold: 1 + erff(t) cancels, and the result keeps the absolute error of erff.  So
    the bound follows the kernel's steps, and every step but erff is a known rounding:
      t = fl(v * fl32(1/sqrt 2)) is computed exactly (the product of two fp32 numbers is exact in float64);
      e = erff(t) is an fp32 number within ERFF_ULP ulp of erf(t), and in [-1, 1]: e in [up(erf(t) - 2u),
          down(erf(t) + 2u)] with u = ulp32(erf(t)) -- for erf(t) in (-1, -1/2] that is an absolute 2^-23 error;
      s = fl(1 + e) is increasing in e (exact for e in [-1, -1/2], Sterbenz);
      h = fl(fl(0.5 v) * s) is decreasing in s for v < 0 (0.5 v is exact).
    Every step is monotone, so the two ends of e run through the kernel's own roundings give the ends of h; then the
    bf16 RNE, also monotone.  Against the real GELU(v) the interval is about |h - GELU(v)| <= 1/2 |v| (2 ulp(erf(t)) +
    |d erf/dt| * |t - v / sqrt 2|) + 2^-24 |GELU(v)| wide, the suggested first-order form; here it is exact for any erff
    within its documented bound.  Where erff may return -1 (t below about -4.1, v below about -5.8) s is 0 and the
    interval admits the -0 the kernel writes, while the real value is a normal bf16 number down to v = -13 or so;
    torch's fp32 GELU does the same."""
    from scipy.special import erf

    v = np.asarray(v, dtype=np.float64)
    assert (v < 0).all()
    t = (v * float(SQRT1_2_F32)).astype(np.float32).astype(np.float64)
    e = erf(t)
    du = ERFF_ULP * ulp32(e)
    e_lo = np.maximum(f32_up(e - du), np.float32(-1))
    e_hi = np.minimum(f32_down(e + du), np.float32(1))
    half = (0.5 * v).astype(np.float32)

    def h_of(e32):
        s = (np.float32(1) + e32).astype(np.float32)
        return (half * s).astype(np.float32)

    return h_of(e_hi), h_of(e_lo)


def gemm1_reference(h_bits: np.ndarray, w_down: np.ndarray, b_down: Optional[np.ndarray], what: str) -> Rounded:
    """y = RNE(h . w_down^T + b_down) for the given h (bf16 bits) -- exact."""
    h = bits_to_f64(h_bits)
    assert_exact_sums(h, w_down, b_down, what)
    v = h @ w_down.T
    if b_down is not None:
        v = v + b_down[None, :]
    b = f64_to_bf16(v)
    return Rounded(b, b, v)


# ----------------------------------------------------------------------------- combine reference
def combine_tokens(y_of: np.ndarray, kept: np.ndarray, pw_bits: np.ndarray, mcw: np.ndarray) -> Rounded:
    """out [n, H] for n tokens: y_of bf16 bits [n, k, H] (the y row of each pick; ignored where not kept), kept bool
    [n, k], pw_bits bf16 [n, k] (topk_w), mcw fp32 [n].
      k == 1: out = y, unscaled; a dropped pick gives +0.
      k >= 2: term_j = RNE(pw_j * RNE(__fdividef(y_j, mcw))), out = bf16 accumulation of the kept terms in pick order
              from +0, each add rounded to fp32 and then to bf16 (combine_rows; for k = 2 the order is immaterial).
    Only __fdividef is approximate (EPS_DIV); both ends of every step go through the same roundings."""
    n, k, H = y_of.shape
    if k == 1:
        b = np.where(kept[:, :, None], y_of, 0).astype(np.uint16)[:, 0]
        return Rounded(b, b, bits_to_f64(b))
    m = np.asarray(mcw, dtype=np.float32).astype(np.float64)[:, None]
    acc_lo = np.zeros((n, H))
    acc_hi = np.zeros((n, H))
    real = np.zeros((n, H))   # the combine in real arithmetic, for the rounding statistics
    for j in range(k):
        y = bits_to_f64(y_of[:, j])
        q = y / m
        qa, qb = q * (1 - EPS_DIV), q * (1 + EPS_DIV)
        ql_b, qh_b = f64_to_bf16(np.minimum(qa, qb)), f64_to_bf16(np.maximum(qa, qb))
        assert (order_key(qh_b) - order_key(ql_b) <= 1).all(), "combine: RNE(y / mcw) interval wider than one ulp"
        ql, qh = bits_to_f64(ql_b), bits_to_f64(qh_b)
        pw = bits_to_f64(pw_bits[:, j])[:, None]
        tl, th = bits_to_f64(f64_to_bf16(pw * ql)), bits_to_f64(f64_to_bf16(pw * qh))
        keep = kept[:, j][:, None]
        real += np.where(keep, pw * q, 0.0)
        acc_lo = np.where(keep, bits_to_f64(f64_to_bf16(acc_lo + tl)), acc_lo)
        acc_hi = np.where(keep, bits_to_f64(f64_to_bf16(acc_hi + th)), acc_hi)
    return Rounded(f64_to_bf16(acc_lo), f64_to_bf16(acc_hi), real)


def combine_routed(y_of: np.ndarray, kept: np.ndarray, w_bits: np.ndarray) -> np.ndarray:
    """out bf16 bits [n, H] on the caller's (or a gated launch's) routing, mcw = 1: y_of bf16 bits [n, k, H] (ignored
    where not kept), kept [n, k], w_bits bf16 [n, k].  out[t] is the bf16 accumulation, in pick order from +0, of
    RNE(w~_j * y_j) over the kept picks, k = 1 included: each term is a single rounding of an exact product, each add
    rounds to fp32 and then to bf16, so the whole output is exact (no __fdividef interval)."""
    n, k, H = y_of.shape
    acc = np.zeros((n, H))
    for j in range(k):
        term = bits_to_f64(f64_to_bf16(bits_to_f64(w_bits[:, j])[:, None] * bits_to_f64(y_of[:, j])))
        acc = np.where(kept[:, j][:, None], bits_to_f64(f64_to_bf16(acc + term)), acc)
    return f64_to_bf16(acc)


def add_shared(r: Rounded, s_bits: np.ndarray) -> Rounded:
    """out = rne_bf16(fl32(r) + fl32(s)): a shared expert's s rows (bf16 bits [n, H]) added to the routed result r after
    r is rounded.  The sum of two bf16 numbers is exact in float64 and rounds once to fp32, then to bf16; the map is
    monotone in r, so the ends of r's interval map to the ends of out's.  `exact` is the sum before those roundings (at
    r's lower end), so rounded_count counts the elements that round in this step."""
    s = bits_to_f64(s_bits)
    lo = bits_to_f64(r.lo) + s
    return Rounded(f64_to_bf16(lo), f64_to_bf16(bits_to_f64(r.hi) + s), lo)


# ----------------------------------------------------------------------------- statistics
class Stats:
    """Per stage: elements checked, elements whose exact value needed rounding, intervals of nonzero width."""

    def __init__(self):
        self.d: Dict[str, np.ndarray] = {}

    def add(self, stage: str, checked: int, rounded: int = 0, wide: int = 0) -> None:
        self.d.setdefault(stage, np.zeros(3, np.int64))
        self.d[stage] += (checked, rounded, wide)

    def merge(self, other: "Stats") -> None:
        for s, v in other.d.items():
            self.d.setdefault(s, np.zeros(3, np.int64))
            self.d[s] += v

    def line(self) -> str:
        return "; ".join(f"{s}: {v[0]} checked, {v[1]} rounded, {v[2]} wide" for s, v in self.d.items())


def rounded_count(r: Rounded) -> int:
    """Elements whose exact (or midpoint) value is not the bf16 value it was rounded to."""
    return int((bits_to_f64(r.lo) != r.exact).sum())


# ----------------------------------------------------------------------------- checkers
def _interval_check(got_bits: np.ndarray, r: Rounded, what: str, labels: Sequence[str],
                    index_of=lambda i: i, max_width: Optional[int] = 1) -> int:
    """got inside [lo, hi] elementwise (+0 == -0); the interval is at most `max_width` bf16 ulps wide (None: any width;
    the combine's sums can cancel, so one ulp of a term may be several of the sum).  Returns the number of intervals of
    nonzero width."""
    g, lo, hi = order_key(got_bits), order_key(r.lo), order_key(r.hi)
    width = hi - lo
    narrow = width if r.wide_ok is None else np.where(r.wide_ok, 0, width)
    assert (width >= 0).all() and (max_width is None or (narrow <= max_width).all()), (
        f"{what}: reference interval wider than one bf16 ulp at {_where(np.argwhere((width < 0) | (narrow > 1))[0], labels, index_of)}")
    bad = (g < lo) | (g > hi)
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements outside the reference; first at "
                             f"{_where(i, labels, index_of)}: device {_fmt(got_bits[i])}, reference "
                             f"[{_fmt(r.lo[i])}, {_fmt(r.hi[i])}]")
    return int((width > 0).sum())


def _where(i, labels, index_of) -> str:
    i = index_of(tuple(int(v) for v in i))
    return ", ".join(f"{n} {v}" for n, v in zip(labels, i))


def check_topk(got: np.ndarray, ref: RouterRef, what: str = "topk_idx") -> None:
    bad = (got != ref.topk).any(axis=1)
    if bad.any():
        t = int(np.flatnonzero(bad)[0])
        j = int(np.flatnonzero(got[t] != ref.topk[t])[0])
        raise AssertionError(f"{what}: {int(bad.sum())} tokens differ; first token {t} pick {j}: device {got[t].tolist()}, "
                             f"reference {ref.topk[t].tolist()} (logits of those experts: "
                             f"{ref.logits[t, got[t]].tolist()} vs {ref.logits[t, ref.topk[t]].tolist()})")


def check_equal(got: np.ndarray, want: np.ndarray, what: str, labels: Sequence[str], signed_zero: bool = True) -> None:
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    bad = got != want
    if not signed_zero and got.dtype == np.uint16:   # an exact zero sum may carry either sign
        bad &= order_key(got) != order_key(want)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        gv, wv = (_fmt(got[i]), _fmt(want[i])) if got.dtype == np.uint16 else (got[i], want[i])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} differ; first at "
                             f"{', '.join(f'{n} {v}' for n, v in zip(labels, i))}: device {gv}, reference {wv}")


@dataclasses.dataclass
class Device:
    """What one launch left behind (host copies); `n` tokens valid."""
    out: np.ndarray = None                 # bf16 bits [n, H]
    topk_idx: np.ndarray = None            # [n, k]
    topk_w: np.ndarray = None              # bf16 bits [n, k]
    mcw: np.ndarray = None                 # fp32 [n]
    gate_out: Optional[np.ndarray] = None  # bf16 bits [n, E] (None on the caller's routing)
    slot: np.ndarray = None                # [n, k]
    counts: np.ndarray = None              # [E]
    recv_cnt: Optional[np.ndarray] = None
    recv_x: Optional[np.ndarray] = None    # [E, pEC, H] or None (the dense path copies nothing)
    hidden: np.ndarray = None              # [E, pEC, P]
    ret_y: Optional[np.ndarray] = None     # [E, pEC, H] (gather path) or None


@dataclasses.dataclass
class SharedRecord:
    """What a launch left of the shared expert (bf16 bits, the first n rows)."""
    h_s: np.ndarray   # [n, Ps]
    y_s: np.ndarray   # [n, H]


def shared_stage(x: np.ndarray, shared: Experts, rec: Optional[SharedRecord] = None,
                 stats: Optional[Stats] = None) -> SharedRecord:
    """h_s against the shared expert's GEMM0 of the tokens x (float64 [n, H]), then y_s bit for bit against GEMM1 of
    the record's own h_s, so a failure names the GEMM that broke.  Without `rec`, the reference's own record (an
    interval's lower end).  `stats` gets both stages."""
    st = stats if stats is not None else Stats()
    h = shared.h(0, x, "GEMM0 of the shared expert")
    rec = rec if rec is not None else SharedRecord(h.lo, None)
    assert rec.h_s.shape == h.lo.shape, f"h_s: shape {rec.h_s.shape}, expected {h.lo.shape}"
    st.add("h_s", h.lo.size, rounded_count(h), _interval_check(rec.h_s, h, "h_s (shared expert)", ("token", "column")))
    y = shared.y(0, rec.h_s, "GEMM1 of the shared expert")
    if rec.y_s is None:
        rec.y_s = y.lo
    check_equal(rec.y_s, y.lo, "y_s (shared expert)", ("token", "column"), signed_zero=False)
    st.add("y_s", y.lo.size, rounded_count(y))
    return rec


# ----------------------------------------------------------------------------- one launch, reference and checker
def reference_launch(route: str, inp: ExactInputs, EC: int, n: int, *, routing=None, router=None, score_bias=None,
                     shared: Optional[Experts] = None, stats: Optional[Stats] = None):
    """(Device, SharedRecord or None) of one launch over the first n tokens computed by the reference itself (interval
    midpoints for the routing, lower ends for h): what a correct kernel could have produced.  The planted-fault tests
    start from it.  Arguments as check_launch's; `stats` gets what checking the record would count."""
    dev, rec, _ = _launch(route, inp, EC, n, None, None, routing, router, score_bias, shared, stats)
    return dev, rec


def check_launch(route: str, inp: ExactInputs, EC: int, n: int, dev: Device, rec: Optional[SharedRecord] = None, *,
                 routing=None, router=None, score_bias=None, shared: Optional[Experts] = None,
                 stats: Optional[Stats] = None) -> int:
    """Every stage of one launch over the first n tokens of `inp`, in pipeline order, at capacity EC.  `route`:
      "router"  the built-in softmax router: topk_idx, gate_out, topk_w and mcw against router_reference, the combine
                of combine_tokens (k = 1 unscaled);
      "routed"  the caller's `routing` = (topk_idx, topk_w) of at least n tokens: topk_idx sanitized, topk_w =
                rne_bf16(w), mcw = 1, the combine of combine_routed;
      "gated"   the rule `router` with `score_bias`: exact_gated.check_gated_routing, then the routed checks on the
                device's own routing.
    Then, the same for every route: slot / counts / recv_cnt, recv_x, h of every expert (through inp.experts), y from
    the device's own h (ret_y on the gather path), out and the rows without a kept pick (+0); with a `shared` expert
    (record `rec`) h_s, y_s and out = rne(r + s).  GEMM1 and the combine are referenced from the device's own values,
    so a failure names the stage that broke.  Returns the gated route's ambiguous tokens (0 elsewhere)."""
    return _launch(route, inp, EC, n, dev, rec, routing, router, score_bias, shared, stats)[2]


def _launch(route, inp, EC, n, dev, rec, routing, router, score_bias, shared, stats):
    """check_launch's walk; with dev = None every stage first takes the reference's value (reference_launch)."""
    cfg, experts = inp.cfg, inp.experts
    E, k, H, P = cfg.E, cfg.k, cfg.H, cfg.P
    st = stats if stats is not None else Stats()
    build = dev is None
    x = inp.x64[:n]
    rows = np.arange(n)[:, None]
    amb = 0
    if route == "router":
        ref = router_reference(x, inp.wg_eff64, k)
        if build:
            p_mid = 0.5 * (ref.p_lo + ref.p_hi)
            mcw = np.zeros(n, np.float32)
            for j in range(k):
                mcw = (mcw + p_mid[rows[:, 0], ref.topk[:, j]].astype(np.float32)).astype(np.float32)
            dev = Device(topk_idx=ref.topk.copy(), topk_w=ref.go_lo[rows, ref.topk], mcw=mcw, gate_out=ref.go_lo.copy())
        check_topk(dev.topk_idx, ref)
        st.add("topk_idx", ref.topk.size)
        w1 = _interval_check(dev.gate_out, Rounded(ref.go_lo, ref.go_hi, 0.5 * (ref.p_lo + ref.p_hi)), "gate_out",
                             ("token", "expert"))
        st.add("gate_out", ref.go_lo.size, int((ref.p_lo != bits_to_f64(ref.go_lo)).sum()), w1)
        check_equal(dev.topk_w, dev.gate_out[rows, dev.topk_idx], "topk_w vs gate_out[t, topk_idx]", ("token", "pick"))
        st.add("topk_w", dev.topk_w.size)
        lo, hi = ref.mcw_bounds()
        bad = ~((dev.mcw >= lo) & (dev.mcw <= hi))
        assert not bad.any(), (f"mcw: token {int(np.flatnonzero(bad)[0])}: device {dev.mcw[bad][0]!r} outside "
                               f"[{lo[bad][0]!r}, {hi[bad][0]!r}]")
        st.add("mcw", n)
    else:
        if route == "gated":
            from tests import exact_gated as eg

            if build:
                picks, w, gate_out = eg.reference_routing(router, score_bias, k, x, inp.wg_eff64)
                dev = Device(topk_idx=picks, topk_w=f32_to_bf16(w), mcw=np.ones(n, np.float32), gate_out=gate_out)
            amb = eg.check_gated_routing(x @ inp.wg_eff64.T, score_bias, router, k, dev.topk_idx, dev.gate_out,
                                         dev.topk_w, (x, inp.wg_eff64))
            routing = (dev.topk_idx, weights_f32(dev.topk_w))
        run = sanitize(routing[0][:n], E)
        w_bits = f32_to_bf16(np.asarray(routing[1][:n], dtype=np.float32))
        if build and route == "routed":
            dev = Device(topk_idx=run, topk_w=w_bits, mcw=np.ones(n, np.float32))
        check_equal(dev.topk_idx, run, "topk_idx (the caller's, invalid ones -1)", ("token", "pick"))
        check_equal(dev.topk_w, w_bits, "topk_w = rne_bf16(w)", ("token", "pick"))
        check_equal(dev.mcw, np.ones(n, np.float32), "mcw = 1", ("token",))
        st.add("routing tables", 3 * run.size)

    topk = dev.topk_idx
    slot, counts, recv_cnt, kept = slots_from_routing(topk, E, EC)
    rmax = max(1, int(recv_cnt.max(initial=0)))
    if build:
        dev.slot, dev.counts, dev.recv_cnt = slot, counts, recv_cnt
        dev.recv_x, dev.ret_y = np.zeros((E, rmax, H), np.uint16), np.zeros((E, rmax, H), np.uint16)
        dev.hidden = np.zeros((E, rmax, P), np.uint16)
    check_equal(dev.slot, slot, "slot", ("token", "pick"))
    check_equal(dev.counts, counts, "counts", ("expert",))
    if dev.recv_cnt is not None:
        check_equal(dev.recv_cnt, recv_cnt, "recv_cnt", ("expert",))
    st.add("slot/counts/recv_cnt", slot.size + 2 * E)

    toks = packet_tokens(topk, slot, E, EC)
    xb = f64_to_bf16(x)
    y_ref = np.zeros((E, rmax, H), np.uint16)
    for e in range(E):
        c = len(toks[e])
        if c == 0:
            continue
        if build:
            dev.recv_x[e, :c] = xb[toks[e]]
        if dev.recv_x is not None:
            check_equal(dev.recv_x[e, :c], xb[toks[e]], f"recv_x of expert {e}", ("slot", "column"))
            st.add("recv_x", c * H)
        h = experts.h(e, x[toks[e]], f"GEMM0 of expert {e}")
        if build:
            dev.hidden[e, :c] = h.lo
        w = _interval_check(dev.hidden[e, :c], h, f"hidden of expert {e}", ("slot", "column"))
        st.add("hidden", c * P, rounded_count(h), w)
        y = experts.y(e, dev.hidden[e, :c], f"GEMM1 of expert {e}")
        y_ref[e, :c] = y.lo
        if build:
            dev.ret_y[e, :c] = y.lo
        if dev.ret_y is not None:
            check_equal(dev.ret_y[e, :c], y.lo, f"ret_y of expert {e}", ("slot", "column"), signed_zero=False)
            st.add("ret_y", c * H, rounded_count(y))
        else:
            st.add("y (in the fused epilogue)", 0, rounded_count(y))

    y_of = y_ref[np.where(kept, topk, 0), np.where(kept, slot, 0)]          # [n, k, H]
    if route == "router":
        r = combine_tokens(y_of, kept, dev.topk_w, dev.mcw)
    else:   # exact; `exact` the combine in real arithmetic, for the rounding statistics
        out = combine_routed(y_of, kept, dev.topk_w)
        r = Rounded(out, out, (np.where(kept, bits_to_f64(dev.topk_w), 0.0)[:, :, None] * bits_to_f64(y_of)).sum(1))
    none = ~kept.any(axis=1)
    empty, what = np.zeros((int(none.sum()), H), np.uint16), "out"
    if shared is not None:
        rec = shared_stage(x, shared, rec, st)
        r, what = add_shared(r, rec.y_s), "out = rne(r + s)"
        empty = add_shared(Rounded(empty, empty, 0), rec.y_s[none]).lo
    if build:
        dev.out = r.lo
    w = _interval_check(dev.out, r, what, ("token", "column"), max_width=None)
    st.add(what, dev.out.size, rounded_count(r), w)
    if none.any():
        check_equal(dev.out[none], empty, f"{what} rows of tokens without a kept pick (r = +0)", ("row", "column"),
                    signed_zero=shared is None)
        st.add("rows without a kept pick", int(none.sum()) * H)
    return dev, rec, amb


def check_preconditions(inp: ExactInputs, EC: int, min_h_rounded: float, min_out_rounded: float,
                        n: Optional[int] = None, dense: bool = False) -> Stats:
    """Check the reference's own router launch (the dense path without recv_x) and assert the rounding shares:
    inputs that never round do not test RNE.  Returns the statistics."""
    n = inp.cfg.S if n is None else n
    dev, _ = reference_launch("router", inp, EC, n)
    if dense:
        dev.recv_x = None
    st = Stats()
    check_launch("router", inp, EC, n, dev, stats=st)
    zero = np.zeros(3, np.int64)   # (a call with no tokens has neither)
    hs, os_ = st.d.get("hidden", zero), st.d.get("out", zero)
    if hs[0]:
        assert hs[1] >= min_h_rounded * hs[0], f"only {hs[1]} of {hs[0]} h elements needed rounding"
    if os_[0] and inp.cfg.k > 1:
        assert os_[1] >= min_out_rounded * os_[0], f"only {os_[1]} of {os_[0]} out elements needed rounding"
    return st


# ----------------------------------------------------------------------------- launches on the GPU
MAX_AMBIGUOUS = 0.01   # gated tokens whose picks the intervals cannot decide (their later stages are still checked)


def gather_path(cfg: MoEConfig, env=None) -> bool:
    """The launch writes y rows to ret_y and combines them apart (FM_FUSED_COMBINE=0, or k > 2)."""
    return (os.environ if env is None else env).get("FM_FUSED_COMBINE") == "0" or cfg.k > 2


def dense_path(cfg: MoEConfig, env=None) -> bool:
    """E = 1 takes the dense path, which reads x in place (no recv_x), unless FM_DENSE_E1=0."""
    return cfg.E == 1 and (os.environ if env is None else env).get("FM_DENSE_E1", "1") != "0"


class Launcher:
    """The inputs of one route uploaded to one context, which was created under the current environment: `launch`
    runs the route's forward, `read` reads a launch back as check_launch takes it, `check` checks it."""

    def __init__(self, ctx, route: str, inp: ExactInputs, *, routing=None, router=None, score_bias=None):
        dev, cfg = ctx.device, inp.cfg
        self.ctx, self.route, self.inp, self.cfg = ctx, route, inp, cfg
        self.routing, self.router, self.score_bias = routing, router, score_bias
        x, self.wg, self.we, self.bu, self.bd = inp.device(dev)
        self.x = x.reshape(cfg.S, cfg.H)
        if routing is not None:
            self.idx, self.w = (torch.from_numpy(a).to(dev) for a in routing)
        self.sb = None if score_bias is None else torch.from_numpy(score_bias).to(dev)
        self.gather, self.dense = gather_path(cfg), dense_path(cfg)

    def launch(self, n: Optional[int], shared=None, out=None, n_tokens=None, x=None):
        """The forward of the first n tokens (of `x` when given), with a runtime.SharedExpert `shared`; n = None:
        MoEContext.forward of all S (router route)."""
        ctx, kw = self.ctx, dict(bias_up=self.bu, bias_down=self.bd, out=out)
        if n is None:
            return ctx.forward(self.x.reshape(self.inp.x.shape), self.wg, self.we, **kw)
        x = self.x[:n] if x is None else x
        m = x.shape[0]
        kw.update(n_tokens=n_tokens, shared_expert=shared)
        if self.route == "router":
            return ctx.forward_tokens(x, self.wg, self.we, **kw)
        if self.route == "routed":
            return ctx.forward_routed(x, self.idx[:m], self.w[:m], self.we, **kw)
        return ctx.forward_gated(x, self.wg, self.we, self.router, score_bias=self.sb, **kw)

    def read(self, out, n: int, shared: bool = False):
        """(Device, SharedRecord or None) of the first n tokens of the last launch, whose output is `out`."""
        ctx = self.ctx
        dev = Device(out=to_bits(out.cpu()).reshape(n, self.cfg.H), topk_idx=ctx.read("topk_idx")[:n],
                     topk_w=ctx.read("topk_w")[:n], mcw=ctx.read("mcw")[:n],
                     gate_out=None if self.route == "routed" else ctx.read("gate_out")[:n], slot=ctx.read("slot")[:n],
                     counts=ctx.read("counts"), recv_cnt=ctx.read("recv_cnt"),
                     recv_x=None if self.dense else ctx.read("recv_x"), hidden=ctx.read("hidden"),
                     ret_y=ctx.read("ret_y") if self.gather else None)
        rec = SharedRecord(ctx.read("shared_hidden")[:n], ctx.read("shared_y")[:n]) if shared else None
        return dev, rec

    def check(self, dev: Device, rec: Optional[SharedRecord], n: int, shared: Optional[Experts] = None,
              stats: Optional[Stats] = None) -> int:
        return check_launch(self.route, self.inp, self.cfg.EC_of(n), n, dev, rec, routing=self.routing,
                            router=self.router, score_bias=self.score_bias, shared=shared, stats=stats)

    def run(self, n: int, shared: Optional[Experts] = None, stats: Optional[Stats] = None):
        """launch, read and check one forward of the first n tokens; returns (Device, SharedRecord, ambiguous)."""
        out = self.launch(n, None if shared is None else shared_expert(shared, self.ctx.device))
        self.ctx.synchronize()
        dev, rec = self.read(out, n, shared is not None)
        return dev, rec, self.check(dev, rec, n, shared, stats)
