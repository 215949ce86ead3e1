"""The exact-input reference (tests/exact.py) for forwards on the caller's routing (fm_moe_forward_routed).

A pick of -1 is no expert: it takes no slot, is not counted and moves no row (its slot reads INT32_MAX).  The combine
is the router path's with mcw = 1: out[t] is the bf16 accumulation, in pick order from +0, of RNE(w~_j * y_j) over the
kept picks, w~ = rne_bf16(w), k = 1 included.  w~ and y are bf16 numbers, so their product is exact in fp32 and the
whole output is checked bit for bit -- there is no __fdividef interval left.  No pytest in here.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from tests import exact as ex

INT32_MAX = 2 ** 31 - 1


def routing_case(n: int, E: int, k: int, seed: int, *, skip_frac: float = 0.1, dup_frac: float = 0.1,
                 hot: int = 0, hot_frac: float = 0.5, empty=(), bad=()):
    """Seeded routing for n tokens: picks drawn from the experts not in `empty`, a `hot_frac` share of them sent to
    expert `hot` (skew that overflows its capacity), a `dup_frac` share of tokens naming one expert twice, a `skip_frac`
    share of picks set to -1, and `bad` (token, pick, value) entries written last.  Weights are fp32 in [-1, 2), with
    some exact zeros.  Returns (topk_idx int32 [n, k], topk_w float32 [n, k])."""
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


def slots_from_routing(topk: np.ndarray, E: int, EC: int):
    """slots_from_topk for routing that may hold -1 (no expert): slot [n, k] (INT32_MAX for -1), counts [E],
    recv_cnt [E] = min(counts, EC), kept [n, k] = slot < EC."""
    topk = np.asarray(topk, dtype=np.int64)
    valid = topk >= 0
    assert (topk[valid] < E).all() and (topk[~valid] == -1).all(), "expert index outside [-1, E)"
    flat, vflat = topk.reshape(-1), valid.reshape(-1)
    slot = np.full(flat.size, INT32_MAX, dtype=np.int64)
    sub = flat[vflat]
    s, counts, recv_cnt, _ = ex.slots_from_topk(sub.reshape(-1, 1), E, EC)   # ascending (token, pick) order kept
    slot[vflat] = s[:, 0]
    slot = slot.reshape(topk.shape).astype(np.int32)
    return slot, counts, recv_cnt, slot < EC


def combine_routed(y_of: np.ndarray, kept: np.ndarray, w_bits: np.ndarray) -> np.ndarray:
    """out bf16 bits [n, H]: y_of bf16 bits [n, k, H] (ignored where not kept), kept [n, k], w_bits bf16 [n, k].
    Each term RNE(w~ * y) is a single rounding of an exact product; each add rounds to fp32 and then to bf16."""
    n, k, H = y_of.shape
    acc = np.zeros((n, H))
    for j in range(k):
        term = ex.bits_to_f64(ex.f64_to_bf16(ex.bits_to_f64(w_bits[:, j])[:, None] * ex.bits_to_f64(y_of[:, j])))
        acc = np.where(kept[:, j][:, None], ex.bits_to_f64(ex.f64_to_bf16(acc + term)), acc)
    return ex.f64_to_bf16(acc)


def sanitize(topk: np.ndarray, E: int) -> np.ndarray:
    """The routing the kernel runs: indices outside [0, E) become -1."""
    t = np.asarray(topk, dtype=np.int32)
    return np.where((t >= 0) & (t < E), t, -1).astype(np.int32)


def check_routed_forward(inp: ex.ExactInputs, dev: ex.Device, topk: np.ndarray, w: np.ndarray, EC: int,
                         stats: Optional[ex.Stats] = None, shared_s: Optional[np.ndarray] = None) -> ex.Stats:
    """Every stage of one routed launch over the first n = len(topk) tokens of `inp`: the routing tables, slots,
    counts, recv_cnt, the dispatched rows, h, y (ret_y on the gather path) and out, bit for bit (GELU's h within its
    interval); rows whose picks were all skipped or dropped must be +0.  GEMM1 and the combine are referenced from
    the device's own hidden, so a failure names the stage that broke.  `shared_s`: a shared expert's s rows (bf16 bits
    [n, H]); out is then rne(r + s) (exact.add_shared), and the rows without a kept pick rne(+0 + s)."""
    cfg = inp.cfg
    E, H = cfg.E, cfg.H
    st = stats if stats is not None else ex.Stats()
    n = topk.shape[0]
    x = inp.x64[:n]
    run = sanitize(topk, E)
    ex.check_equal(dev.topk_idx, run, "topk_idx (the caller's, invalid ones -1)", ("token", "pick"))
    w_bits = ex.f32_to_bf16(np.asarray(w, dtype=np.float32))
    ex.check_equal(dev.topk_w, w_bits, "topk_w = rne_bf16(w)", ("token", "pick"))
    ex.check_equal(dev.mcw, np.ones(n, np.float32), "mcw = 1", ("token",))
    st.add("routing tables", 3 * run.size)
    slot, counts, recv_cnt, kept = slots_from_routing(run, E, EC)
    ex.check_equal(dev.slot, slot, "slot", ("token", "pick"))
    ex.check_equal(dev.counts, counts, "counts", ("expert",))
    if dev.recv_cnt is not None:
        ex.check_equal(dev.recv_cnt, recv_cnt, "recv_cnt", ("expert",))
    st.add("slot/counts/recv_cnt", slot.size + 2 * E)
    toks = ex.packet_tokens(run, slot, E, EC)
    xb = ex.f64_to_bf16(x)
    y_ref = np.zeros((E, max(1, int(recv_cnt.max(initial=0))), H), np.uint16)
    for e in range(E):
        c = len(toks[e])
        if c == 0:
            continue
        ex.check_equal(dev.recv_x[e, :c], xb[toks[e]], f"recv_x of expert {e}", ("slot", "column"))
        st.add("recv_x", c * H)
        h_ref = ex.gemm0_reference(x[toks[e]], inp.w_up64[e], None if inp.bu is None else inp.bias64("up")[e],
                                   cfg.hidden_act, f"GEMM0 of expert {e}")
        h_dev = dev.hidden[e, :c]
        if cfg.hidden_act == 0:
            ex.check_equal(h_dev, h_ref.lo, f"hidden of expert {e}", ("slot", "column"), signed_zero=False)
        else:
            ex._interval_check(h_dev, h_ref, f"hidden of expert {e}", ("slot", "column"))
        st.add("hidden", h_dev.size, ex.rounded_count(h_ref))
        y = ex.gemm1_reference(h_dev, inp.w_down64[e], None if inp.bd is None else inp.bias64("down")[e],
                               f"GEMM1 of expert {e}")
        y_ref[e, :c] = y.lo
        if dev.ret_y is not None:
            ex.check_equal(dev.ret_y[e, :c], y.lo, f"ret_y of expert {e}", ("slot", "column"), signed_zero=False)
            st.add("ret_y", c * H)
    y_of = y_ref[np.where(kept, run, 0), np.where(kept, slot, 0)]
    out = combine_routed(y_of, kept, w_bits)
    none = ~kept.any(axis=1)
    empty, what, rounded = np.zeros((int(none.sum()), H), np.uint16), "out", 0
    if shared_s is not None:
        r = ex.add_shared(ex.Rounded(out, out, 0), shared_s)
        out, what, rounded = r.lo, "out = rne(r + s)", ex.rounded_count(r)
        empty = ex.add_shared(ex.Rounded(empty, empty, 0), shared_s[none]).lo
    ex.check_equal(dev.out, out, what, ("token", "column"), signed_zero=False)
    st.add(what, dev.out.size, rounded)
    if none.any():
        ex.check_equal(dev.out[none], empty, f"{what} rows of tokens whose picks were all skipped or dropped (r = +0)",
                       ("row", "column"), signed_zero=shared_s is None)
        st.add("rows without a kept pick", int(none.sum()) * H)
    return st


def reference_out(inp: ex.ExactInputs, topk: np.ndarray, w: np.ndarray, EC: int) -> np.ndarray:
    """out bf16 bits [n, H] of the routed forward computed by the reference alone (ReLU: exact)."""
    cfg = inp.cfg
    assert cfg.hidden_act == 0, "the GELU reference is an interval"
    E, H = cfg.E, cfg.H
    n = topk.shape[0]
    x = inp.x64[:n]
    run = sanitize(topk, E)
    slot, _, recv_cnt, kept = slots_from_routing(run, E, EC)
    toks = ex.packet_tokens(run, slot, E, EC)
    y_ref = np.zeros((E, max(1, int(recv_cnt.max(initial=0))), H), np.uint16)
    for e in range(E):
        c = len(toks[e])
        if c == 0:
            continue
        h = ex.gemm0_reference(x[toks[e]], inp.w_up64[e], None if inp.bu is None else inp.bias64("up")[e], 0, "GEMM0")
        y_ref[e, :c] = ex.gemm1_reference(h.lo, inp.w_down64[e], None if inp.bd is None else inp.bias64("down")[e],
                                          "GEMM1").lo
    y_of = y_ref[np.where(kept, run, 0), np.where(kept, slot, 0)]
    return combine_routed(y_of, kept, ex.f32_to_bf16(np.asarray(w, dtype=np.float32)))
