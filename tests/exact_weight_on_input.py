"""The router weight on the input (fm_set_weight_on_input, k = 1) in the exact checks of tests/exact.py.

With the setting on, a launch keeps the routing tables of the same call with it off (topk_idx, topk_w = rne_bf16(w),
mcw = 1, slot, counts, gate_out), and from the dispatch on it is the weight-1 routed launch of the scaled rows
x'[t] = rne_bf16(x[t] * w~[t]): recv_x holds x', h comes from x', y from the device's h, and out[t] = y (bias included)
or +0 without a kept pick.  A shared expert runs on the unscaled x: out = rne(fl32(y) + fl32(s)).  check_launch and
reference_launch take exact.py's arguments; with weight_on_input=False they are exact.py's own.

The inputs (inputs()) keep every sum exact although x' has up to 8 significant bits: x in {0, 3, 5, 6, 7}, weights from
WEIGHTS (some of which make rne(x * w) round), and sparse non-negative W_up / W_gate, so no pre-activation cancels to a
tiny value whose fine bf16 grid would break the exactness of GEMM1.  No pytest in here.
"""
from __future__ import annotations

import dataclasses
from typing import Optional

import numpy as np
import torch

from flashmoe_b200.config import MoEConfig
from tests import exact as ex

# w~ values of the caller-routed cases: 97/128, 127/128 and 65/64 make rne(x * w) round for x in {3, 5, 6, 7}
# (65/64 * 5 is a tie); 0 gives zero rows
WEIGHTS = np.array([0.0, 0.75, 97 / 128, 127 / 128, 1.0, 65 / 64, 1.25, 1.5], np.float32)
X_VALUES = np.array([0.0, 3.0, 5.0, 6.0, 7.0])


def scaled_rows(x64: np.ndarray, w_bits: np.ndarray) -> np.ndarray:
    """x' = rne_bf16(x * w~) (float64 [n, H]) for the rows x (float64 bf16 values [n, H]) and w~ (bf16 bits [n, 1]): the
    product of two bf16 numbers is exact in float64 and in fp32, so this is the kernel's single rounding."""
    return ex.bits_to_f64(ex.f64_to_bf16(x64 * ex.bits_to_f64(w_bits)[:, :1]))


def _sparse(E: int, rows: int, cols: int, nz: int, vals, rng) -> np.ndarray:
    w = np.zeros((E, rows, cols))
    for e in range(E):
        for r in range(rows):
            c = rng.choice(cols, size=nz, replace=False)
            w[e, r, c] = rng.choice(vals, size=nz)
    return w


def experts(E: int, P: int, H: int, act: int, rng: np.random.Generator, bias: bool) -> ex.Experts:
    """E experts of activation `act` for non-negative inputs: W_up (and W_gate) rows with 2 entries in {1/2, 1}, W_down
    on 2^-5 with about 8 nonzeros per output column, b_up in {0, 1/2, 1}, b_down on 2^-5 (the grid of
    a ReLU expert's GEMM1 on the unscaled x)."""
    pre = [_sparse(E, P, H, 2, [0.5, 1.0], rng) for _ in range(2 if act == 2 else 1)]
    down = (rng.integers(-4, 5, size=(E, H, P)) * (rng.random((E, H, P)) < 8.0 / P)) * 2.0 ** ex.WDOWN_GRID
    w = np.stack(pre + [down.reshape(E, -1).reshape(E, P, H)], axis=1)
    bu = bd = None
    if bias:
        bu = rng.integers(0, 3, size=(E, len(pre), P)).reshape(E, -1) * 0.5
        bu = bu.reshape(E, 2, P) if act == 2 else bu
        bd = rng.integers(-32, 33, size=(E, H)) * 2.0 ** ex.WDOWN_GRID
    bf = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).bfloat16()   # noqa: E731
    return ex.Experts(bf(w), bf(bu), bf(bd), act)


def inputs(cfg: MoEConfig, seed: int, bias: bool = True) -> ex.ExactInputs:
    """Seeded exact inputs: x in X_VALUES, gate weights in [0, 2] * 2^-6 (non-negative logits: a sigmoid rule's weights
    lie in [1/2, 1)), the experts of experts()."""
    g = np.random.default_rng(seed)
    S, H, E = cfg.S, cfg.H, cfg.E
    x = g.choice(X_VALUES, size=(S, H))
    wg = g.integers(0, 3, size=(E, H)) * 2.0 ** ex.WG_GRID
    xp = experts(E, cfg.P, H, cfg.hidden_act, np.random.default_rng(seed + 1), bias)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).bfloat16()   # noqa: E731
    return ex.ExactInputs(cfg, t(x).reshape(cfg.mini_batch, cfg.sequence_len, H), t(wg.reshape(-1).reshape(H, E)), xp,
                          np.zeros(0, np.int64), np.zeros(0, np.int64))


def shared(H: int, Ps: int, act: int, seed: int, bias: bool = True) -> ex.Experts:
    """A seeded shared expert (E = 1) for inputs()."""
    return experts(1, Ps, H, act, np.random.default_rng(seed), bias)


def routing(n: int, E: int, seed: int, **kw):
    """exact.routing_case for k = 1 (skew past EC onto expert `hot`, -1 picks) with weights drawn from WEIGHTS."""
    idx, _ = ex.routing_case(n, E, 1, seed, **kw)
    return idx, np.random.default_rng(seed + 1).choice(WEIGHTS, size=(n, 1)).astype(np.float32)


def reference_launch(route: str, inp: ex.ExactInputs, EC: int, n: int, *, routing=None, router=None, score_bias=None,
                     shared: Optional[ex.Experts] = None, stats: Optional[ex.Stats] = None,
                     weight_on_input: bool = True):
    """exact.reference_launch, with the weight on the input when `weight_on_input`."""
    if not weight_on_input:
        return ex.reference_launch(route, inp, EC, n, routing=routing, router=router, score_bias=score_bias,
                                   shared=shared, stats=stats)
    dev, rec, _ = _launch(route, inp, EC, n, None, None, routing, router, score_bias, shared, stats)
    return dev, rec


def check_launch(route: str, inp: ex.ExactInputs, EC: int, n: int, dev: ex.Device,
                 rec: Optional[ex.SharedRecord] = None, *, routing=None, router=None, score_bias=None,
                 shared: Optional[ex.Experts] = None, stats: Optional[ex.Stats] = None,
                 weight_on_input: bool = True) -> int:
    """exact.check_launch, with the weight on the input when `weight_on_input` (module docstring).  Returns the gated
    route's ambiguous tokens (0 on the caller's routing)."""
    if not weight_on_input:
        return ex.check_launch(route, inp, EC, n, dev, rec, routing=routing, router=router, score_bias=score_bias,
                               shared=shared, stats=stats)
    return _launch(route, inp, EC, n, dev, rec, routing, router, score_bias, shared, stats)[2]


def _weight_one_out(inp: ex.ExactInputs, EC: int, dev: ex.Device) -> np.ndarray:
    """The weight-1 combine from the device's own h: y of each kept pick (-0 added onto +0 is +0), +0 elsewhere."""
    cfg, n = inp.cfg, dev.topk_idx.shape[0]
    slot, _, _, kept = ex.slots_from_routing(dev.topk_idx, cfg.E, EC)
    y_of = np.zeros((n, 1, cfg.H), np.uint16)
    for e, toks in enumerate(ex.packet_tokens(dev.topk_idx, slot, cfg.E, EC)):
        if len(toks):
            y_of[toks, 0] = inp.experts.y(e, dev.hidden[e, :len(toks)], f"GEMM1 of expert {e}").lo
    return ex.combine_routed(y_of, kept, ex.f32_to_bf16(np.ones((n, 1), np.float32)))


def _launch(route, inp, EC, n, dev, rec, routing, router, score_bias, shared, stats):
    cfg = inp.cfg
    assert route in ("routed", "gated") and cfg.k == 1 and cfg.E > 1, "the weight on the input: caller or gated, k = 1"
    st = stats if stats is not None else ex.Stats()
    build = dev is None
    x = inp.x64[:n]
    amb = 0
    # the routing tables are those of the call with the weight on the output, decided on the unscaled x
    if route == "gated":
        from tests import exact_gated as eg

        if build:
            picks, w, gate_out = eg.reference_routing(router, score_bias, 1, x, inp.wg_eff64)
            dev = ex.Device(topk_idx=picks, topk_w=ex.f32_to_bf16(w), mcw=np.ones(n, np.float32), gate_out=gate_out)
        amb = eg.check_gated_routing(x @ inp.wg_eff64.T, score_bias, router, 1, dev.topk_idx, dev.gate_out,
                                     dev.topk_w, (x, inp.wg_eff64))
    else:
        w_bits = ex.f32_to_bf16(np.asarray(routing[1][:n], dtype=np.float32))
        if build:
            dev = ex.Device(topk_idx=ex.sanitize(routing[0][:n], cfg.E), topk_w=w_bits, mcw=np.ones(n, np.float32))
        ex.check_equal(dev.topk_w, w_bits, "topk_w = rne_bf16(w)", ("token", "pick"))
    # from the dispatch on: the weight-1 routed launch of x' (which also checks topk_idx and mcw = 1)
    xs = inp.x64.copy()
    xs[:n] = scaled_rows(x, dev.topk_w)
    inp1 = dataclasses.replace(inp, x=ex.from_bits(ex.f64_to_bf16(xs)).reshape(inp.x.shape))
    ones = (dev.topk_idx, np.ones((n, 1), np.float32))
    if build:
        one, _ = ex.reference_launch("routed", inp1, EC, n, routing=ones, stats=st)
        one.topk_w, one.gate_out = dev.topk_w, dev.gate_out
        dev = one
        r = dev.out
    else:
        r = _weight_one_out(inp1, EC, dev) if shared is not None else dev.out
        ex.check_launch("routed", inp1, EC, n, dataclasses.replace(dev, topk_w=ex.f32_to_bf16(ones[1]), out=r),
                        routing=ones, stats=st)
    if shared is not None:   # the shared expert's term, from the unscaled x
        rec = ex.shared_stage(x, shared, rec, st)
        out = ex.add_shared(ex.Rounded(r, r, ex.bits_to_f64(r)), rec.y_s)
        if build:
            dev.out = out.lo
        ex.check_equal(dev.out, out.lo, "out = rne(y + s)", ("token", "column"), signed_zero=False)
        st.add("out = rne(y + s)", out.lo.size, ex.rounded_count(out))
    return dev, rec, amb
