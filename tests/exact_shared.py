"""The exact-input reference (tests/exact.py) for the shared expert (fm_moe_forward_shared).

A shared expert is a dense FFN of intermediate size Ps on every token: h_s = RNE(act(x W_up_s^T + b_up_s)) [n, Ps] and
s = y_s = RNE(h_s W_down_s^T + b_down_s) [n, H], with a routed expert's arithmetic; the launch's output is
out = rne_bf16(fl32(r) + fl32(s)) (exact.add_shared), r the routed result the same call writes without one.  Its weights
are drawn on the routed experts' grids, so h_s and y_s are exact under the conditions of exact.py: h_s bit for bit for
ReLU and inside the GELU interval, y_s bit for bit from the device's own h_s.

`regime` states where the kernel's shared-expert items fall (column tiles TN0s of Ps and TN1 of H, their partial last
tiles, row blocks s_rb, tokens per CTA, and the work-list block the GEMM1 items follow); tests/test_shared_exact_cases.py
pins its constants to the sources.  No pytest in here.
"""
from __future__ import annotations

import dataclasses
import functools
from typing import Optional

import numpy as np
import torch

from tests import exact as ex
from tests import exact_gated as eg
from tests import exact_routed as er

# ----------------------------------------------------------------------------- the kernel's tiling (fm_kernel.cuh)
BLOCK_M = 128   # token rows per tile: a row block of the shared expert
BLOCK_N = 256   # output columns per tile


@dataclasses.dataclass(frozen=True)
class Regime:
    TN0s: int            # GEMM0 column tiles, ceil(Ps / BLOCK_N)
    ps_tail: int         # columns of the last, partial Ps tile (0: none)
    TN1: int             # GEMM1 column tiles, ceil(H / BLOCK_N)
    h_tail: int          # columns of the last, partial H tile (0: none)
    s_rb: int            # row blocks of tokens, ceil(n / BLOCK_M)
    tpc: int             # tokens per CTA, ceil(n / grid)
    rb_per_cta: int      # most row blocks one CTA's tokens touch (wait_shared_rows' loop)
    split_blk: int       # routed work-list blocks ahead of the shared GEMM1 items

    def line(self) -> str:
        return (f"TN0s {self.TN0s}{f' (tail {self.ps_tail})' if self.ps_tail else ''}, TN1 {self.TN1}"
                f"{f' (tail {self.h_tail})' if self.h_tail else ''}, s_rb {self.s_rb}, tpc {self.tpc}, "
                f"row blocks per CTA {self.rb_per_cta}, split_blk {self.split_blk}")


def split_blk(E: int, lag: int = -1) -> int:
    """Leading local GEMM0 blocks of a one-rank work list (fm_create): all E GEMM0 blocks, or with FM_G1_LAG = lag in
    [1, E) the GEMM0 blocks up to the first GEMM1 block, which comes after GEMM0 of unit lag."""
    kinds = []
    if 1 <= lag < E:
        for i in range(E):
            kinds.append(0)
            if i >= lag:
                kinds.append(1)
    else:
        kinds = [0] * E + [1] * E
    return kinds.index(1)


def regime(H: int, Ps: int, n: int, grid: int, E: int, lag: int = -1) -> Regime:
    tpc = -(-n // grid)
    rbs = 0
    for c in range(grid):
        t0, nt = c * tpc, max(0, min(tpc, n - c * tpc))
        if nt:
            rbs = max(rbs, (t0 + nt - 1) // BLOCK_M - t0 // BLOCK_M + 1)
    return Regime(-(-Ps // BLOCK_N), Ps % BLOCK_N, -(-H // BLOCK_N), H % BLOCK_N, -(-n // BLOCK_M), tpc, rbs,
                  split_blk(E, lag))


# ----------------------------------------------------------------------------- inputs
@dataclasses.dataclass
class SharedInputs:
    """Exact shared-expert weights: w bf16 [2, Ps, H] ([0] = W_up_s, [1] flat-viewed as W_down_s [H, Ps]), biases or
    None; the float64 copies are made once."""
    w: torch.Tensor
    bu: Optional[torch.Tensor]
    bd: Optional[torch.Tensor]

    @property
    def Ps(self) -> int:
        return int(self.w.shape[1])

    @functools.cached_property
    def w_up64(self) -> np.ndarray:      # [Ps, H]
        return self.w[0].double().numpy()

    @functools.cached_property
    def w_down64(self) -> np.ndarray:    # [H, Ps]
        _, Ps, H = self.w.shape
        return self.w[1].reshape(-1).reshape(H, Ps).double().numpy()

    @functools.cached_property
    def bu64(self) -> Optional[np.ndarray]:
        return None if self.bu is None else self.bu.double().numpy()

    @functools.cached_property
    def bd64(self) -> Optional[np.ndarray]:
        return None if self.bd is None else self.bd.double().numpy()

    def device(self, dev):
        """The SharedExpert on `dev` (the weights uploaded in one piece)."""
        from flashmoe_b200.runtime import SharedExpert

        return SharedExpert(self.w.to(dev), None if self.bu is None else self.bu.to(dev),
                            None if self.bd is None else self.bd.to(dev))


def shared_inputs(H: int, Ps: int, seed: int, *, up_range: int = 8, down_range: int = 4, bias: bool = False,
                  gelu_friendly: bool = False, down_density: float = 1.0) -> SharedInputs:
    """Seeded exact shared weights on exact.exact_inputs' grids: W_up_s integers in [-up_range, up_range] * 2^-3 (with
    `gelu_friendly`, sparse ones in [1, up_range] at density 4 / H, as exact_inputs draws W_up), W_down_s integers in
    [-down_range, down_range] * 2^-5, kept at density `down_density` (a sparse W_down_s keeps a long GEMM1 sum exact);
    b_up_s on 2^-3 (>= 0 with `gelu_friendly`), b_down_s on 2^-8.  Drawn as int8, so that model-sized experts
    (exact_gated.LayerInputs' ranges: up_range = down_range = 2) stay cheap."""
    g = np.random.default_rng(seed)
    if gelu_friendly:
        up = g.integers(1, up_range + 1, size=(Ps, H), dtype=np.int8) * (g.random((Ps, H), dtype=np.float32) < 4.0 / H)
    else:
        up = g.integers(-up_range, up_range + 1, size=(Ps, H), dtype=np.int8)
    down = g.integers(-down_range, down_range + 1, size=(H, Ps), dtype=np.int8)
    if down_density < 1.0:
        down *= (g.random((H, Ps), dtype=np.float32) < down_density).astype(np.int8)
    w = torch.stack([torch.from_numpy(up.astype(np.int8)).float() * 2.0 ** ex.WUP_GRID,
                     (torch.from_numpy(down).float() * 2.0 ** ex.WDOWN_GRID).reshape(Ps, H)]).bfloat16()
    bu = bd = None
    if bias:
        lo = 0 if gelu_friendly else -16
        bu = torch.from_numpy(g.integers(lo, 17, size=Ps).astype(np.float32) * 2.0 ** ex.WUP_GRID).bfloat16()
        bd = torch.from_numpy(g.integers(-256, 257, size=H).astype(np.float32)
                              * 2.0 ** (ex.WUP_GRID + ex.WDOWN_GRID)).bfloat16()
    return SharedInputs(w, bu, bd)


# ----------------------------------------------------------------------------- reference and checker
@dataclasses.dataclass
class SharedRecord:
    """What a launch left of the shared expert (bf16 bits, the first n rows)."""
    h_s: np.ndarray   # [n, Ps]
    y_s: np.ndarray   # [n, H]


def shared_record(x64: np.ndarray, se: SharedInputs, act: int, stats: Optional[ex.Stats] = None) -> SharedRecord:
    """h_s and y_s of the tokens x64 [n, H] computed by the reference (GELU: the interval's lower end): what a correct
    kernel could have produced.  `stats` gets the h_s elements and those that round."""
    h = ex.gemm0_reference(x64, se.w_up64, se.bu64, act, "GEMM0 of the shared expert")
    if stats is not None:
        stats.add("h_s", h.lo.size, ex.rounded_count(h))
    return SharedRecord(h.lo, ex.gemm1_reference(h.lo, se.w_down64, se.bd64, "GEMM1 of the shared expert").lo)


def check_shared(inp, se: SharedInputs, dev_h_s: np.ndarray, dev_y_s: np.ndarray, n: int, act: int,
                 stats: Optional[ex.Stats] = None) -> ex.Stats:
    """h_s [n, Ps] against GEMM0 of the first n tokens of `inp` (ReLU bit for bit, GELU inside its interval), then y_s
    [n, H] bit for bit against GEMM1 of the device's own h_s, so a failure names the GEMM that broke.  Both references
    assert that their sums are exact in fp32."""
    st = stats if stats is not None else ex.Stats()
    assert dev_h_s.shape == (n, se.Ps), f"h_s: shape {dev_h_s.shape}, expected {(n, se.Ps)}"
    h = ex.gemm0_reference(inp.x64[:n], se.w_up64, se.bu64, act, "GEMM0 of the shared expert")
    if act == 0:
        ex.check_equal(dev_h_s, h.lo, "h_s (shared expert)", ("token", "column"), signed_zero=False)
        st.add("h_s", h.lo.size, ex.rounded_count(h))
    else:
        w = ex._interval_check(dev_h_s, h, "h_s (shared expert)", ("token", "column"))
        st.add("h_s", h.lo.size, ex.rounded_count(h), w)
    y = ex.gemm1_reference(dev_h_s, se.w_down64, se.bd64, "GEMM1 of the shared expert")
    ex.check_equal(dev_y_s, y.lo, "y_s (shared expert)", ("token", "column"), signed_zero=False)
    st.add("y_s", y.lo.size, ex.rounded_count(y))
    return st


def check_launch(route: str, inp, se: SharedInputs, dev: ex.Device, rec: SharedRecord, EC: int, act: int, *,
                 routing=None, router=None, score_bias=None, stats: Optional[ex.Stats] = None) -> int:
    """One launch with a shared expert, stage by stage: h_s and y_s (check_shared), then the route's own checker with
    out = rne(r + s) on the device's s rows -- `route` "router" (exact.check_forward), "routed" (`routing` = the
    caller's (topk_idx, topk_w)) or "gated" (`router`, `score_bias`).  Returns the gated route's ambiguous tokens."""
    n = dev.topk_idx.shape[0]
    check_shared(inp, se, rec.h_s, rec.y_s, n, act, stats)
    if route == "router":
        ex.check_forward(inp, dev, EC, n=n, stats=stats, shared_s=rec.y_s)
        return 0
    if route == "routed":
        er.check_routed_forward(inp, dev, routing[0][:n], routing[1][:n], EC, stats, shared_s=rec.y_s)
        return 0
    return eg.check_gated_forward(inp, dev, router, score_bias, EC, stats, shared_s=rec.y_s)


def reference_launch(route: str, inp, se: SharedInputs, n: int, EC: int, *, routing=None, router=None,
                     score_bias=None, stats: Optional[ex.Stats] = None):
    """(Device, SharedRecord) of one launch computed by the reference: the route's own record (exact.reference_device,
    exact_gated.routed_device / reference_device_gated) with out = rne(r + s).  The planted-fault tests start from it.
    `stats` gets the h_s and y_s elements, and the out elements that round in the r + s step."""
    act = inp.cfg.hidden_act
    if route == "router":
        dev = ex.reference_device(inp, EC, n)
    elif route == "routed":
        dev = eg.routed_device(inp, routing[0][:n], routing[1][:n], EC)
    else:
        dev = eg.reference_device_gated(inp, router, score_bias, EC, n)
    rec = shared_record(inp.x64[:n], se, act, stats)
    out = ex.add_shared(ex.Rounded(dev.out, dev.out, 0), rec.y_s)
    dev.out = out.lo
    if stats is not None:
        stats.add("out = rne(r + s)", out.lo.size, ex.rounded_count(out))
    return dev, rec
